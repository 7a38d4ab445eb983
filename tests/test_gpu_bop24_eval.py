"""Row f8 on the GPU: gp_bop_match labels equal to the port's (oracle/bop24_port.detection_labels), gp_bop_average_precision
bit-identical to oracle/bop24_port.average_precision, evaluate_detection end to end against the port pipeline, and the
launch counter against the launches the plan predicts (no profiler session: see tests/test_gpu_z_bop_launch_count.py)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from bop_tree import rot, spheroid, tetra, write_tree
from gigapose_b200 import _lib, bop_eval
from oracle import bop24_port
from test_bop24_eval_cpu import port_pipeline

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _report(name, obj):
    print(name, json.dumps(obj))


def _i32(a):
    a = np.ascontiguousarray(a, np.int32)
    return (C.c_int32 * max(1, len(a)))(*a.tolist())


def _f64(a):
    a = np.ascontiguousarray(a, np.float64).reshape(-1)
    return (C.c_double * len(a))(*a.tolist())


def _dev(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a, dtype), device=DEV)


def _match(groups, thr):
    """groups: dicts (obj, mssd [n_est, n_gt], mspd, valid [n_gt]); thr [n_obj, 2, T] -> labels [n_est total, 2, T]."""
    lib = _lib.load()
    T = thr.shape[2]
    est_off = np.cumsum([0] + [g["mssd"].shape[0] for g in groups])
    gt_off = np.cumsum([0] + [len(g["valid"]) for g in groups])
    mssd = _dev(np.concatenate([g["mssd"].ravel() for g in groups] + [np.zeros(1)]), np.float32)
    mspd = _dev(np.concatenate([g["mspd"].ravel() for g in groups] + [np.zeros(1)]), np.float32)
    valid = _dev(np.concatenate([g["valid"] for g in groups] + [np.zeros(1)]), np.uint8)
    ws = torch.empty(8 * thr.size + 32 * len(groups), dtype=torch.uint8, device=DEV)
    labels = torch.full((max(int(est_off[-1]), 1), 2, T), 7, dtype=torch.int8, device=DEV)
    _lib.check(lib.gp_bop_match(len(groups), thr.shape[0], T, _i32(est_off), _i32(gt_off), _i32([g["obj"] for g in groups]),
                                _f64(thr), mssd.data_ptr(), mspd.data_ptr(), valid.data_ptr(), ws.data_ptr(),
                                labels.data_ptr(), None))
    return labels.cpu().numpy()[:int(est_off[-1])]


def test_match_labels_equal_the_port_on_random_groups():
    rng = np.random.default_rng(11)
    T, n_obj = 10, 3
    thr = np.stack([np.stack([np.linspace(0.5, 5.0, T) * (o + 1), np.linspace(1.0, 10.0, T)]) for o in range(n_obj)])
    shapes = [(0, 3), (1, 0), (4, 0), (1, 1), (5, 3), (12, 7), (40, 33), (3, 64), (30, 70), (6, 1024), (100, 5)]
    shapes += [(int(rng.integers(0, 20)), int(rng.integers(0, 40))) for _ in range(20)]
    groups = []
    for i, (ne, ng) in enumerate(shapes):
        valid = rng.random(ng) > 0.3
        if i % 5 == 3:
            valid[:] = False                                    # all ignored
        # a coarse grid of errors: many exact ties between ground truths and with the thresholds
        mssd = np.round(rng.random((ne, ng)) * 12, 1)
        mspd = np.round(rng.random((ne, ng)) * 12, 0)
        mssd[rng.random((ne, ng)) < 0.05] = np.nan
        mspd[rng.random((ne, ng)) < 0.05] = np.nan
        groups.append(dict(obj=i % n_obj, mssd=mssd.astype(np.float32), mspd=mspd.astype(np.float32), valid=valid))
    got = _match(groups, thr)
    row, counts = 0, np.zeros(3, int)
    for g in groups:
        ne = g["mssd"].shape[0]
        for m, err in enumerate((g["mssd"], g["mspd"])):
            want = bop24_port.detection_labels(err.astype(np.float64), g["valid"], thr[g["obj"], m])
            np.testing.assert_array_equal(got[row:row + ne, m], want)
        row += ne
    for v in range(3):
        counts[v] = int((got == v).sum())
    assert counts.min() > 10, counts                            # every label occurs
    _report("match labels", dict(groups=len(groups), estimates=row, fp_tp_ignored=counts.tolist()))


def _ap(labels, rank_off, rank, n_valid, rec=bop_eval.RECALL_THRESHOLDS):
    lib = _lib.load()
    n_obj, T = len(n_valid), labels.shape[2]
    out = torch.empty(n_obj, 2, T, dtype=torch.float64, device=DEV)
    lab = _dev(labels, np.int8)
    rk = _dev(np.concatenate([rank, [0]]), np.int32)
    _lib.check(lib.gp_bop_average_precision(n_obj, T, labels.shape[0], lab.data_ptr(), _i32(rank_off), rk.data_ptr(),
                                            _i32(n_valid), len(rec), _f64(rec), out.data_ptr(), None))
    return out.cpu().numpy()


def test_average_precision_is_bit_identical_to_the_port():
    rng = np.random.default_rng(5)
    T = 4
    sizes = [1, 0, 7, 256, 257, 3000, 12345, 2]           # one estimate, none, partial and several scan tiles
    n_valid = [1, 3, 4, 100, 50, 1000, 4000, 1]            # 100 / 50 / 1000: recalls landing exactly on r_k
    n = sum(sizes)
    labels = rng.choice(np.array([0, 1, 2], np.int8), size=(n, 2, T), p=[0.4, 0.45, 0.15])
    labels[:1, 0, 0] = bop24_port.LABEL_TP
    labels[-2:] = bop24_port.LABEL_TP                        # the last object: 2 TPs on 1 valid gt
    rank = rng.permutation(n).astype(np.int32)
    rank_off = np.cumsum([0] + sizes)
    got = _ap(labels, rank_off, rank, n_valid)
    exact = 0
    for o in range(len(sizes)):
        ranked = labels[rank[rank_off[o]:rank_off[o + 1]]]
        for m in range(2):
            for t in range(T):
                want = bop24_port.average_precision(ranked[:, m, t], n_valid[o])
                assert np.float64(got[o, m, t]).view(np.uint64) == np.float64(want).view(np.uint64), (o, m, t)
                tp = np.cumsum(ranked[:, m, t] == bop24_port.LABEL_TP) / n_valid[o]
                exact += int(np.isin(tp, bop_eval.RECALL_THRESHOLDS).sum())
    assert got[1].tolist() == [[0.0] * T] * 2 and exact > 100
    _report("average precision", dict(objects=len(sizes), ranked=n, recalls_equal_to_an_r_k=exact))


def _tree(root):
    """Two scenes of three images: repeated instances, ~15 % ignored, perturbed estimates, duplicates, wrong-object
    estimates, score ties and 24 estimates per image (above the cap of 20 the test sets), except one image without
    estimates; no depth images (the width comes from rgb/)."""
    import os
    models = {1: tetra(60.0), 2: spheroid(40.0, 25.0, n_lat=10, n_lon=24), 3: tetra(45.0), 4: tetra(30.0)}
    flip = np.diag([-1.0, -1, 1, 1])
    info = {1: dict(diameter=84.9), 2: dict(diameter=80.0, symmetries_discrete=[flip.ravel().tolist()]),
            3: dict(diameter=63.6, symmetries_continuous=[dict(axis=[0, 0, 1], offset=[0, 0, 0])]), 4: dict(diameter=42.4)}
    rng = np.random.default_rng(3)
    K = np.array([[600.0, 0, 321.0], [0, 601.0, 239.0], [0, 0, 1]])
    scenes, results, targets = {}, [], []
    for s in (1, 2):
        scenes[s] = {}
        for im in range(3):
            objs = [1, 1, 2, 2, 3, 1] if im != 2 else [2, 3, 3]
            gts = [(o, rot(rng.normal(size=3), rng.uniform(0, 180)),
                    [(k % 3 - 1) * 120.0 + rng.normal(), (k // 3 - 0.5) * 150.0, rng.uniform(600, 900)])
                   for k, o in enumerate(objs)]
            visib = [0.05 if rng.random() < 0.15 else rng.uniform(0.1, 1.0) for _ in gts]
            scenes[s][im] = dict(gt=gts, visib=visib, K=K, depth_scale=1.0, png=np.zeros((480, 640), np.uint16))
            targets.append((s, im))
            if (s, im) == (2, 2):
                continue                                            # a target image without estimates
            for o, R, t in gts:
                for rep in range(3):
                    dR = rot(rng.normal(size=3), rng.uniform(0, 15 * rep))
                    dt = rng.normal(size=3) * [3, 3, 10] * rep
                    score = float(np.round(rng.random(), 1))           # coarse scores: ties
                    results.append(dict(scene_id=s, im_id=im, obj_id=o, score=score, R=dR @ R,
                                        t=(np.asarray(t) + dt).reshape(3, 1), time=0.1))
                results.append(dict(scene_id=s, im_id=im, obj_id=4, score=0.3, R=R, t=np.asarray(t).reshape(3, 1),
                                    time=0.1))                          # a wrong object (4 has no ground truth)
    write_tree(str(root), models, info, scenes, [(s, im, 1, 1) for s, im in targets])
    with open(os.path.join(root, "test_targets_bop24.json"), "w") as f:
        json.dump([dict(scene_id=s, im_id=im) for s, im in targets], f)
    for s in scenes:
        os.rename(os.path.join(root, "test", f"{s:06d}", "depth"), os.path.join(root, "test", f"{s:06d}", "rgb"))
    return results


def test_evaluate_detection_end_to_end_matches_the_port_pipeline(tmp_path, monkeypatch):
    results = _tree(tmp_path)
    lib = _lib.load()
    monkeypatch.setattr(bop_eval, "MAX_PAIRS_PER_CALL", 37)   # several gp_bop_mssd_mspd calls
    before = lib.gp_launch_count()
    ms = {}
    out = bop_eval.evaluate_detection(results, str(tmp_path), out_dir=str(tmp_path / "eval"), device=DEV,
                                      max_estimates_per_image=20, stage_ms=ms)
    torch.cuda.synchronize(DEV)
    launched = lib.gp_launch_count() - before
    n_pairs = len(out["errors"]["group"])
    assert launched == -(-n_pairs // 37) + 2, (launched, n_pairs)
    setup = bop_eval.prepare_detection(results, str(tmp_path), max_estimates_per_image=20)
    assert setup["objects"] == [1, 2, 3] and out["objects"] == [1, 2, 3]
    assert any(len(g["est"]) == 0 for g in setup["groups"]) and n_pairs > 100
    port = port_pipeline(setup, 640 / 640)
    err = out["errors"]
    for p in range(n_pairs):
        g = setup["groups"][int(err["group"][p])]
        key = (port["pos"][int(err["est"][p])], port["gpos"][(g["scene_id"], g["im_id"], int(err["gt"][p]))])
        want = port["errors"][key]
        assert err["mssd"][p].view(np.uint32) == np.float32(want[0]).view(np.uint32), p
        assert err["mspd"][p].view(np.uint32) == np.float32(want[1]).view(np.uint32), p
    np.testing.assert_array_equal(out["labels"], port["labels"][[port["pos"][e] for e in out["rows"]]])
    np.testing.assert_array_equal(out["ap_mssd"].view(np.uint64), port["ap_mssd"].view(np.uint64))
    np.testing.assert_array_equal(out["ap_mspd"].view(np.uint64), port["ap_mspd"].view(np.uint64))
    for k in ("map", "map_mssd", "map_mspd"):
        assert np.float64(out[k]).view(np.uint64) == np.float64(port[k]).view(np.uint64), k
    assert 0 < out["map"] < 1
    assert (out["labels"] == bop24_port.LABEL_IGNORED).any() and (out["labels"] == bop24_port.LABEL_TP).any()
    scores = json.load(open(tmp_path / "eval" / "scores_bop24.json"))
    assert scores["bop24_mAP"] == out["map"] and scores["bop24_mAP_mssd"] == out["map_mssd"]
    assert scores["bop24_average_time_per_image"] == pytest.approx(0.1)
    assert set(ms) == {"mssd_mspd", "match", "ap"}
    # one call per stage gives the same bits
    monkeypatch.setattr(bop_eval, "MAX_PAIRS_PER_CALL", 1 << 18)
    again = bop_eval.evaluate_detection(results, str(tmp_path), device=DEV, max_estimates_per_image=20)
    np.testing.assert_array_equal(again["ap_mssd"].view(np.uint64), out["ap_mssd"].view(np.uint64))
    np.testing.assert_array_equal(again["errors"]["mspd"].view(np.uint32), err["mspd"].view(np.uint32))
    _report("end to end", dict(pairs=n_pairs, map=out["map"], map_mssd=out["map_mssd"], map_mspd=out["map_mspd"]))


def test_cli_detection_task_writes_scores_bop24(tmp_path):
    """`--task detection` on a tree without depth images, from a results csv."""
    import os
    import subprocess
    import sys
    results = _tree(tmp_path)
    csv = tmp_path / "res.csv"
    with open(csv, "w") as f:
        f.write("scene_id,im_id,obj_id,score,R,t,time\n")
        for r in results:
            R = " ".join(repr(float(x)) for x in np.asarray(r["R"]).ravel())
            t = " ".join(repr(float(x)) for x in np.asarray(r["t"]).ravel())
            f.write(f"{r['scene_id']},{r['im_id']},{r['obj_id']},{r['score']},{R},{t},{r['time']}\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    run = subprocess.run([sys.executable, "-m", "gigapose_b200.bop_eval", "--task", "detection", "--results", str(csv),
                          "--dataset-dir", str(tmp_path), "--out", str(tmp_path / "o")], capture_output=True, text=True,
                         env=env, cwd=root)
    assert run.returncode == 0, run.stderr
    scores = json.load(open(tmp_path / "o" / "scores_bop24.json"))
    direct = bop_eval.evaluate_detection(str(csv), str(tmp_path), device=DEV)
    assert scores["bop24_mAP"] == direct["map"] and 0 < scores["bop24_mAP"] < 1
