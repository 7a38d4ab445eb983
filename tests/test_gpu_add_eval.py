"""Row f12 on the GPU: gp_bop_add bit for bit against oracle/add_port.py (objects of 1 to 100 000 vertices in one call,
frames with their own K, K01 != 0, repeated pairs, a call split at MAX_PAIRS_PER_CALL), exact zeros and NaNs, the launch
count of evaluate_add, and evaluate_add / `--task add` end to end on the golden tree against the reference's matches,
recalls and AUCs (tests/golden/add_reference.*)."""
import json
import math
import os

import numpy as np
import pytest
import torch

import add_fp64 as af
from gigapose_b200 import _lib, bop_eval
from oracle import add_port

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = (1, 3, 255, 256, 257, 10002, 100000)


def _t(a, dt=None):
    return torch.as_tensor(np.ascontiguousarray(a, dt), device=DEV)


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _axis_angle(axis, deg):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    t = np.deg2rad(deg)
    return np.eye(3) + np.sin(t) * k + (1 - np.cos(t)) * (k @ k)


def _pose(rng, R=None, t=None):
    P = np.eye(4)
    P[:3, :3] = _rot(rng) if R is None else R
    P[:3, 3] = rng.uniform([-150, -150, 900], [150, 150, 1800]) if t is None else t
    return P


def call_case(seed=0):
    """Objects of every size in SIZES, three frames with their own K (one with K01 != 0), pairs near and far, one pair
    repeated at three batch positions, identical poses, invalid indices and NaN poses."""
    rng = np.random.default_rng(seed)
    objs = [(rng.normal(size=(n, 3)) * rng.uniform(20, 90, 3)).astype(np.float32) for n in SIZES]
    vo = np.cumsum([0] + [len(v) for v in objs]).tolist()
    K = np.array([[[600, 0, 320], [0, 600, 240], [0, 0, 1]], [[572.4, 1.75, 325.3], [0, 573.6, 242.0], [0, 0, 1]],
                  [[1066.8, -3.0, 960.0], [0, 1067.5, 540.0], [0, 0, 1]]], np.float32)
    obj, frame, pe, pg = [], [], [], []
    for o in range(len(SIZES)):
        for k in range(3):                   # a small, a larger and an unrelated rotation
            P = _pose(rng)
            Q = _pose(rng, R=_rot(rng) if k == 2 else P[:3, :3] @ _axis_angle(rng.normal(size=3), (2.0, 10.0)[k]),
                      t=P[:3, 3] + rng.normal(size=3) * (5, 20, 60)[k])
            obj.append(o)
            frame.append(k)
            pe.append(Q)
            pg.append(P)
    same = len(obj)                          # pair 12 again at same and same + 1, pair 16 at same + 2
    for p in (12, 12, 16):
        obj.append(obj[p])
        frame.append(frame[p])
        pe.append(pe[p])
        pg.append(pg[p])
    ident = len(obj)
    for o in (2, 5):
        obj.append(o)
        frame.append(1)
        P = _pose(rng)
        pe.append(P)
        pg.append(P)
    bad = len(obj)
    P = _pose(rng)
    nanp = P.copy()
    nanp[1, 2] = np.nan
    for o, f, a, b in ((-1, 0, P, P), (len(SIZES), 0, P, P), (1, -1, P, P), (1, 3, P, P), (3, 0, nanp, P), (3, 0, P, nanp)):
        obj.append(o)
        frame.append(f)
        pe.append(a)
        pg.append(b)
    return dict(objs=objs, vertices=np.concatenate(objs), vo=vo, K=K, obj=np.array(obj, np.int32),
                frame=np.array(frame, np.int32), pe=np.array(pe, np.float32), pg=np.array(pg, np.float32),
                same=same, ident=ident, bad=bad)


def run_kernel(c, obj=None, frame=None, pe=None, pg=None):
    pick = lambda a, d: c[d] if a is None else a
    return bop_eval.add_errors(_t(pick(obj, "obj")), c["vo"], _t(c["vertices"]), _t(c["K"]), _t(pick(frame, "frame")),
                               _t(pick(pe, "pe")), _t(pick(pg, "pg"))).cpu().numpy()


_CASE = {}


def case():
    if not _CASE:
        c = call_case()
        c["kernel"] = run_kernel(c)
        c["port"] = add_port.add_errors_pairs(c["vertices"], c["vo"], c["obj"], c["K"], c["frame"], c["pe"], c["pg"],
                                              device=DEV)
        _CASE.update(c)
    return _CASE


def _same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint64),
                                                                        b[~np.isnan(b)].view(np.uint64))


def test_kernel_equals_the_port_bit_for_bit():
    c = case()
    n_chunks = [math.ceil(n / _lib.BOP_ADD_CHUNK) for n in SIZES]
    assert max(n_chunks) >= 98 and 1 in n_chunks and 10002 in SIZES        # tile and chunk borders are crossed
    for p in range(c["bad"]):
        assert _same_bits(c["kernel"][p], c["port"][p]), (p, c["obj"][p], c["kernel"][p], c["port"][p])
    assert _same_bits(c["kernel"], c["port"])


def test_repeated_pairs_identical_poses_and_invalid_pairs():
    c = case()
    k = c["kernel"]
    s = c["same"]
    assert _same_bits(k[12], k[s]) and _same_bits(k[12], k[s + 1]) and _same_bits(k[16], k[s + 2])
    assert (k[c["ident"]:c["bad"]] == 0).all()
    assert np.isnan(k[c["bad"]:]).all() and len(k) - c["bad"] == 6


def test_split_at_max_pairs_per_call_and_launch_count(monkeypatch):
    c = case()
    n = c["bad"]
    sel = np.r_[0:n:2]                       # 16 pairs
    lib = _lib.load()
    monkeypatch.setattr(bop_eval, "MAX_PAIRS_PER_CALL", 5)
    before = lib.gp_launch_count()
    split = run_kernel(c, c["obj"][sel], c["frame"][sel], c["pe"][sel], c["pg"][sel])
    torch.cuda.synchronize()
    assert lib.gp_launch_count() - before == 2 * math.ceil(len(sel) / 5)
    one = np.concatenate([run_kernel(c, c["obj"][[p]], c["frame"][[p]], c["pe"][[p]], c["pg"][[p]]) for p in sel])
    assert _same_bits(split, one) and _same_bits(split, c["kernel"][sel])
    before = lib.gp_launch_count()
    empty = bop_eval.add_errors(_t(np.zeros(0, np.int32)), c["vo"], _t(c["vertices"]), _t(c["K"]),
                                _t(np.zeros(0, np.int32)), _t(np.zeros((0, 4, 4), np.float32)),
                                _t(np.zeros((0, 4, 4), np.float32)))
    assert empty.shape == (0, 3) and lib.gp_launch_count() == before


def test_kernel_argument_checks():
    import ctypes as C
    lib = _lib.load()
    vo = (C.c_int32 * 3)(0, 4, 4)
    d = torch.empty(8, dtype=torch.float64, device=DEV)
    assert lib.gp_bop_add(1, 2, d.data_ptr(), vo, d.data_ptr(), 1, d.data_ptr(), d.data_ptr(), d.data_ptr(),
                          d.data_ptr(), d.data_ptr(), d.data_ptr(), None) != 0
    assert b"offsets" in lib.gp_last_error()
    vo = (C.c_int32 * 2)(0, 4)
    assert lib.gp_bop_add(1, 1, d.data_ptr(), vo, d.data_ptr(), 1, d.data_ptr(), d.data_ptr(), d.data_ptr(),
                          d.data_ptr(), d.data_ptr() + 4, d.data_ptr(), None) != 0
    assert b"aligned" in lib.gp_last_error()
    assert lib.gp_bop_add(0, 1, d.data_ptr(), vo, d.data_ptr(), 1, d.data_ptr(), d.data_ptr(), d.data_ptr(),
                          d.data_ptr(), d.data_ptr(), d.data_ptr(), None) != 0


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
    tree, models, faces, results, ref = af.golden(golden_dir)
    root = str(tmp_path_factory.mktemp("add_tree"))
    af.write_golden_tree(root, tree, models, faces)
    return dict(tree=tree, models=models, results=results, ref=ref, root=root, setup=bop_eval.prepare(results, root))


def test_evaluate_add_gives_the_reference_scores(fx, tmp_path, monkeypatch):
    lib = _lib.load()
    out = str(tmp_path / "out")
    monkeypatch.setattr(bop_eval, "MAX_PAIRS_PER_CALL", 4)
    torch.cuda.synchronize()
    before = lib.gp_launch_count()
    res = bop_eval.evaluate_add(fx["results"], fx["root"], out_dir=out, device=DEV)
    torch.cuda.synchronize()
    n_pairs = len(res["errors"]["group"])
    assert n_pairs == 21 and lib.gp_launch_count() - before == 2 * math.ceil(n_pairs / 4)
    ref = fx["ref"]
    assert res["n_targets"] == ref["n_targets"]
    for m in af.METRICS:
        got = sorted((int(e), int(k)) for (_, k), e in zip(res["target_gt"], res["matched_est"][m]) if e >= 0)
        assert got == sorted((a, b) for a, b, _ in ref["matches"][m]), m
        assert res["recall"][m] == ref["recall"][m], m
    worst = max(abs(a - b) for m in ("add(-s)", "add-s") for a, b in
                zip(sorted(x for x in res["matched"][m] if np.isfinite(x)), sorted(x[2] for x in ref["matches"][m])))
    for m in ("add(-s)", "add-s"):
        assert af.close_auc(res["auc"][m], ref["auc"][m], 20 * worst / 1000 + 1e-15), m
        for o, v in res["objects"].items():
            assert af.close_auc(v["auc"][m], ref["auc_objects"][m][str(o)], 20 * worst / 1000 + 1e-15), (m, o)
    assert res["matched"]["add(-s)"].tolist().count(100.0) == 1 and 100.0078125 in res["matched"]["add(-s)"].tolist()
    with open(os.path.join(out, "scores_add.json")) as f:
        js = json.load(f)
    assert js["add(-s)_0.1d"] == res["recall"]["add(-s)"] and js["n_targets"] == 9
    assert set(js) == {"add(-s)_0.1d", "add-s_0.1d", "proj_5px", "auc_add(-s)", "auc_add-s", "n_targets", "objects"}
    assert set(js["objects"]) == {"1", "2", "3"} and math.isnan(js["objects"]["3"]["auc_add-s"])


def test_task_add_writes_scores_add_json(fx, tmp_path):
    csv = tmp_path / "est.csv"
    with open(csv, "w") as f:
        f.write("scene_id,im_id,obj_id,score,R,t,time\n")
        for r in fx["results"]:
            f.write(f"{r['scene_id']},{r['im_id']},{r['obj_id']},{r['score']!r},"
                    f"{' '.join(repr(float(x)) for x in np.ravel(r['R']))},"
                    f"{' '.join(repr(float(x)) for x in np.ravel(r['t']))},{r['time']!r}\n")
    bop_eval.main(["--task", "add", "--results", str(csv), "--dataset-dir", fx["root"]])
    with open(tmp_path / "scores_add.json") as f:
        js = json.load(f)
    assert js["add-s_0.1d"] == fx["ref"]["recall"]["add-s"] and js["n_targets"] == fx["ref"]["n_targets"]
