"""Rows f7 and f8 on the GPU against the independent fp64 evaluator (tests/bop_fp64.py): gp_bop_vsd at 1080 x 1920 and
480 x 640, gp_bop_mssd_mspd on a 10 002-vertex, 630-transform object in one call and past MAX_PAIRS_PER_CALL, and
evaluate() / evaluate_detection() end to end; every mutated definition fails against the kernels.  Worst ratios to the
bars, excluded fractions and mutation margins are printed (pytest -s) for DESIGN.md."""
import json
import os

import numpy as np
import pytest
import torch

import bop_fp64 as bf
from bop_tree import write_tree
from gigapose_b200 import bop_eval, icp

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TAUS16 = tuple(i / 40 for i in range(1, 17))


def _report(name, obj):
    print(name, json.dumps(obj))


def _t(a, dt=None):
    return torch.as_tensor(np.ascontiguousarray(a, dt), device=DEV)


def gpu_render(V, F, P, K, H, W):
    """gp_render_depth of one view (what evaluate() renders)."""
    dm = icp.device_meshes([dict(vertices=np.asarray(V, np.float32), faces=np.asarray(F, np.int32))], DEV)[0]
    ws = torch.empty(8 * H * W, dtype=torch.uint8, device=DEV)
    d = torch.empty(1, H, W, device=DEV)
    b = torch.empty(1, 4, dtype=torch.int64, device=DEV)
    bop_eval.render_depth(dm, _t(np.asarray(P, np.float32).reshape(1, 4, 4)), _t(K, np.float32), H, W, 10.0, ws, d, b)
    return d[0].cpu().numpy()


def _boxes(renders):
    out = []
    for r in renders:
        ys, xs = np.nonzero(r > 0)
        out.append([xs.min(), ys.min(), xs.max() + 1, ys.max() + 1] if len(xs) else [0, 0, r.shape[1], r.shape[0]])
    return np.array(out, np.int64)


_FRAMES = {}


def _frames(H, W):
    """The scene, the kernel's counts and errors for 10, 1 and 16 tolerances, with invalid pairs appended."""
    if (H, W) not in _FRAMES:
        fr = bf.vsd_frames(H, W, gpu_render, seed=H, n_renders=20)
        n_r, n_f = len(fr["renders"]), len(fr["depth"])
        bad = np.array([(-1, 0, 1), (n_f, 0, 1), (0, -1, 1), (0, n_r, 1), (0, 0, -1), (0, 0, n_r)], np.int64)
        pairs = np.concatenate([fr["pairs"], bad])
        diam = np.concatenate([fr["diameter"], np.full(len(bad), 100.0)])
        dev = dict(depth=_t(fr["depth"]), K=_t(fr["K"]), r=_t(fr["renders"]), b=_t(_boxes(fr["renders"])))
        out = {}
        for taus in (bf.TAUS, (0.3,), TAUS16):
            c, e = bop_eval.vsd(dev["depth"], dev["K"], _t(pairs[:, 0], np.int32), dev["r"], dev["b"], _t(pairs[:, 1], np.int32),
                                dev["r"], dev["b"], _t(pairs[:, 2], np.int32), _t(diam, np.float32), bf.DELTA, taus)
            out[taus] = (c.cpu().numpy(), e.cpu().numpy())
        del dev
        torch.cuda.empty_cache()
        fr["kernel"], fr["n_bad"] = out, len(bad)
        _FRAMES[(H, W)] = fr
    return _FRAMES[(H, W)]


@pytest.mark.parametrize("H,W", [(1080, 1920), (480, 640)])
def test_vsd_kernel_against_the_fp64_definition(H, W):
    fr = _frames(H, W)
    n = len(fr["pairs"])
    assert n >= 1000 and len(fr["depth"]) >= 3 and len({fr["K"][f].tobytes() for f in range(len(fr["K"]))}) == len(fr["K"])
    boxes = _boxes(fr["renders"])
    assert (boxes[:, 0] == 0).any() and (boxes[:, 1] == 0).any() and (boxes[:, 2] == W).any() and (boxes[:, 3] == H).any()
    report = {}
    for taus, (counts, errors) in fr["kernel"].items():
        assert (counts[n:] == -1).all() and np.isnan(errors[n:]).all()            # invalid frame / estimate / gt
        worst, amb, union, empty = 0.0, {}, {}, 0
        for p, (f, e, g) in enumerate(fr["pairs"]):
            ref = bf.vsd(fr["depth"][f], fr["K"][f], fr["renders"][e], fr["renders"][g], fr["diameter"][p], bf.DELTA, taus)
            excess, ratio = bf.compare_vsd(counts[p], errors[p], ref)
            assert excess <= 0 and ratio <= 1, (taus, p, counts[p], ref["counts"], ref["n_amb"], errors[p], ref["errors"])
            worst = max(worst, ratio)
            amb[int(f)] = amb.get(int(f), 0) + ref["n_amb"]
            union[int(f)] = union.get(int(f), 0) + int(ref["counts"][1])
            empty += int(ref["counts"][1] == 0)
        frac = {f: amb[f] / max(union[f], 1) for f in amb}
        assert max(frac.values()) < 1e-3 and empty >= 2
        report[len(taus)] = dict(worst_ratio=worst, excluded_fraction=frac, union_pixels=sum(union.values()), empty=empty)
    _report(f"vsd {H}x{W}", dict(pairs=n, per_n_tau=report))


@pytest.mark.parametrize("mutation", bf.VSD_MUTATIONS)
def test_vsd_mutation_fails_against_the_kernel(mutation):
    fr = _frames(480, 640)
    counts, errors = fr["kernel"][bf.TAUS]
    fails, worst = 0, 0.0
    for p, (f, e, g) in enumerate(fr["pairs"]):
        ref = bf.vsd(fr["depth"][f], fr["K"][f], fr["renders"][e], fr["renders"][g], fr["diameter"][p], mutation=mutation)
        excess, ratio = bf.compare_vsd(counts[p], errors[p], ref)
        fails += excess > 0 or ratio > 1
        worst = max(worst, ratio)
    _report("vsd gpu mutation", dict(mutation=mutation, failing_pairs=fails, worst_ratio=worst))
    assert fails >= 1 and worst >= 10


_POSES = {}


def _poses(tmp_dir):
    """Every pose case in ONE gp_bop_mssd_mspd call with the production symmetry tables (bop_eval.symmetry_transforms
    of the models_info.json the reader loads), plus pairs with invalid object and frame indices."""
    if not _POSES:
        objects = bf.pose_objects()
        with open(os.path.join(tmp_dir, "models_info.json"), "w") as f:
            json.dump({str(o + 1): info for o, (_, info) in enumerate(objects)}, f)
        loaded = bop_eval.load_models_info(tmp_dir)
        syms = [bop_eval.symmetry_transforms(loaded[o + 1]) for o in range(len(objects))]
        assert [len(s) for s in syms] == [630, 1, 9] and len(objects[0][0]) == 10002
        cases = bf.pose_cases(objects)
        bad = [(-1, 0), (3, 0), (0, -1), (1, 2)]
        obj = [c[0] for c in cases] + [b[0] for b in bad]
        frame = [c[1] for c in cases] + [b[1] for b in bad]
        Pe = np.stack([c[2] for c in cases] + [np.eye(4)] * len(bad))
        Pg = np.stack([c[3] for c in cases] + [np.eye(4)] * len(bad))
        vo = np.cumsum([0] + [len(V) for V, _ in objects]).tolist()
        so = np.cumsum([0] + [len(s) for s in syms]).tolist()
        mssd, mspd = bop_eval.mssd_mspd(_t(obj, np.int32), vo, _t(np.concatenate([V for V, _ in objects]), np.float32), so,
                                        _t(np.concatenate(syms), np.float32), _t(np.stack(bf.POSE_KS)),
                                        _t(frame, np.int32), _t(Pe, np.float32), _t(Pg, np.float32))
        _POSES.update(objects=objects, cases=cases, n_bad=len(bad), mssd=mssd.cpu().numpy(), mspd=mspd.cpu().numpy())
    return _POSES


def test_mssd_mspd_kernel_against_the_fp64_definition(tmp_path):
    P = _poses(str(tmp_path))
    n = len(P["cases"])
    assert (P["mssd"][n:].view(np.uint32) == 0xFFFFFFFF).all() and (P["mspd"][n:].view(np.uint32) == 0xFFFFFFFF).all()
    worst = [0.0, 0.0]
    for p, (o, f, Pe, Pg) in enumerate(P["cases"]):
        V, info = P["objects"][o]
        ref = bf.mssd_mspd(V, bf.symmetries(info), Pe, Pg, bf.POSE_KS[f])
        bars = bf.pose_bars(V, Pe, Pg, bf.POSE_KS[f])
        for m, k in enumerate((P["mssd"][p], P["mspd"][p])):
            worst[m] = max(worst[m], abs(float(k) - ref[m]) / bars[m])
    _report("mssd / mspd gpu, ratio to bar", dict(pairs=n, mssd=worst[0], mspd=worst[1], bar_u=[bf.POSE_BAR_MSSD, bf.POSE_BAR_MSPD]))
    assert max(worst) <= 1


@pytest.mark.parametrize("mutation", bf.POSE_MUTATIONS)
def test_pose_mutation_fails_against_the_kernel(tmp_path, mutation):
    P = _poses(str(tmp_path))
    worst = 0.0
    for p, (o, f, Pe, Pg) in enumerate(P["cases"]):
        V, info = P["objects"][o]
        ref = bf.mssd_mspd(V, bf.symmetries(info, mutation), Pe, Pg, bf.POSE_KS[f], mutation)
        bars = bf.pose_bars(V, Pe, Pg, bf.POSE_KS[f])
        worst = max(worst, abs(float(P["mssd"][p]) - ref[0]) / bars[0], abs(float(P["mspd"][p]) - ref[1]) / bars[1])
    _report("pose gpu mutation", dict(mutation=mutation, worst_ratio=worst))
    assert worst >= 10


def test_mssd_mspd_split_past_max_pairs_per_call_equals_the_per_pair_results():
    V, info = bf.pose_objects()[1]
    rng = np.random.default_rng(9)
    distinct = [(f, bf.pose(bf.rot(rng.normal(size=3), rng.uniform(0, 20)), rng.normal(size=3) * 10 + [0, 0, 700]),
                 bf.pose(np.eye(3), [0, 0, 700.0])) for f in (0, 1, 1, 0, 1)]
    n = bop_eval.MAX_PAIRS_PER_CALL + 4099
    pick = np.arange(n) % len(distinct)
    vo, so = [0, len(V)], [0, 1]
    args = lambda idx: (_t(np.zeros(len(idx)), np.int32), vo, _t(V, np.float32), so, _t(np.eye(4)[None], np.float32),
                        _t(np.stack(bf.POSE_KS)), _t([distinct[i][0] for i in idx], np.int32),
                        _t(np.stack([distinct[i][1] for i in idx]), np.float32),
                        _t(np.stack([distinct[i][2] for i in idx]), np.float32))
    big = [x.cpu().numpy() for x in bop_eval.mssd_mspd(*args(pick))]
    one = [x.cpu().numpy() for x in bop_eval.mssd_mspd(*args(np.arange(len(distinct))))]
    for m in range(2):
        np.testing.assert_array_equal(big[m].view(np.uint32), one[m][pick].view(np.uint32))
    for i, (f, Pe, Pg) in enumerate(distinct):
        ref = bf.mssd_mspd(V, np.eye(4)[None], Pe, Pg, bf.POSE_KS[f])
        bars = bf.pose_bars(V, Pe, Pg, bf.POSE_KS[f])
        assert abs(one[0][i] - ref[0]) <= bars[0] and abs(one[1][i] - ref[1]) <= bars[1]
    _report("mssd / mspd split", dict(pairs=n, calls=-(-n // bop_eval.MAX_PAIRS_PER_CALL)))


@pytest.fixture(scope="module")
def ar_case(tmp_path_factory):
    root = tmp_path_factory.mktemp("ar_gpu")
    tree, results = bf.ar_tree(gpu_render)
    write_tree(str(root), tree["models"], tree["info"], tree["scenes"], tree["targets"])
    render = lambda o, P, K, h, w: gpu_render(*tree["models"][o], P, K, h, w)
    out = bop_eval.evaluate(results, str(root), device=DEV)
    return tree, results, render, out


def test_evaluate_equals_the_fp64_reference(ar_case):
    tree, results, render, out = ar_case
    ref = bf.evaluate_bop19(tree, results, render)
    assert ref["margin"] > 1, ref["margin"]
    assert out["n_targets"] == ref["n_targets"]
    for k in ("recall_vsd", "recall_mssd", "recall_mspd"):
        np.testing.assert_array_equal(out[k], ref[k])
    for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd"):
        assert out[k] == ref[k], k
    assert 0 < out["ar"] < 1
    _report("evaluate vs fp64", dict(ar=out["ar"], n_targets=out["n_targets"], pairs=len(ref["pairs"]),
                                     smallest_margin_in_bars=ref["margin"]))


@pytest.mark.parametrize("mutation", bf.AR_MUTATIONS)
def test_average_recall_mutation_fails_against_evaluate(ar_case, mutation):
    tree, results, render, out = ar_case
    ref = bf.evaluate_bop19(tree, results, render, mutation=mutation)
    diff = max(float(np.abs(out[k] - ref[k]).max()) for k in ("recall_vsd", "recall_mssd", "recall_mspd"))
    _report("ar gpu mutation", dict(mutation=mutation, recall_difference=diff, ar_difference=ref["ar"] - out["ar"]))
    assert diff >= 1 / 7 - 1e-12


@pytest.fixture(scope="module")
def ap_case(tmp_path_factory):
    root = tmp_path_factory.mktemp("ap_gpu")
    tree, results = bf.ap_tree()
    write_tree(str(root), tree["models"], tree["info"], tree["scenes"], tree["targets"])
    with open(os.path.join(root, "test_targets_bop24.json"), "w") as f:
        json.dump([dict(scene_id=s, im_id=im) for s, im in tree["images"]], f)
    return tree, results, bop_eval.evaluate_detection(results, str(root), device=DEV)


def test_evaluate_detection_equals_the_fp64_reference(ap_case):
    tree, results, out = ap_case
    ref = bf.evaluate_bop24(tree, results)
    assert ref["margin"] > 1 and out["objects"] == ref["objects"] == [1, 3]
    assert sorted(out["rows"].tolist()) == sorted(ref["labels"])
    np.testing.assert_array_equal(out["labels"], np.stack([ref["labels"][e] for e in out["rows"].tolist()]))
    bound = 101 * 2.0 ** -53
    np.testing.assert_allclose(out["ap_mssd"], ref["ap_mssd"], rtol=0, atol=bound)
    np.testing.assert_allclose(out["ap_mspd"], ref["ap_mspd"], rtol=0, atol=bound)
    assert abs(out["map"] - ref["map"]) <= bound and 0 < out["map"] < 1
    _report("evaluate_detection vs fp64", dict(map=out["map"], estimates=len(out["rows"]),
                                               ap_difference=float(np.abs(out["ap_mssd"] - ref["ap_mssd"]).max()),
                                               smallest_margin_in_bars=ref["margin"]))


@pytest.mark.parametrize("mutation", bf.AP_MUTATIONS)
def test_detection_mutation_fails_against_evaluate_detection(ap_case, mutation):
    tree, results, out = ap_case
    ref = bf.evaluate_bop24(tree, results, mutation=mutation)
    diff = abs(ref["map"] - out["map"])
    _report("ap gpu mutation", dict(mutation=mutation, map_difference=diff))
    assert diff >= 1e-3
