"""Rows f7 and f8 without a GPU: the independent fp64 evaluator (tests/bop_fp64.py) against hand-computed cases, against
the float32 ports (oracle/bop_port.py, oracle/bop24_port.py, which the kernels equal bit for bit), and every mutated
definition failing against those ports.  Measured ratios, excluded fractions and margins are printed (pytest -s)."""
import json
import math

import numpy as np
import pytest

import bop_fp64 as bf
from bop_tree import write_tree
from gigapose_b200 import bop_eval
from oracle import bop_port
from test_bop24_eval_cpu import port_pipeline

H, W = 240, 320


def _report(name, obj):
    print(name, json.dumps(obj))


def _render(V, F, P, K, h, w):
    return bop_port.render_depth(V, F, np.asarray(P, np.float32), np.asarray(K, np.float32), h, w, 10.0)["depth"]


def _box(d):
    ys, xs = np.nonzero(d > 0)
    return np.array([xs.min(), ys.min(), xs.max() + 1, ys.max() + 1] if len(xs) else [0, 0, d.shape[1], d.shape[0]])


@pytest.fixture(scope="module")
def frames():
    fr = bf.vsd_frames(H, W, _render, n_renders=12)
    boxes = [_box(r) for r in fr["renders"]]
    fr["port"] = [bop_port.vsd_fp32(fr["depth"][f], fr["K"][f], fr["renders"][e], boxes[e], fr["renders"][g], boxes[g],
                                    np.float32(fr["diameter"][p]), bf.DELTA, bf.TAUS)
                  for p, (f, e, g) in enumerate(fr["pairs"])]
    return fr


def test_hand_computed_vsd_and_distance():
    K = np.array([[100.0, 0, 1], [0, 100.0, 1], [0, 0, 1]], np.float32)
    d, bar = bf.distances(np.array([500.0, 500.0], np.float32), np.array([1.0, 4.0]), np.array([1.0, 5.0]), K)
    assert d[0] == 500.0 and bar[0] == 0.0                                # the principal point: exact
    assert d[1] == pytest.approx(500.0 * math.sqrt(1 + 0.03 ** 2 + 0.04 ** 2), rel=1e-15) and bar[1] > 0
    test = np.zeros((3, 3), np.float32)
    gt = np.zeros((3, 3), np.float32)
    est = np.zeros((3, 3), np.float32)
    gt[1, :] = 500.0
    est[1, 1:] = 518.0                                                    # 18 mm behind the ground truth
    test[1, 1] = 485.0                                                    # the gt exactly delta behind: visible
    test[1, 2] = 600.0
    v = bf.vsd(test, K, est, gt, 100.0)
    # gt visible at (1,0) (missing depth), (1,1) (= delta) and (1,2); est at (1,2) and, through the gt, at (1,1);
    # cost 0.18 (x sqrt(1.0001) at (1,2))
    assert v["counts"].tolist() == [2, 3, 2, 2, 2, 0, 0, 0, 0, 0, 0, 0] and v["n_amb"] == 0
    np.testing.assert_allclose(v["errors"], [1.0] * 3 + [1 / 3] * 7, rtol=0, atol=1e-16)
    assert bf.vsd(test, K, est, gt, 100.0, mutation="strict_delta")["counts"][:2].tolist() == [1, 2]
    empty = bf.vsd(test, K, np.zeros_like(est), np.zeros_like(gt), 100.0)
    assert empty["counts"][1] == 0 and empty["errors"].tolist() == [1.0] * 10


def test_hand_computed_matching_symmetries_and_ap():
    e = np.array([[17.0, 13.0], [4.0, 26.0]])
    assert [g for g, _ in bf.greedy(e, [True, True], 20.0)] == [1, 0]
    assert [g for g, _ in bf.greedy(e, [True, True], 20.0, "first_come")] == [0, -1]
    assert [g for g, _ in bf.greedy(e, [True, True], 17.0)] == [1, 0]
    assert [g for g, _ in bf.greedy(e, [True, True], 13.0, "theta_le")] == [1, 0]
    assert bf.greedy(np.array([[1.0, 2.0]]), [False, True], 3.0, ignored=True) == [(1, True)]
    assert bf.average_precision([bf.TP, bf.FP, bf.TP], 2) == pytest.approx(253 / 303, abs=1e-15)
    assert bf.average_precision([bf.IGNORED, bf.TP, bf.FP, bf.TP], 2) == bf.average_precision([bf.TP, bf.FP, bf.TP], 2)
    assert bf.average_precision([bf.FP, bf.TP], 1) == 0.5
    assert bf.average_precision([bf.FP, bf.TP], 1, "no_interpolation") == pytest.approx(50 / 101, abs=1e-15)
    o = np.array([20.0, -12.0, 0.0])
    S = bf.symmetries(dict(symmetries_continuous=[dict(axis=[0, 0, 2.0], offset=o.tolist())]))
    assert len(S) == 315
    x = np.array([35.0, 4.0, 7.0])
    for k in (1, 100):
        y = S[k][:3, :3] @ x + S[k][:3, 3]                             # a turn about the line through o
        a = 2 * math.pi * k / 315
        want = np.array([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]]) @ (x - o) + o
        np.testing.assert_allclose(y, want, rtol=0, atol=1e-12)
    flip = np.diag([1.0, -1, -1, 1])
    S = bf.symmetries(dict(symmetries_discrete=[flip.ravel().tolist()],
                           symmetries_continuous=[dict(axis=[0, 0, 1], offset=[0, 0, 0])]))
    assert len(S) == 630 and np.allclose(S[315 + 5], S[5] @ flip) and not np.allclose(S[315 + 5], flip @ S[5])


def test_distance_float32_error_is_within_its_count(frames):
    worst = 0.0
    for f in range(len(frames["depth"])):
        z = frames["depth"][f]
        d32 = bop_port.dist_fp32(z, frames["K"][f], 0, 0).astype(np.float64)
        vs, us = np.mgrid[:H, :W]
        d64, bar = bf.distances(z.reshape(-1), us.reshape(-1).astype(float), vs.reshape(-1).astype(float), frames["K"][f])
        err = np.abs(d32.reshape(-1) - d64)
        worst = max(worst, float((err / np.maximum(bf.ulp32(d64), 1e-300)).max()))
        assert np.all(err <= bar)
    _report("distance float32 error, ulps", dict(worst=worst, bar=bf.DIST_ULPS))
    assert worst * 3 <= bf.DIST_ULPS


def test_vsd_reference_against_the_fp32_port(frames):
    worst, excluded = 0.0, {}
    for p, (f, e, g) in enumerate(frames["pairs"]):
        ref = bf.vsd(frames["depth"][f], frames["K"][f], frames["renders"][e], frames["renders"][g], frames["diameter"][p])
        excess, ratio = bf.compare_vsd(*frames["port"][p], ref)
        assert excess <= 0 and ratio <= 1, (p, excess, ratio)
        worst = max(worst, ratio)
        a, u = excluded.get(int(f), (0, 0))
        excluded[int(f)] = (a + ref["n_amb"], u + int(ref["counts"][1]))
    frac = {f: a / max(u, 1) for f, (a, u) in excluded.items()}
    _report("vsd cpu", dict(pairs=len(frames["pairs"]), worst_ratio=worst, excluded_fraction=frac))
    assert max(frac.values()) < 1e-3


@pytest.mark.parametrize("mutation", bf.VSD_MUTATIONS)
def test_vsd_mutation_fails_against_the_port(frames, mutation):
    fails, worst = 0, 0.0
    for p, (f, e, g) in enumerate(frames["pairs"]):
        ref = bf.vsd(frames["depth"][f], frames["K"][f], frames["renders"][e], frames["renders"][g], frames["diameter"][p],
                     mutation=mutation)
        excess, ratio = bf.compare_vsd(*frames["port"][p], ref)
        fails += excess > 0 or ratio > 1
        worst = max(worst, ratio)
    _report("vsd cpu mutation", dict(mutation=mutation, failing_pairs=fails, worst_ratio=worst))
    assert fails >= 1 and worst >= 10


def _bop_eval_info(info):
    return dict(symmetries_discrete=[np.reshape(s, (4, 4)) for s in info.get("symmetries_discrete", [])],
                symmetries_continuous=[(np.asarray(c["axis"], float), np.asarray(c["offset"], float))
                                       for c in info.get("symmetries_continuous", [])])


@pytest.fixture(scope="module")
def poses():
    objects = bf.pose_objects()
    cases = [c for c in bf.pose_cases(objects) if c[0] != 0 or c[1] == 0]      # the 630-transform object on one K
    port = []
    for o, f, Pe, Pg in cases:
        V, info = objects[o]
        S = bop_eval.symmetry_transforms(_bop_eval_info(info)).astype(np.float32)
        port.append(bop_port.mssd_mspd_fp32(V, S, Pe.astype(np.float32), Pg.astype(np.float32), bf.POSE_KS[f]))
    return objects, cases, port


def test_mssd_mspd_reference_against_the_fp32_port(poses):
    objects, cases, port = poses
    worst = [0.0, 0.0]
    for (o, f, Pe, Pg), k in zip(cases, port):
        V, info = objects[o]
        ref = bf.mssd_mspd(V, bf.symmetries(info), Pe, Pg, bf.POSE_KS[f])
        bars = bf.pose_bars(V, Pe, Pg, bf.POSE_KS[f])
        for m in range(2):
            worst[m] = max(worst[m], abs(float(k[m]) - ref[m]) / bars[m])
    _report("mssd / mspd cpu, ratio to bar", dict(mssd=worst[0], mspd=worst[1]))
    assert max(worst) <= 1


@pytest.mark.parametrize("mutation", bf.POSE_MUTATIONS)
def test_pose_mutation_fails_against_the_port(poses, mutation):
    objects, cases, port = poses
    worst = 0.0
    for (o, f, Pe, Pg), k in zip(cases, port):
        V, info = objects[o]
        ref = bf.mssd_mspd(V, bf.symmetries(info, mutation), Pe, Pg, bf.POSE_KS[f], mutation)
        bars = bf.pose_bars(V, Pe, Pg, bf.POSE_KS[f])
        worst = max(worst, max(abs(float(k[m]) - ref[m]) / bars[m] for m in range(2)))
    _report("pose cpu mutation", dict(mutation=mutation, worst_ratio=worst))
    assert worst >= 10


def _ar_port(root, tree, results):
    """bop_eval.prepare on the written tree, the fp32 ports' errors and bop_port.average_recalls."""
    setup = bop_eval.prepare(results, str(root))
    pairs, targets = [], []
    for gi, g in enumerate(setup["groups"]):
        s, im, o = g["scene_id"], g["im_id"], g["obj_id"]
        sc = setup["scenes"][s]
        K = sc["K"][im].astype(np.float32)
        depth = bop_eval.load_depth(str(root), "test", s, im, sc["depth_scale"][im])
        V, F = tree["models"][o]
        S = bop_eval.symmetry_transforms(setup["info"][o]).astype(np.float32)
        targets.append(dict(valid=dict(zip(g["gt"], g["valid"].tolist())), diameter=setup["info"][o]["diameter"]))
        for rank, e in enumerate(g["est"]):
            Pe = bop_eval._pose(results[e]["R"], results[e]["t"]).astype(np.float32)
            re = bop_port.render_depth(V, F, Pe, K, *depth.shape, 10.0)
            for k in g["gt"]:
                Pg = bop_eval._pose(sc["gt"][im][k]["R"], sc["gt"][im][k]["t"]).astype(np.float32)
                rg = bop_port.render_depth(V, F, Pg, K, *depth.shape, 10.0)
                _, v = bop_port.vsd_fp32(depth, K, re["depth"], re["box"], rg["depth"], rg["box"],
                                         np.float32(setup["info"][o]["diameter"]), 15.0, bop_eval.TAUS)
                m = bop_port.mssd_mspd_fp32(V, S, Pe, Pg, K)
                pairs.append(dict(target=gi, rank=rank, gt=k, vsd=v, mssd=m[0], mspd=m[1]))
    return bop_port.average_recalls(pairs, targets, bop_eval.TAUS, bop_eval.THETA_VSD, bop_eval.THETA_MSSD,
                                    bop_eval.THETA_MSPD, W_AR / 640)


W_AR = 400


@pytest.fixture(scope="module")
def ar_case(tmp_path_factory):
    root = tmp_path_factory.mktemp("ar")
    tree, results = bf.ar_tree(_render)
    write_tree(str(root), tree["models"], tree["info"], tree["scenes"], tree["targets"])
    render = lambda o, P, K, h, w: _render(*tree["models"][o], P, K, h, w)
    return tree, results, render, _ar_port(root, tree, results)


def test_average_recall_reference_equals_the_port_pipeline(ar_case):
    tree, results, render, port = ar_case
    ref = bf.evaluate_bop19(tree, results, render)
    assert ref["margin"] > 1, ref["margin"]
    for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd"):
        assert ref[k] == pytest.approx(port[k], abs=1e-15), k
    for k in ("recall_vsd", "recall_mssd", "recall_mspd"):
        np.testing.assert_allclose(ref[k], port[k], rtol=0, atol=1e-15)
    assert 0 < ref["ar"] < 1 and any(p["vsd"][0] == 0.25 and p["vsd_bar"][0] == 0 for p in ref["pairs"])
    _report("ar cpu", dict(ar=ref["ar"], n_targets=ref["n_targets"], pairs=len(ref["pairs"]), margin=ref["margin"]))


@pytest.mark.parametrize("mutation", bf.AR_MUTATIONS)
def test_average_recall_mutation_fails_against_the_port(ar_case, mutation):
    tree, results, render, port = ar_case
    ref = bf.evaluate_bop19(tree, results, render, mutation=mutation)
    diff = max(float(np.abs(ref[k] - port[k]).max()) for k in ("recall_vsd", "recall_mssd", "recall_mspd"))
    _report("ar cpu mutation", dict(mutation=mutation, recall_difference=diff, ar_difference=ref["ar"] - port["ar"]))
    assert diff >= 1 / 7 - 1e-12


@pytest.fixture(scope="module")
def ap_case(tmp_path_factory):
    import os
    root = tmp_path_factory.mktemp("ap")
    tree, results = bf.ap_tree()
    write_tree(str(root), tree["models"], tree["info"], tree["scenes"], tree["targets"])
    with open(os.path.join(root, "test_targets_bop24.json"), "w") as f:
        json.dump([dict(scene_id=s, im_id=im) for s, im in tree["images"]], f)
    setup = bop_eval.prepare_detection(results, str(root))
    return tree, results, setup, port_pipeline(setup, W_AR / 640)


def test_detection_reference_equals_the_port_pipeline(ap_case):
    tree, results, setup, port = ap_case
    ref = bf.evaluate_bop24(tree, results)
    assert ref["margin"] > 1 and ref["objects"] == port["objects"] == [1, 3]
    assert sorted(ref["labels"]) == port["kept"]
    for e, lab in ref["labels"].items():
        np.testing.assert_array_equal(lab, port["labels"][port["pos"][e]])
    bound = 101 * 2.0 ** -53
    np.testing.assert_allclose(ref["ap_mssd"], port["ap_mssd"], rtol=0, atol=bound)
    np.testing.assert_allclose(ref["ap_mspd"], port["ap_mspd"], rtol=0, atol=bound)
    assert abs(ref["map"] - port["map"]) <= bound and 0 < ref["map"] < 1
    _report("ap cpu", dict(map=ref["map"], estimates=len(ref["labels"]), margin=ref["margin"]))


@pytest.mark.parametrize("mutation", bf.AP_MUTATIONS)
def test_detection_mutation_fails_against_the_port(ap_case, mutation):
    tree, results, setup, port = ap_case
    ref = bf.evaluate_bop24(tree, results, mutation=mutation)
    diff = abs(ref["map"] - port["map"])
    _report("ap cpu mutation", dict(mutation=mutation, map_difference=diff))
    assert diff >= 1e-3
