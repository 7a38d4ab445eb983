"""Row f8 without a GPU: the numpy port of the BOP 2024 detection matching and AP against hand-computed cases, the
detection readers (both target formats, the per-image cap), prepare_detection + the port on a small synthetic tree
against a hand-computed mAP, and the argument checks of gp_bop_match and gp_bop_average_precision."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from bop_tree import rot, tetra, write_tree
from gigapose_b200 import _lib, bop_eval, build
from oracle import bop24_port, bop_port

FP, TP, IG = bop24_port.LABEL_FP, bop24_port.LABEL_TP, bop24_port.LABEL_IGNORED
K = np.array([[500.0, 0, 80.0], [0, 500.0, 60.0], [0, 0, 1]])


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_port_average_precision_hand_computed():
    ap = bop24_port.average_precision
    assert ap([TP, FP, TP], 2) == pytest.approx(253 / 303, abs=1e-14)
    assert ap([IG, TP, FP, TP], 2) == ap([TP, FP, TP], 2)
    assert ap([TP, TP, FP, FP, TP], 3) == pytest.approx(87.4 / 101, abs=1e-14)
    assert ap([FP, TP], 1) == 0.5
    assert ap([], 4) == 0.0
    assert ap([FP, FP], 2) == 0.0


def test_port_matching_rules():
    lab = lambda err, valid, th: bop24_port.detection_labels(np.asarray(err, float), np.asarray(valid, bool), th)[:, 0].tolist()
    assert lab([[2.0]], [True], [2.0]) == [FP]                                # equal to the threshold: no match
    assert lab([[2.0]], [True], [np.nextafter(2.0, 3)]) == [TP]
    assert lab([[1.0], [0.5]], [True], [3.0]) == [TP, FP]                     # a second estimate on the same gt
    assert lab([[1.0, 9.0]], [False, True], [3.0]) == [IG]                    # only an ignored candidate
    assert lab([[1.0, 2.0]], [False, True], [3.0]) == [TP]                    # valid preferred over a closer ignored
    assert lab([[1.0, 2.0], [0.5, 0.5]], [False, True], [3.0]) == [TP, IG]
    assert lab([[np.nan, 1.0], [np.nan, 5.0]], [True, True], [3.0]) == [TP, FP]   # NaN never matches
    assert lab([[1.0, 1.0], [1.0, 1.0]], [True, True], [3.0]) == [TP, TP]
    both = bop24_port.detection_labels(np.array([[1.0, 1.0]]), np.array([True, True]), [0.5, 3.0])
    assert both.tolist() == [[FP, TP]]
    assert bop24_port.detection_labels(np.zeros((2, 0)), np.zeros(0, bool), [1.0]).tolist() == [[FP], [FP]]


def test_port_excludes_objects_without_a_valid_ground_truth():
    ests = [dict(image=0, obj=1, score=0.9), dict(image=0, obj=2, score=0.8)]
    gts = [dict(image=0, obj=1, valid=True), dict(image=0, obj=2, valid=False)]
    errors = {(0, 0): (0.0, 0.0), (1, 1): (0.0, 0.0)}
    out = bop24_port.detection_scores(ests, gts, errors, (0.1,), (5.0,), {1: 10.0, 2: 10.0}, 1.0)
    assert out["objects"] == [1] and out["map"] == pytest.approx(1.0, abs=1e-14)
    assert out["labels"][0].tolist() == [[TP], [TP]] and out["labels"][1].tolist() == [[-1], [-1]]


def _images(scene):
    """Two images: object 1 twice (visible), object 2 once visible and once barely, object 3 only barely visible,
    object 4 visible and never estimated."""
    V = [rot([0, 1, 0], 10), rot([1, 0, 0], 30), rot([1, 1, 0], 20), rot([0, 0, 1], 40)]
    im0 = dict(gt=[(1, V[0], [-60.0, 0, 600]), (2, V[1], [40.0, 30, 700]), (2, V[2], [0.0, -40, 800]),
                   (3, V[3], [50.0, 50, 650])], visib=[0.8, 0.6, 0.05, 0.09])
    im1 = dict(gt=[(1, V[1], [30.0, 0, 640]), (4, V[2], [-20.0, 20, 700])], visib=[0.5, 0.9])
    out = {}
    for im, v in ((0, im0), (1, im1)):
        out[im] = dict(v, K=K + scene, depth_scale=1.0, png=np.zeros((12, 16), np.uint16))
    return out


def write_detection_tree(root, targets_bop24=True):
    V, F = tetra(60.0)
    info = {1: dict(diameter=85.0), 2: dict(diameter=85.0, symmetries_discrete=[np.diag([-1.0, -1, 1, 1]).ravel().tolist()]),
            3: dict(diameter=85.0), 4: dict(diameter=85.0)}
    scenes = {2: _images(2)}
    write_tree(str(root), {o: (V, F) for o in info}, info, scenes, [(2, 0, 1, 1), (2, 1, 1, 1)])
    if targets_bop24:
        with open(os.path.join(root, "test_targets_bop24.json"), "w") as f:
            json.dump([dict(scene_id=2, im_id=0), dict(scene_id=2, im_id=1)], f)
    # a dataset without depth: the width comes from the rgb image
    os.rename(os.path.join(root, "test", "000002", "depth"), os.path.join(root, "test", "000002", "rgb"))
    return scenes, info


def _res(s, im, o, score, R, t, time=0.2):
    return dict(scene_id=s, im_id=im, obj_id=o, score=score, R=np.asarray(R), t=np.asarray(t, float).reshape(3, 1),
                time=time)


def detection_results(scenes):
    g = lambda im, k: scenes[2][im]["gt"][k]
    far = lambda im, k: (g(im, k)[1], np.asarray(g(im, k)[2]) + [500.0, 0, 0])
    return [_res(2, 0, 1, 0.9, g(0, 0)[1], g(0, 0)[2]),            # object 1: TP, FP, TP over the two images
            _res(2, 1, 1, 0.8, *far(1, 0)),
            _res(2, 1, 1, 0.7, g(1, 0)[1], g(1, 0)[2]),
            _res(2, 0, 2, 0.95, g(0, 2)[1], g(0, 2)[2]),           # object 2: on the ignored gt, then the valid one
            _res(2, 0, 2, 0.5, g(0, 1)[1], g(0, 1)[2]),
            _res(2, 0, 3, 0.99, g(0, 3)[1], g(0, 3)[2]),           # object 3 has no valid gt: not evaluated
            _res(2, 7, 1, 1.0, g(0, 0)[1], g(0, 0)[2])]            # not a target image


def port_pipeline(setup, r, theta_mssd=bop_eval.THETA_MSSD, theta_mspd=bop_eval.THETA_MSPD):
    """The errors (fp32 port of gp_bop_mssd_mspd) and the score (port) of what prepare_detection kept."""
    res, scenes, info = setup["results"], setup["scenes"], setup["info"]
    kept = sorted({e for g in setup["groups"] for e in g["est"]})
    pos = {e: i for i, e in enumerate(kept)}
    estimates = [dict(image=(res[e]["scene_id"], res[e]["im_id"]), obj=res[e]["obj_id"], score=res[e]["score"])
                 for e in kept]
    gts, gpos = [], {}
    for s, im in setup["images"]:
        for k, (g, v) in enumerate(zip(scenes[s]["gt"][im], scenes[s]["visib"][im])):
            gpos[(s, im, k)] = len(gts)
            gts.append(dict(image=(s, im), obj=g["obj_id"], valid=v >= bop_eval.VISIB_GT_MIN))
    meshes = {o: bop_eval.read_ply(os.path.join(setup["mdir"], f"obj_{o:06d}.ply"))["vertices"] for o in setup["objects"]}
    errors = {}
    for g in setup["groups"]:
        s, im, o = g["scene_id"], g["im_id"], g["obj_id"]
        S = bop_eval.symmetry_transforms(info[o]).astype(np.float32)
        Kf = scenes[s]["K"][im].astype(np.float32)
        for e in g["est"]:
            Pe = bop_eval._pose(res[e]["R"], res[e]["t"]).astype(np.float32)
            for k in g["gt"]:
                gt = scenes[s]["gt"][im][k]
                Pg = bop_eval._pose(gt["R"], gt["t"]).astype(np.float32)
                errors[(pos[e], gpos[(s, im, k)])] = bop_port.mssd_mspd_fp32(meshes[o], S, Pe, Pg, Kf)
    diam = {o: info[o]["diameter"] for o in info}
    out = bop24_port.detection_scores(estimates, gts, errors, theta_mssd, theta_mspd, diam, r)
    out.update(kept=kept, errors=errors, pos=pos, gpos=gpos)
    return out


def test_readers_load_both_target_formats_and_cap_estimates_per_image(tmp_path):
    scenes, _ = write_detection_tree(tmp_path)
    assert bop_eval.load_target_images(str(tmp_path)) == [(2, 0), (2, 1)]
    assert bop_eval.load_target_images(str(tmp_path), "test_targets_bop19.json") == [(2, 0), (2, 1)]
    assert bop_eval.image_width(str(tmp_path), "test", 2, 1) == 16
    with pytest.raises(bop_eval.BopEvalError, match="rgb or gray"):
        bop_eval.image_width(str(tmp_path), "test", 2, 5)
    R, t = np.eye(3), [0.0, 0, 500]
    # scores with ties: csv order breaks them, and the cap counts every object's estimates of the image
    results = [_res(2, 0, o, s, R, t) for o, s in ((1, 0.5), (2, 0.7), (1, 0.7), (3, 0.9), (1, 0.5), (2, 0.1))]
    setup = bop_eval.prepare_detection(results, str(tmp_path), max_estimates_per_image=4)
    assert setup["objects"] == [1, 2, 4] and setup["n_valid"] == {1: 2, 2: 1, 4: 1}
    g = {(x["im_id"], x["obj_id"]): x for x in setup["groups"]}
    assert g[(0, 1)]["est"] == [2, 0] and g[(0, 2)]["est"] == [1]       # kept: 3, 1, 2, 0 (3 is object 3)
    assert g[(0, 2)]["gt"] == [1, 2] and g[(0, 2)]["valid"].tolist() == [True, False]
    assert (0, 3) not in g and g[(1, 4)]["est"] == [] and g[(1, 4)]["valid"].tolist() == [True]
    setup = bop_eval.prepare_detection(results, str(tmp_path), targets_name="test_targets_bop19.json")
    assert g[(0, 1)]["gt"] == [0] and [x["est"] for x in setup["groups"] if x["obj_id"] == 1][0] == [2, 0, 4]
    pairs = bop_eval.detection_pairs(setup)
    assert len(pairs["group"]) == sum(len(x["est"]) * len(x["gt"]) for x in setup["groups"])


def test_prepare_and_port_give_the_hand_computed_map(tmp_path):
    scenes, info = write_detection_tree(tmp_path)
    setup = bop_eval.prepare_detection(detection_results(scenes), str(tmp_path))
    assert setup["objects"] == [1, 2, 4]
    assert sorted(e for g in setup["groups"] for e in g["est"]) == [0, 1, 2, 3, 4]
    out = port_pipeline(setup, 16 / 640)
    want = (253 / 303 + 1.0 + 0.0) / 3
    for k in ("map", "map_mssd", "map_mspd"):
        assert out[k] == pytest.approx(want, abs=1e-14), k
    assert out["ap_mssd"][0].tolist() == [bop24_port.average_precision([TP, FP, TP], 2)] * 10
    assert out["ap_mssd"][1] == pytest.approx([1.0] * 10, abs=1e-14) and out["ap_mspd"][2].tolist() == [0.0] * 10
    assert out["labels"][out["pos"][3]].tolist() == [[IG] * 10] * 2
    assert bop_eval.average_time_per_image(setup["results"]) == pytest.approx(0.2)


def test_new_entry_points_reject_bad_arguments_without_a_gpu(lib):
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first
    i32 = lambda v: None if v is None else (C.c_int32 * max(1, len(v)))(*v)
    f64 = lambda v: None if v is None else (C.c_double * max(1, len(v)))(*v)

    def match(ng=2, no=1, nt=2, eo=(0, 2, 3), go=(0, 1, 1), gobj=(0, 0), thr=(1.0, 2.0, 3.0, 4.0), **null):
        p = dict(mssd=fake, mspd=fake, valid=fake, ws=fake, lab=fake)
        p.update(null)
        return lib.gp_bop_match(ng, no, nt, i32(eo), i32(go), i32(gobj), f64(thr), p["mssd"], p["mspd"], p["valid"],
                                p["ws"], p["lab"], None)
    cases = [(dict(ng=0), b"n_groups"), (dict(no=0), b"n_objects"), (dict(no=257), b"n_objects"),
             (dict(nt=0), b"n_theta"), (dict(nt=17), b"n_theta"), (dict(eo=None), b"null host"),
             (dict(thr=None), b"null host"), (dict(gobj=None), b"null host"), (dict(eo=(1, 2, 3)), b"offsets"),
             (dict(go=(0, 2, 1)), b"offsets"), (dict(thr=(1.0, float("nan"), 3.0, 4.0)), b"thresholds[1]"),
             (dict(thr=(1.0, 2.0, float("inf"), 4.0)), b"thresholds[2]"), (dict(gobj=(0, 1)), b"group_obj[1]"),
             (dict(go=(0, 1025, 1025)), b"more than 1024"), (dict(ws=fake + 4), b"aligned")]
    cases += [(dict(**{k: None}), b"null argument") for k in ("mssd", "mspd", "valid", "ws", "lab")]
    for kw, word in cases:
        assert match(**kw) == -1 and word in lib.gp_last_error(), (kw, lib.gp_last_error())

    def ap(no=2, nt=1, ne=3, ro=(0, 2, 3), nv=(1, 2), rec=(0.0, 0.5, 1.0), **null):
        p = dict(lab=fake, rank=fake, out=fake)
        p.update(null)
        return lib.gp_bop_average_precision(no, nt, ne, p["lab"], i32(ro), p["rank"], i32(nv), len(rec or ()) or 1,
                                            f64(rec), p["out"], None)
    cases = [(dict(no=0, ro=(0,)), b"n_objects"), (dict(nt=0), b"n_theta"), (dict(ne=0), b"n_est"),
             (dict(rec=tuple(np.linspace(0, 1, 129))), b"n_recall"), (dict(ro=None), b"null host"),
             (dict(nv=None), b"null host"), (dict(rec=None), b"null host"), (dict(ro=(0, 3, 2)), b"rank offsets"),
             (dict(ro=(2, 3, 3)), b"rank offsets"), (dict(nv=(1, 0)), b"n_valid[1]"),
             (dict(rec=(0.0, float("nan"))), b"recall_thresholds[1]"), (dict(rec=(0.0, 1.0, 0.5)), b"must not decrease")]
    cases += [(dict(**{k: None}), b"null argument") for k in ("lab", "rank", "out")]
    for kw, word in cases:
        assert ap(**kw) == -1 and word in lib.gp_last_error(), (kw, lib.gp_last_error())


def test_scores_bop24_keys_and_the_cli_default():
    src = open(bop_eval.__file__).read()
    for key in ("bop24_mAP", "bop24_mAP_mssd", "bop24_mAP_mspd", "bop24_average_time_per_image"):
        assert json.dumps(key) in src
    assert 'default="localization"' in src
