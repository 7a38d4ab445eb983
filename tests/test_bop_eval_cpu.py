"""Row f7 without a GPU: the BOP dataset readers, the symmetry discretisation, the matching into recalls, the numpy
port's VSD on cases with a known answer, and the argument checks of gp_render_depth, gp_bop_vsd and gp_bop_mssd_mspd."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from bop_tree import rot, tetra, write_tree
from gigapose_b200 import _lib, bop_eval, build
from oracle import bop_port

K = np.array([[500.0, 0, 80.0], [0, 500.0, 60.0], [0, 0, 1]])


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def _tree(root):
    rng = np.random.default_rng(0)
    V, F = tetra()
    info = {1: dict(diameter=70.7), 2: dict(diameter=55.0, symmetries_discrete=[np.diag([-1.0, -1, 1, 1]).ravel().tolist()]),
            3: dict(diameter=80.0, symmetries_continuous=[dict(axis=[0, 0, 1], offset=[1.0, 2.0, 0])])}
    scenes = {}
    for s in (1, 4):
        scenes[s] = {}
        for im in (0, 3):
            scenes[s][im] = dict(gt=[(1, rot([0, 1, 0], 10 * im + s), [1.5, -2.0, 600.0 + s]), (2, np.eye(3), [0, 0, 700.0])],
                                 visib=[0.5 + 0.1 * im, 0.09], K=K + s, depth_scale=0.1 * (s + 1),
                                 png=rng.integers(0, 65535, (12, 16)))
    write_tree(str(root), {1: (V, F), 2: (V, F), 3: (V, F)}, info, scenes,
               [(1, 0, 1, 1), (1, 3, 2, 1), (4, 0, 1, 2)])
    return scenes, info


def test_readers_read_back_a_synthetic_tree(tmp_path):
    scenes, info = _tree(tmp_path)
    for s, ims in scenes.items():
        sc = bop_eval.load_scene(str(tmp_path), "test", s)
        assert sorted(sc["gt"]) == sorted(ims)
        for im, v in ims.items():
            assert sc["visib"][im] == v["visib"]
            np.testing.assert_array_equal(sc["K"][im], v["K"])
            assert sc["depth_scale"][im] == v["depth_scale"]
            for got, (o, R, t) in zip(sc["gt"][im], v["gt"]):
                assert got["obj_id"] == o
                np.testing.assert_array_equal(got["R"], np.asarray(R, float))
                np.testing.assert_array_equal(got["t"], np.asarray(t, float))
            d = bop_eval.load_depth(str(tmp_path), "test", s, im, sc["depth_scale"][im])
            assert d.dtype == np.float32
            np.testing.assert_array_equal(d, (v["png"].astype(np.float64) * v["depth_scale"]).astype(np.float32))
    mi = bop_eval.load_models_info(bop_eval.models_dir(str(tmp_path)))
    assert mi[1]["diameter"] == 70.7 and mi[1]["symmetries_discrete"] == [] and mi[1]["symmetries_continuous"] == []
    np.testing.assert_array_equal(mi[2]["symmetries_discrete"][0], np.diag([-1.0, -1, 1, 1]))
    axis, off = mi[3]["symmetries_continuous"][0]
    np.testing.assert_array_equal(axis, [0, 0, 1])
    np.testing.assert_array_equal(off, [1, 2, 0])
    assert bop_eval.load_targets(str(tmp_path)) == [
        dict(scene_id=1, im_id=0, obj_id=1, inst_count=1), dict(scene_id=1, im_id=3, obj_id=2, inst_count=1),
        dict(scene_id=4, im_id=0, obj_id=1, inst_count=2)]


def test_a_dataset_without_depth_is_refused(tmp_path):
    _tree(tmp_path)
    os.rename(tmp_path / "test" / "000001" / "depth", tmp_path / "test" / "000001" / "nodepth")
    with pytest.raises(bop_eval.BopEvalError, match="depth"):
        bop_eval.load_depth(str(tmp_path), "test", 1, 0, 1.0)


def test_a_targets_file_without_targets_is_refused(tmp_path):
    """Refused while reading the dataset, before any device work: there is nothing to score."""
    _tree(tmp_path)
    with open(tmp_path / "test_targets_bop19.json", "w") as f:
        json.dump([], f)
    with pytest.raises(bop_eval.BopEvalError, match="lists no targets"):
        bop_eval.evaluate([], str(tmp_path), device="cuda:0")


def test_symmetry_counts_fixed_axis_and_composition_order():
    n = int(np.ceil(np.pi / 0.01))
    assert n == 315
    assert len(bop_eval.symmetry_transforms({})) == 1
    D = [np.diag([-1.0, -1, 1, 1]), np.diag([1.0, -1, -1, 1])]
    assert len(bop_eval.symmetry_transforms(dict(symmetries_discrete=D))) == 3
    axis, off = np.array([0.3, -0.2, 1.0]), np.array([5.0, -7.0, 2.0])
    cont = dict(symmetries_continuous=[(axis, off)])
    T = bop_eval.symmetry_transforms(cont)
    assert len(T) == n
    np.testing.assert_allclose(T[0], np.eye(4), atol=1e-15)
    line = off + np.linspace(-50, 50, 7)[:, None] * axis / np.linalg.norm(axis)
    for Tk in T:
        np.testing.assert_allclose(line @ Tk[:3, :3].T + Tk[:3, 3], line, atol=1e-11)
        np.testing.assert_allclose(Tk[:3, :3] @ Tk[:3, :3].T, np.eye(3), atol=1e-12)
    # consecutive steps are 2 pi / n apart
    ang = np.arccos(np.clip((np.trace(T[1][:3, :3] @ T[0][:3, :3].T) - 1) / 2, -1, 1))
    assert abs(ang - 2 * np.pi / n) < 1e-12
    both = bop_eval.symmetry_transforms(dict(symmetries_discrete=D, **cont))
    assert len(both) == 3 * n
    disc = [np.eye(4)] + D
    for i, Dm in enumerate(disc):
        for k in (0, 1, 200):
            np.testing.assert_allclose(both[i * n + k], T[k] @ Dm, atol=1e-15)
    two = bop_eval.symmetry_transforms(dict(symmetries_continuous=[(axis, off), (np.array([1.0, 0, 0]), np.zeros(3))]))
    assert len(two) == 2 * n


def test_matching_rules():
    inf = np.inf
    valid = np.array([True, True])
    # descending score order: the first estimate takes the ground truth both want
    assert bop_eval.match_group([[1.0, 5.0], [1.0, inf]], valid, [2.0]).tolist() == [1]
    assert bop_eval.match_group([[1.0, inf], [1.0, 5.0]], valid, [2.0, 6.0]).tolist() == [1, 2]
    # an error equal to the threshold does not match
    assert bop_eval.match_group([[2.0, inf]], valid, [2.0, np.nextafter(2.0, 3)]).tolist() == [0, 1]
    # the smallest error wins among the unmatched
    assert bop_eval.match_group([[3.0, 1.0], [0.5, 0.6]], valid, [4.0]).tolist() == [2]
    # a ground truth below the visibility cut is not matchable
    assert bop_eval.match_group([[0.1, 0.2]], np.array([False, True]), [1.0]).tolist() == [1]
    assert bop_eval.match_group(np.zeros((0, 2)), valid, [1.0]).tolist() == [0]


def test_prepare_applies_top_n_and_the_visibility_cut(tmp_path):
    scenes, _ = _tree(tmp_path)
    R = np.eye(3)
    results = [dict(scene_id=4, im_id=0, obj_id=1, score=s, R=R, t=np.zeros((3, 1)), time=0.5) for s in (0.2, 0.9, 0.5)]
    results.append(dict(scene_id=1, im_id=3, obj_id=2, score=1.0, R=R, t=np.zeros((3, 1)), time=0.25))
    setup = bop_eval.prepare(results, str(tmp_path))
    g = {(x["scene_id"], x["im_id"], x["obj_id"]): x for x in setup["groups"]}
    assert g[(4, 0, 1)]["est"] == [1, 2]                  # the top inst_count = 2 by score
    assert g[(1, 0, 1)]["est"] == []                      # a target image without estimates
    assert g[(1, 3, 2)]["gt"] == [1] and g[(1, 3, 2)]["valid"].tolist() == [False]    # visib_fract 0.09
    assert g[(1, 0, 1)]["valid"].tolist() == [True]
    # targets: only visib_fract >= 0.1 counts; a target without estimates still counts
    groups = [dict(vsd=np.zeros((0, 1, 1)), mssd=np.zeros((0, 1)), mspd=np.zeros((0, 1)), valid=np.array([True]),
                   diameter=10.0),
              dict(vsd=np.zeros((1, 2, 1)), mssd=np.zeros((1, 2)), mspd=np.zeros((1, 2)),
                   valid=np.array([np.float64(0.1) >= bop_eval.VISIB_GT_MIN, np.float64(0.09) >= bop_eval.VISIB_GT_MIN]),
                   diameter=10.0)]
    assert groups[1]["valid"].tolist() == [True, False]
    rec = bop_eval.recalls(groups, 2, taus=(0.3,), theta_vsd=(0.1,), theta_mssd=(0.1,), theta_mspd=(5.0,))
    assert rec["vsd"].tolist() == [[0.5]] and rec["mssd"].tolist() == [0.5] and rec["mspd"].tolist() == [0.5]
    assert bop_eval.average_time_per_image(results) == 0.375
    assert bop_eval.average_time_per_image(results + [dict(scene_id=9, im_id=9, time=-1)]) == -1.0


def test_port_matcher_agrees_with_the_product_matcher():
    rng = np.random.default_rng(4)
    groups, pairs, targets = [], [], []
    for ti in range(40):
        ne, ng = rng.integers(0, 4), rng.integers(1, 4)
        valid = rng.random(ng) > 0.2
        vsd = rng.random((ne, ng, 3)).round(2)
        mssd, mspd = rng.random((ne, ng)) * 20, rng.random((ne, ng)) * 40
        groups.append(dict(vsd=vsd, mssd=mssd, mspd=mspd, valid=valid, diameter=50.0))
        targets.append(dict(valid=dict(enumerate(valid.tolist())), diameter=50.0))
        for a in range(ne):
            for b in range(ng):
                pairs.append(dict(target=ti, rank=a, gt=b, vsd=vsd[a, b], mssd=mssd[a, b], mspd=mspd[a, b]))
    n = sum(int(g["valid"].sum()) for g in groups)
    taus, th = (0.1, 0.2, 0.3), (0.05, 0.2, 0.35, 0.5)
    mine = bop_eval.recalls(groups, n, taus, th, th, (5.0, 20.0), r=1.5)
    port = bop_port.average_recalls(pairs, targets, taus, th, th, (5.0, 20.0), r=1.5)
    np.testing.assert_array_equal(mine["vsd"], port["recall_vsd"])
    np.testing.assert_array_equal(mine["mssd"], port["recall_mssd"])
    np.testing.assert_array_equal(mine["mspd"], port["recall_mspd"])


def _plate(H, W, box, z):
    d = np.zeros((H, W), np.float32)
    x0, y0, x1, y1 = box
    d[y0:y1, x0:x1] = z
    return d


def test_port_vsd_analytic_cases():
    H, W, taus = 120, 160, (0.05, 0.099, 0.101, 0.3)
    box = (75, 55, 86, 66)                         # 11 x 11 px around the principal point (80, 60)
    gt = _plate(H, W, box, 1000.0)
    test = gt.copy()
    for fn in (bop_port.vsd_fp32, lambda t, k, e, eb, g, gb, *a: bop_port.vsd_fp64(t, k, e, g, *a)):
        c, e = fn(test, K, gt, box, gt, box, 100.0, 15.0, taus)
        assert c[:2].tolist() == [121, 121] and np.all(e == 0)                        # identical renders
        other = (10, 10, 20, 20)
        est = _plate(H, W, other, 1000.0)
        c, e = fn(test, K, est, other, gt, box, 100.0, 15.0, taus)
        assert c[0] == 0 and c[1] == 221 and np.all(e == 1)                          # no overlap
        # a plate 10 mm behind: |dist difference| / diameter = 0.1 x (1 + < 1e-4) -> a step between 0.099 and 0.101
        est = _plate(H, W, box, 1010.0)
        c, e = fn(test, K, est, box, gt, box, 100.0, 15.0, taus)
        assert c.tolist() == [121, 121, 121, 121, 0, 0], c
        assert e.tolist() == [1, 1, 0, 0]
        # half of the ground truth behind an occluder 200 mm in front: that half leaves visib_gt (and the estimate,
        # identical, keeps only what visib_gt keeps)
        occ = test.copy()
        occ[:, :81] = np.where(gt[:, :81] > 0, 800.0, 0)
        c, e = fn(occ, K, gt, box, gt, box, 100.0, 15.0, taus)
        assert c[:2].tolist() == [55, 55] and np.all(e == 0)
        # an estimate where the test depth is missing is visible (d_test == 0)
        c, e = fn(np.zeros_like(test), K, est, box, gt, box, 100.0, 15.0, taus)
        assert c[:2].tolist() == [121, 121]
    # fp32 distance at the principal point is the depth itself
    assert bop_port.dist_fp32(np.full((1, 1), 1234.5, np.float32), K, 80, 60)[0, 0] == np.float32(1234.5)


def test_port_mssd_of_a_declared_symmetry_is_zero():
    V, _ = tetra()
    P = np.eye(4, dtype=np.float32)
    P[:3, 3] = (0, 0, 500)
    S = np.eye(4)
    S[:3, :3] = rot([0, 0, 1], 90)
    Pe = P.copy()
    Pe[:3, :3] = (P[:3, :3] @ S[:3, :3]).astype(np.float32)
    syms = np.stack([np.eye(4), S]).astype(np.float32)
    m32 = bop_port.mssd_mspd_fp32(V, syms, Pe, P, K)
    m64 = bop_port.mssd_mspd_fp64(V, syms, Pe, P, K)
    assert m32[0] < 1e-4 and m64[0] < 1e-9
    no_sym = bop_port.mssd_mspd_fp64(V, syms[:1], Pe, P, K)
    assert no_sym[0] > 50


def test_new_entry_points_reject_bad_arguments_without_a_gpu(lib):
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first

    def rd(n=1, H=10, W=10, nv=3, V=fake, nf=1, Fc=fake, poses=fake, Km=fake, z=1.0, ws=fake, d=fake, b=fake):
        return lib.gp_render_depth(n, H, W, nv, V, nf, Fc, poses, Km, z, ws, d, b, None)
    for kw, word in ((dict(n=-1), b"n_views"), (dict(H=0), b"image size"), (dict(W=9000), b"image size"),
                     (dict(z=0.0), b"z_near"), (dict(z=float("inf")), b"z_near"), (dict(nv=-1), b"negative"),
                     (dict(V=None), b"null"), (dict(d=None), b"null"), (dict(b=None), b"null"),
                     (dict(ws=None), b"null"), (dict(Km=None), b"null")):
        assert rd(**kw) == -1 and word in lib.gp_last_error(), kw
    assert rd(n=0) == 0                                # nothing to do

    def vsd(n=1, F=1, H=10, W=10, ne=1, ng=1, delta=15.0, n_tau=2, tau=(0.1, 0.2), **null):
        p = dict(dt=fake, K=fake, fi=fake, ed=fake, eb=fake, ei=fake, gd=fake, gb=fake, gi=fake, diam=fake, cnt=fake,
                 err=fake)
        p.update(null)
        t = None if tau is None else (C.c_float * max(1, len(tau)))(*tau)
        return lib.gp_bop_vsd(n, F, H, W, p["dt"], p["K"], p["fi"], ne, p["ed"], p["eb"], p["ei"], ng, p["gd"], p["gb"],
                              p["gi"], p["diam"], delta, n_tau, t, p["cnt"], p["err"], None)
    cases = [(dict(n=0), b"n_pairs"), (dict(n=-2), b"n_pairs"), (dict(F=0), b"n_frames"), (dict(ne=0), b"n_est"),
             (dict(H=0), b"image size"), (dict(n_tau=0), b"n_tau"), (dict(n_tau=17, tau=(0.1,) * 17), b"n_tau"),
             (dict(delta=0.0), b"delta"), (dict(delta=-1.0), b"delta"), (dict(delta=float("nan")), b"delta"),
             (dict(tau=(0.1, 0.0)), b"tau[1]"), (dict(tau=(float("inf"), 0.1)), b"tau[0]"), (dict(tau=None), b"null")]
    cases += [(dict(**{k: None}), b"null") for k in ("dt", "K", "fi", "ed", "eb", "ei", "gd", "gb", "gi", "diam", "cnt",
                                                     "err")]
    for kw, word in cases:
        assert vsd(**kw) == -1 and word in lib.gp_last_error(), (kw, lib.gp_last_error())

    def ms(n=1, vo=(0, 4, 9), so=(0, 1, 3), F=1, **null):
        p = dict(obj=fake, V=fake, S=fake, K=fake, fi=fake, pe=fake, pg=fake, o1=fake, o2=fake)
        p.update(null)
        v = None if vo is None else (C.c_int32 * len(vo))(*vo)
        s = None if so is None else (C.c_int32 * len(so))(*so)
        return lib.gp_bop_mssd_mspd(n, len(vo or so or (0, 0)) - 1, p["obj"], v, p["V"], s, p["S"], F, p["K"], p["fi"],
                                    p["pe"], p["pg"], p["o1"], p["o2"], None)
    cases = [(dict(n=0), b"n_pairs"), (dict(F=0), b"n_frames"), (dict(vo=(0,), so=(0,)), b"n_objects"),
             (dict(vo=(1, 4, 9)), b"offsets at object 0"), (dict(so=(0, 1, 1)), b"offsets at object 2"),
             (dict(vo=(0, 4, 3)), b"offsets at object 2"), (dict(so=(0, -1, 3)), b"offsets at object 1"),
             (dict(vo=None), b"null offsets"), (dict(so=None), b"null offsets"),
             (dict(vo=tuple(range(258)), so=tuple(range(258))), b"n_objects")]
    cases += [(dict(**{k: None}), b"null") for k in ("obj", "V", "S", "K", "fi", "pe", "pg", "o1", "o2")]
    for kw, word in cases:
        assert ms(**kw) == -1 and word in lib.gp_last_error(), (kw, lib.gp_last_error())


def test_scores_keys_match_what_the_reference_reads():
    """The keys eval_bop.py copies out of scores_bop19.json."""
    src = open(bop_eval.__file__).read()
    for key in ("bop19_average_recall", "bop19_average_recall_vsd", "bop19_average_recall_mssd",
                "bop19_average_recall_mspd", "bop19_average_time_per_image"):
        assert json.dumps(key) in src
