"""The TEASER++ refiner's numpy restatement (oracle/teaser_port.py, row f13) against the independent fp64 evaluator
tests/teaser_fp64.py and against planted cases, and gp_teaser_refine's argument checks, without a GPU."""
import ctypes as C
import os

import numpy as np
import pytest

import teaser_fp64 as ev
import teaser_scenes as ts
from gigapose_b200 import _lib, build, teaser
from oracle import teaser_port as tp


GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "teaser_scenes.npz"))


@pytest.mark.parametrize("case", ["full", "padded", "skip", "rejected"])
def test_port_reproduces_the_reference_refiner(case):
    """tests/golden/teaser_scenes.npz, written by oracle/make_golden_teaser.py from the reference's own
    compute_teaserpp_refinement and TeaserppRefiner.refine_poses (metres; planted FPS indices and R, t)."""
    g = {k[len(case) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(case + "_")}
    K = GOLDEN["K"]
    D, R, T0 = g["depth"], g["rendered"], g["T0"]
    H, W = D.shape
    src, tgt = tp.points(D, R, (0, 0, W, H), K)
    assert len(src) == int(g["mask_count"])                                     # the mask count
    if case == "skip":                                                          # below n_min_points = 100
        assert len(src) == 99 and g["pose"].tobytes() == T0.tobytes()
        o = tp.refine_one(D, R, (0, 0, W, H), K, T0, unit_per_m=1.0)
        assert o["status"] == tp.TOO_FEW_POINTS and o["pose"].tobytes() == T0.tobytes()
        return
    assert src.tobytes() == g["pc_src_mask"].tobytes() and tgt.tobytes() == g["pc_tgt_mask"].tobytes()
    # the reference's samples: pytorch3d's indices, -1 past N, which its indexing turns into the last masked point
    idx = g["fps"]
    assert np.array_equal(idx, tp.fps(src, min(1000, len(src))))
    pad = np.concatenate([idx, np.full(1000 - len(idx), len(src) - 1)]) if len(idx) < 1000 else idx
    assert src[pad].tobytes() == g["pc_src"].tobytes() and tgt[pad].tobytes() == g["pc_tgt"].tobytes()
    assert np.array_equal(g["solver_src"], g["pc_src"].T)                      # teaserpp_python gets [3,N]
    o = tp.refine_one(D, R, (0, 0, W, H), K, T0, unit_per_m=1.0, mutate=dict(pad_copies=True))
    assert np.array_equal(o["samples"], pad)                                    # the mutation is the reference's padding
    if case == "padded":                                                        # the port's deviation: N distinct samples
        assert np.array_equal(tp.refine_one(D, R, (0, 0, W, H), K, T0, unit_per_m=1.0)["samples"], idx)
    # the strict inlier count on the reference's sampled clouds, with its planted R, t and noise_bound = 0.01 m
    n_in = tp.inliers(g["R"].reshape(-1), g["t"], g["pc_src"], g["pc_tgt"], 0.01)
    assert n_in == int(g["num_inliers"])
    # acceptance at >= 50 inliers, and the pose T @ TCO
    accepted = g["pose"].tobytes() != T0.tobytes()
    assert accepted == (int(g["num_inliers"]) >= 50) and accepted == (case != "rejected")
    if accepted:
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = g["R"], g["t"]
        np.testing.assert_array_max_ulp(tp.compose(T, T0), g["pose"], maxulp=1)
        assert np.abs(tp.compose(T, T0, right=True) - g["pose"]).max() > 1e-3


def scene(seed=7, outliers=0.9, noise=4.0, box=(5, 5, 40, 40), H=64, W=64):
    K = ts.intrinsics(H, W, seed=seed)
    r0 = ts.patch(H, W, (0, 0, W, H), seed=seed)
    m = ts.measured(r0, K, seed=seed + 10, noise=noise, outliers=outliers)
    r = np.zeros_like(r0)
    x0, y0, x1, y1 = box
    r[y0:y1, x0:x1] = r0[y0:y1, x0:x1]
    return m, r, box, K


def test_points_are_the_reference_back_projection():
    """get_pointcloud's formula (meshcat_utils.py:306-312) on the full frame, then boolean indexing."""
    m, r, box, K = scene()
    src, tgt = tp.points(m, r, box, K)
    H, W = m.shape
    px, py = np.meshgrid(np.linspace(0, W - 1, W), np.linspace(0, H - 1, H))
    mask = (m > 0) & (r > 0)
    for d, got in ((r, src), (m, tgt)):
        ref = np.float32([(px - K[0, 2]) * (d / K[0, 0]), (py - K[1, 2]) * (d / K[1, 1]), d]).transpose(1, 2, 0)
        assert ref[mask].tobytes() == got.tobytes()


def test_fps_agrees_with_fp64_except_at_ties():
    m, r, box, K = scene(outliers=0.1, noise=0.5)
    src, _ = tp.points(m, r, box, K)
    got = tp.fps(src, 300)
    ref, gaps = ev.fps(src, 300)
    diff = np.nonzero(got != ref)[0]
    # the sequences agree up to the first step whose winner leads by less than the fp32 rounding of the distances
    if len(diff):
        k = diff[0]
        scale = float((src.astype(np.float64) ** 2).sum(1).max())
        assert gaps[k - 1] <= 1e-5 * scale, (k, gaps[k - 1])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_clique_is_maximum(seed):
    m, r, box, K = scene(seed=seed)
    src, tgt = tp.points(m, r, box, K)
    idx = tp.fps(src, 200)
    adj = tp.graph(src[idx], tgt[idx], 10.0, 1.0)
    members, size, nodes, over = tp.max_clique(adj, 10 ** 7)
    assert not over and size == len(members) and ev.is_clique(adj, members)
    assert size == ev.clique_size(adj)


def test_clique_on_1000_vertices_is_certified_by_a_colouring():
    m, r, box, K = scene(outliers=0.05, noise=1.0, box=(0, 0, 64, 64))
    src, tgt = tp.points(m, r, box, K)
    idx = tp.fps(src, 1000)
    adj = tp.graph(src[idx], tgt[idx], 10.0, 1.0)
    members, size, nodes, over = tp.max_clique(adj, 20000)
    assert not over and ev.is_clique(adj, members)
    assert size == ev.colouring_bound(adj)             # a colouring with as many colours as members certifies it


def test_gnc_steps_agree_with_svd_from_the_traced_weights():
    m, r, box, K = scene(seed=5, outliers=0.3, noise=3.0, box=(5, 5, 60, 60))
    o = tp.refine_one(m, r, box, K, ts.pose(), min_points=50)
    assert len(o["gnc"]) > 1
    s, t = tp.points(m, r, box, K)
    s, t = s[o["samples"]], t[o["samples"]]
    a, b = o["members"], np.roll(o["members"], -1)
    S, T = s[b].astype(np.float64) - s[a], t[b].astype(np.float64) - t[a]
    eps2 = (float(np.float32(0.01)) * 1000.0) ** 2       # noise_bound is an fp32 parameter
    worst = 0.0
    for k, g in enumerate(o["gnc"]):
        R = ev.kabsch(g["weights"], S, T)
        worst = max(worst, float(np.abs(R - g["R"].reshape(3, 3)).max()))
        if k + 1 < len(o["gnc"]):
            res = ((T - S @ g["R"].reshape(3, 3).T) ** 2).sum(1)
            # w = sqrt(eps2 mu (mu + 1) / r) - mu cancels as mu grows: the bar scales with the two terms
            bar = 1e-9 * (np.sqrt(eps2 * g["mu"] * (g["mu"] + 1) / np.maximum(res, 1e-300)) + g["mu"])
            assert (np.abs(ev.gnc_weights(res, g["mu"], eps2) - o["gnc"][k + 1]["weights"]) <= bar).all()
    assert worst < 1e-9, worst


def test_voting_agrees_with_the_brute_force():
    rng = np.random.default_rng(0)
    for _ in range(20):
        x = np.concatenate([rng.normal(3.0, 2.0, 40), rng.uniform(-200, 200, 30)])
        got, ref = tp.vote(x, 10.0, 1000.0), ev.vote(x, 10.0, 1000.0)
        assert abs(got - ref) < 1e-9 * max(1.0, abs(ref))


def test_edge_at_the_threshold_and_one_ulp_either_side():
    s = np.zeros((4, 3), np.float32)
    s[:, 2] = 700
    s[1, 0], s[2, 0], s[3, 0] = 100.0, 50.0, 30.0
    t = s.copy()
    t[1, 0] = 120.0                                     # | 120 - 100 | = 20 = 2 noise exactly: an edge
    t[2, 0] = np.nextafter(np.float32(70.0), np.float32(100))    # one ulp past: none
    t[3, 0] = np.nextafter(np.float32(50.0), np.float32(0))      # one ulp inside: an edge
    adj = tp.graph(s, t, 10.0, 1.0)
    assert adj[0, 1] and not adj[0, 2] and adj[0, 3]
    assert not tp.graph(s, t, 10.0, 1.0, edge_scale=1.0)[0, 1]


def test_skip_below_min_points():
    m, r, box, K = scene(box=(5, 5, 15, 14))
    src, _ = tp.points(m, r, box, K)
    o = tp.refine_one(m, r, box, K, np.eye(4), min_points=len(src) + 1)
    assert o["status"] == tp.TOO_FEW_POINTS
    assert tp.refine_one(m, r, box, K, np.eye(4), min_points=len(src))["status"] != tp.TOO_FEW_POINTS


def test_padding_copies_inflate_the_clique():
    """The reference's padding (the golden `padded` case: 400 masked points, 600 copies of the last one) makes the
    copies mutually consistent members of the clique and inliers: 943 inliers of 400 points."""
    g = {k[7:]: GOLDEN[k] for k in GOLDEN.files if k.startswith("padded_")}
    assert int(g["mask_count"]) == 400 and int(g["num_inliers"]) > 400
    D, R, T0, K = g["depth"], g["rendered"], g["T0"], GOLDEN["K"]
    o = tp.refine_one(D, R, (0, 0, 64, 48), K, T0, unit_per_m=1.0)
    p = tp.refine_one(D, R, (0, 0, 64, 48), K, T0, unit_per_m=1.0, mutate=dict(pad_copies=True))
    assert o["M"] == 400 and p["M"] == 1000 and p["clique"] >= o["clique"] + 600


def test_teaser_argument_checks_need_no_gpu():
    build.build()
    lib = _lib.load()
    ok = teaser.make_params()
    b = C.c_size_t()
    assert lib.gp_teaser_query_sizes(2, 480, 640, C.byref(b)) == 0 and b.value >= 2 * 28 * 480 * 640
    assert lib.gp_teaser_query_sizes(0, 480, 640, C.byref(b)) == -1
    for bad in (dict(n_points=2), dict(n_points=1025), dict(noise_bound=0.0), dict(cbar2=-1.0), dict(min_points=0),
                dict(gnc_factor=1.0), dict(gnc_max_iters=0), dict(clique_budget=0), dict(min_inliers=-1)):
        p = teaser.make_params(**bad)
        rc = lib.gp_teaser_refine(1, 1, 17, 17, 1, 1, 1, 1, 1, 1, C.byref(p), 1, 1, 1, 1, 1024, None)
        assert rc == -1, bad
    rc = lib.gp_teaser_refine(1, 1, 17, 17, None, 1, 1, 1, 1, 1, C.byref(ok), 1, 1, 1, 1, 1024, None)
    assert rc == -1 and b"null" in lib.gp_last_error()
    with pytest.raises(TypeError):
        teaser.make_params(noise=1)


def test_bop_run_flag_parses_and_refuses_masks():
    from gigapose_b200 import bop_run
    a = bop_run.parser().parse_args(["--dataset-dir", "d", "--checkpoint", "c", "--template-poses", "p",
                                     "--refine-depth", "2", "--depth-refiner", "teaserpp"])
    assert a.depth_refiner == "teaserpp" and a.refine_depth == 2
    assert bop_run.parser().parse_args(["--dataset-dir", "d", "--checkpoint", "c",
                                        "--template-poses", "p"]).depth_refiner == "icp"
    with pytest.raises(SystemExit):
        bop_run.main(["--dataset-dir", "d", "--checkpoint", "c", "--template-poses", "p", "--refine-depth", "2",
                      "--depth-refiner", "teaserpp", "--refine-masks"])
