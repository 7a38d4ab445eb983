"""gp_teaser_refine (row f13) against its numpy restatement oracle/teaser_port.py on an H100: compacted points, sampled
indices, adjacency bits, clique, statuses and inlier counts exactly, R and t bit for bit; the planted edge cases;
batch determinism; each mutated definition fails; and the refiner on the rendered scenes of tests/icp_scenes.py."""
import numpy as np
import pytest
import torch

from gigapose_b200 import teaser
from gigapose_b200._lib import GpTeaserGnc
from oracle import teaser_port as tp
import teaser_scenes as ts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def frames(H, W, boxes_per_frame, seed=0, **kw):
    """Several frames with their own K; each box is one hypothesis of its frame."""
    depth, Ks, rendered, boxes, fidx = [], [], [], [], []
    for f, bxs in enumerate(boxes_per_frame):
        K = ts.intrinsics(H, W, seed=seed + f)
        r0 = ts.patch(H, W, (0, 0, W, H), seed=seed + f)
        depth.append(ts.measured(r0, K, seed=seed + 10 + f, **kw))
        Ks.append(K)
        for b in bxs:
            r = np.zeros_like(r0)
            x0, y0, x1, y1 = b
            r[y0:y1, x0:x1] = r0[y0:y1, x0:x1]
            rendered.append(r)
            boxes.append(b)
            fidx.append(f)
    return (np.stack(depth), np.stack(Ks), np.asarray(fidx), np.stack(rendered), np.asarray(boxes, np.int64),
            np.stack([ts.pose(seed + i) for i in range(len(boxes))]))


def run(depth, K, fidx, rendered, boxes, T0, debug=True, **params):
    n, H, W = rendered.shape
    p = dict(teaser.DEFAULTS, **params)
    cap = 8
    t = lambda a, dt=None: torch.as_tensor(np.ascontiguousarray(a), device=DEV, dtype=dt)  # noqa: E731
    dbg = dict(counts=torch.zeros(n, 4, dtype=torch.int32, device=DEV),
               points=torch.zeros(n, H * W, 6, device=DEV),
               samples=torch.full((n, p["n_points"]), -1, dtype=torch.int32, device=DEV),
               adjacency=torch.zeros(n, p["n_points"], 32, dtype=torch.int32, device=DEV),
               clique=torch.zeros(n, p["n_points"], dtype=torch.int32, device=DEV),
               gnc=torch.zeros(n, cap, np.dtype(GpTeaserGnc).itemsize, dtype=torch.uint8, device=DEV),
               gnc_weights=torch.zeros(n, cap, p["n_points"], dtype=torch.float64, device=DEV),
               transform=torch.zeros(n, 12, dtype=torch.float64, device=DEV)) if debug else None
    out = teaser.refine_rendered(t(depth), t(K), t(fidx, torch.int32), t(rendered), t(boxes), t(T0),
                                 debug=dict(dbg, gnc_capacity=cap) if debug else None, **params)
    torch.cuda.synchronize()
    res = [o.cpu().numpy() for o in out]
    if debug:
        d = {k: v.cpu().numpy() for k, v in dbg.items()}
        d["gnc"] = d["gnc"].view(np.dtype(GpTeaserGnc)).reshape(n, cap)
        res.append(d)
    return res


def compare(depth, K, fidx, rendered, boxes, T0, mutate=None, **params):
    poses, status, inl, clq, d = run(depth, K, fidx, rendered, boxes, T0, **params)
    ref = tp.refine(depth, K, fidx, rendered, boxes, T0, mutate=mutate, **params)
    for i, r in enumerate(ref):
        assert status[i] == r["status"], (i, status[i], r["status"])
        assert d["counts"][i, 0] == r["N"]
        if r["N"] > 0:
            np.testing.assert_array_equal(d["points"][i, :r["N"]], np.concatenate([r["src"], r["tgt"]], 1))
        if "samples" in r:
            M = r["M"]
            np.testing.assert_array_equal(d["samples"][i, :M], r["samples"])
            np.testing.assert_array_equal(d["adjacency"][i, :M].view(np.uint32), r["adjacency"])
            assert clq[i] == r["clique"]
        if "R" in r:
            m = len(r["members"])
            np.testing.assert_array_equal(d["clique"][i, :m], r["members"])
            np.testing.assert_array_equal(d["transform"][i, :9], r["R"].reshape(-1))
            np.testing.assert_array_equal(d["transform"][i, 9:], r["t"])
            assert inl[i] == r["inliers"]
            for it, g in enumerate(r["gnc"][:8]):
                np.testing.assert_array_equal(d["gnc"][i, it]["R"], g["R"])
                np.testing.assert_array_equal(d["gnc_weights"][i, it, :m], g["weights"])
        assert poses[i].tobytes() == r["pose"].tobytes(), i
    return poses, status, inl, clq, d, ref


@pytest.mark.parametrize("H,W,boxes", [
    (17, 17, [[(1, 1, 16, 16), (0, 0, 17, 9)], [(3, 2, 14, 17)]]),
    (480, 640, [[(250, 180, 330, 260), (200, 150, 380, 300)], [(100, 100, 160, 150), (300, 200, 420, 330)]]),
    (1080, 1920, [[(900, 500, 1100, 700)], [(400, 300, 520, 380), (1500, 800, 1920, 1080)]]),
])
def test_kernel_equals_port(H, W, boxes):
    params = dict(min_points=50) if H == 17 else {}
    _, status, *_ = compare(*frames(H, W, boxes), **params)
    assert (status == tp.OK).any()


def test_gnc_iterates_and_matches_on_noisy_scenes():
    """Noise of 3 mm makes the chain residuals large enough for GNC-TLS to iterate; its trace stays bit for bit."""
    args = frames(480, 640, [[(220, 160, 340, 280)], [(300, 200, 400, 300)]], seed=5, noise=3.0, outliers=0.3)
    *_, d, ref = compare(*args)
    assert max(len(r.get("gnc", [])) for r in ref) > 1


def test_clique_search_matches_on_outlier_graphs():
    """90 % outliers: the root's bound does not settle the clique, and the branch and bound visits the same nodes and
    keeps the same clique as the port's."""
    *_, d, ref = compare(*frames(64, 64, [[(5, 5, 40, 40)], [(0, 0, 64, 64)]], seed=7, noise=4.0, outliers=0.9))
    assert [d["counts"][i, 2] for i in range(2)] == [r["nodes"] for r in ref]
    assert min(r["nodes"] for r in ref) > 100


def test_edge_cases():
    H, W = 120, 160
    depth, K, fidx, rendered, boxes, T0 = frames(H, W, [[(10, 10, 60, 60)] * 7])
    r0 = rendered[0].copy()
    ys, xs = np.nonzero((r0 > 0) & (depth[0] > 0))
    for i, keep in enumerate((99, 100, 999)):          # 99, 100 and 999 masked points
        r = np.zeros_like(r0)
        r[ys[:keep], xs[:keep]] = r0[ys[:keep], xs[:keep]]
        rendered[i] = r
    rendered[3] = 0                                     # an empty render
    boxes[4] = (0, 0, 0, 0)                             # an empty box
    fidx[5] = 3                                         # an invalid frame
    # every correspondence identical: the measured depth equals the render -> mu <= 0 at the first iteration
    depth = np.concatenate([depth, rendered[6][None]])
    fidx[6] = 1
    poses, status, inl, clq, d, ref = compare(depth, K[[0, 0]], fidx, rendered, boxes, T0)
    assert [status[i] for i in (0, 3, 4, 5)] == [tp.TOO_FEW_POINTS, tp.TOO_FEW_POINTS, tp.TOO_FEW_POINTS, tp.INVALID]
    assert status[1] != tp.TOO_FEW_POINTS and status[2] != tp.TOO_FEW_POINTS
    assert d["counts"][1, 1] == 100 and d["counts"][2, 1] == 999
    assert status[6] == tp.OK and d["gnc"][6, 0]["stopped"] == 1


def planted_exact(H=33, W=33):
    """Integer principal point (16, 16), exact depths (multiples of 1/4 mm): the measured depth equals the render
    everywhere but at the principal point, where it is 1 mm deeper.  That pixel back-projects to (0, 0, d) in both
    clouds, so its correspondence is displaced by exactly (0, 0, 1) = noise_bound; every other correspondence is
    exact (depth / 1024 and the back-projection are exact), the clique is the exact ones, the solve gives R = I and
    t = 0 exactly, and that sample's residual is exactly the bound."""
    K = np.array([[1024.0, 0, 16.0], [0, 1024.0, 16.0], [0, 0, 1]], np.float32)
    v, u = np.mgrid[0:H, 0:W]
    r = np.zeros((H, W), np.float32)
    r[2:31, 2:31] = (700.0 + 0.25 * ((3 * u + 5 * v) % 8))[2:31, 2:31]
    m = r.copy()
    m[16, 16] += 1.0
    # edge bound 2 * 1 * sqrt(0.0625) = 0.5 mm: the displaced sample is inconsistent with its near neighbours (0.68 mm
    # apart) and stays out of the clique
    params = dict(unit_per_m=1.0, noise_bound=1.0, cbar2=0.0625, min_points=50, min_inliers=50)
    return (m[None], K[None], np.zeros(1, np.int64), r[None], np.array([[2, 2, 31, 31]], np.int64),
            np.stack([ts.pose(0)])), params


def test_inlier_exactly_at_the_noise_bound():
    """The reference counts ||T s - t|| < noise_bound: the planted sample at exactly the bound is an outlier in the
    kernel, and `<=` (the port's inlier_le mutation) would count it."""
    args, params = planted_exact()
    poses, status, inl, clq, d, ref = compare(*args, **params)
    N = int(d["counts"][0, 0])
    assert status[0] == tp.OK and N == 29 * 29
    assert np.array_equal(d["transform"][0], [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0])
    assert inl[0] == N - 1
    assert tp.refine(*args, mutate=dict(inlier_le=True), **params)[0]["inliers"] == N


def test_planted_fps_tie():
    """The first masked pixel sits on the principal column; the two farthest pixels are mirrored about that column at
    the same depth, so they are exactly as far from it in fp32: the lower index is sampled, in the kernel as in the
    port."""
    H = W = 33
    K = np.array([[64.0, 0, 16.0], [0, 64.0, 16.0], [0, 0, 1]], np.float32)
    r = np.zeros((H, W), np.float32)
    r[10, 16] = 700.0
    r[12, 14], r[13, 18] = 702.0, 701.0
    r[28, 4] = r[28, 28] = 704.0
    args = (r[None], K[None], np.zeros(1, np.int64), r[None], np.array([[0, 0, W, H]], np.int64),
            np.stack([ts.pose(0)]))
    src, _ = tp.points(r, r, (0, 0, W, H), K)
    dist = [(((p - src[0])[0] ** 2 + (p - src[0])[1] ** 2) + (p - src[0])[2] ** 2) for p in src]
    assert dist[3] == dist[4] and dist[3] > max(dist[1], dist[2])       # the tie is real, and at the maximum
    *_, d, ref = compare(*args, min_points=3, min_inliers=3)
    assert d["samples"][0, 1] == 3 and list(ref[0]["samples"]) == list(d["samples"][0, :5])


def test_tiny_node_budget_keeps_the_pose():
    """A one-node budget stops every search that the root's colouring bound does not settle: the budget status, and
    the input pose bit for bit (compare checks both against the port)."""
    args = frames(64, 64, [[(5, 5, 40, 40)], [(0, 0, 64, 64)]], seed=7, noise=4.0, outliers=0.9)
    poses, status, *_ = compare(*args, clique_budget=1)
    assert (status == tp.CLIQUE_BUDGET).any()
    for i in np.nonzero(status == tp.CLIQUE_BUDGET)[0]:
        assert poses[i].tobytes() == args[5][i].tobytes()


def test_batch_is_deterministic_and_per_hypothesis():
    args = frames(480, 640, [[(200 + 3 * i, 150 + 2 * i, 330 + 3 * i, 270 + 2 * i) for i in range(20)],
                             [(100 + 4 * i, 100, 220 + 4 * i, 200) for i in range(20)]], seed=11, noise=2.0)
    a = run(*args, debug=False)
    b = run(*args, debug=False)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    depth, K, fidx, rendered, boxes, T0 = args
    for i in (0, 17, 39):
        one = run(depth, K, fidx[i:i + 1], rendered[i:i + 1], boxes[i:i + 1], T0[i:i + 1], debug=False)
        for x, y in zip(one, a):
            assert x[0].tobytes() == y[i].tobytes()


@pytest.mark.parametrize("mutate", [dict(fps_start=1), dict(edge_scale=1.0), dict(compose_right=True),
                                    dict(pad_copies=True)])
def test_each_mutation_fails(mutate):
    """Each altered definition in the port gives another sample, clique, status, inlier count or pose than the
    kernel on these scenes; the first box has fewer than 1000 masked points, so restoring the padding copies shows.
    (`<=` for the inlier count needs a sample exactly at the bound: test_inlier_exactly_at_the_noise_bound.)"""
    args = frames(64, 64, [[(5, 5, 30, 30), (10, 8, 60, 50)], [(0, 0, 64, 64)]], seed=3, noise=2.0)
    poses, status, inl, clq, d = run(*args)
    ref = tp.refine(*args, mutate=mutate)
    same = all(status[i] == r["status"] and inl[i] == r["inliers"] and poses[i].tobytes() == r["pose"].tobytes()
               and d["counts"][i, 1] == r["M"] and clq[i] == r["clique"]
               and (r["M"] == 0 or np.array_equal(d["samples"][i, :r["M"]], r["samples"])) for i, r in enumerate(ref))
    assert not same


@pytest.fixture(scope="module")
def scenes():
    import icp_scenes as S
    from gigapose_b200.icp import device_meshes, refine_icp
    meshes = device_meshes([S.ellipsoid(), S.assembly()], DEV)
    out = []
    for lab, T in ((0, S.T_ELL), (1, S.T_ASM)):
        d, _ = S.scene([S.ellipsoid(), S.assembly()][lab], T)
        out.append((lab, T, d))
    d, _ = S.noisy_occluded_scene(S.ellipsoid(), S.T_ELL)
    out.append((0, S.T_ELL, d))
    return S, meshes, out, refine_icp


def _errors(T, T_true):
    dR = T[:3, :3].astype(np.float64).T @ T_true[:3, :3].astype(np.float64)
    return (float(np.linalg.norm(T[:3, 3] - T_true[:3, 3])),
            float(np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))))


# reached errors (mm, degrees) measured on an H100, per scene and start; pinned with a 25 % + 0.1 margin
PINNED = {(0, 0): (7.03, 6.14), (0, 1): (0.97, 1.07), (1, 0): (6.53, 16.65), (1, 1): (0.87, 1.22), (2, 0): (4.58, 6.81),
          (2, 1): (0.07, 2.28)}


def test_rendered_scenes_reached_errors(scenes):
    """Started from row f6's offsets and from a depth-only offset, every pose is accepted, its translation error is
    lower than the coarse pose's, and both errors are pinned.  The rotation is not improved from a 6 degree start
    (pixel-aligned correspondences assume the pose is right in the image plane).  The ICP's result on the same starts
    is printed beside, without asserting which is better."""
    S, meshes, sc, refine_icp = scenes
    for k, (lab, T_true, d) in enumerate(sc):
        for j, (axis, deg, dt) in enumerate((([0.2, 1.0, 0.1], 6.0, [8.0, -5.0, 6.0]), ([1, 0, 0], 0.0, [0.0, 0.0, 15.0]))):
            T0 = S.perturb(T_true, axis, deg, dt)
            args = (meshes, [lab], torch.as_tensor(T0[None], device=DEV), d, S.K, [0])
            p, st, inl, clq = teaser.refine_teaserpp(*args)
            pi, sti, *_ = refine_icp(*args)
            e0, e1, ei = _errors(T0, T_true), _errors(p[0].cpu().numpy(), T_true), _errors(pi[0].cpu().numpy(), T_true)
            print(f"scene {k} start {e0} teaser {teaser.STATUS_NAMES[int(st[0])]} {e1} inliers {int(inl[0])} "
                  f"clique {int(clq[0])}  icp {int(sti[0])} {ei}")
            assert int(st[0]) == tp.OK and e1[0] < e0[0]
            bt, br = PINNED[(k, j)]
            assert e1[0] <= 1.25 * bt + 0.1 and e1[1] <= 1.25 * br + 0.1, (k, j, e1)
