"""Row f6 without a GPU: the numpy restatement of the depth refiner (oracle/icp_port.py) against point sets the
reference's own `icp_refinement` produced (tests/golden/icp_scenes.npz, oracle/make_golden_icp.py), its ICP on a
rendered scene and on analytic cases, and the argument checks of the gp_icp_* entry points."""
import ctypes as C
import os

import numpy as np
import pytest

from gigapose_b200 import _lib, build
from oracle import icp_port

K = np.array([[500.0, 0, 80.0], [0, 500.0, 60.0], [0, 0, 1]], np.float32)


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def _surface(n=4000, seed=0):
    """Points and unit normals of a bumpy, non-planar surface patch around z = 700 mm."""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-60, 60, (n, 2))
    f = lambda x, y: 700 + 20 * np.sin(x / 15) * np.cos(y / 20) + 0.004 * x * y
    z = f(xy[:, 0], xy[:, 1])
    fx = 20 / 15 * np.cos(xy[:, 0] / 15) * np.cos(xy[:, 1] / 20) + 0.004 * xy[:, 1]
    fy = -20 / 20 * np.sin(xy[:, 0] / 15) * np.sin(xy[:, 1] / 20) + 0.004 * xy[:, 0]
    nrm = np.stack([-fx, -fy, np.ones(n)], 1)
    return np.c_[xy, z], nrm / np.linalg.norm(nrm, axis=1, keepdims=True)


def test_point_to_plane_steps_recover_a_planted_transform():
    """With the true correspondences, the linearised point-to-plane steps and the left-multiplied Rodrigues update
    converge to the planted rigid transform to fp64 rounding."""
    X, N = _surface()
    Rt = icp_port.rodrigues(np.array([0.05, -0.08, 0.03]))
    tt = np.array([12.0, -7.0, 9.0])
    Q, Nq = X @ Rt.T + tt, N @ Rt.T
    dT = np.c_[np.eye(3), np.zeros(3)]
    for _ in range(30):
        S = X @ dT[:, :3].T + dT[:, 3]
        A, b, _ = icp_port.normal_equations(S, Q, Nq, 1000.0)
        xi = icp_port.solve(A, b)
        dT, wn, vn = icp_port.apply_step(dT, xi, 1000.0)
        if wn < 1e-14 and vn < 1e-12:
            break
    assert np.abs(dT[:, :3] - Rt).max() < 1e-12
    assert np.abs(dT[:, 3] - tt).max() < 1e-9


@pytest.mark.parametrize("case", ["mask", "threshold"])
def test_port_reproduces_the_reference_point_sets(golden_dir, case):
    """Stages 2-6 against the reference on hole-free scenes (metres, integer principal point).

    - Target and source counts and sets are exact.
    - Target points are bit-identical.
    - Source points after the centroid shift, and the shifted pose, agree to 1e-6 m. The reference takes float32 means
      (numpy's pairwise float32 sum) and adds the float64 shift into float32 arrays; the port sums in fp64.
    - Target normals agree to 4 float32 ulps of the smoothed depth, carried through get_normal. The reference smooths
      with scipy (fp64 accumulation, one rounding to float32); the port takes a float32 normalised convolution. The two
      smoothed depths S differ by about one ulp. A gradient (S[i+1] - S[i-1]) / 4 then differs by about ulp(S) / 2. A
      normal tilts by that over the tangent length S / f. So the bar is 4 ulp(S) f / (2 S): 7e-5 at 1 m and f = 310.
      The largest difference on these scenes is 1.8e-5, one ulp. This is why a fixed 1e-5 bar cannot hold: the
      gradients cancel float32 depths of about 1 m at a spacing of about 2 mm."""
    g = np.load(os.path.join(golden_dir, "icp_scenes.npz"))
    K, D, R, T0 = g["K"], g[f"{case}_depth"], g[f"{case}_rendered"], g[f"{case}_T0"]
    H, W = D.shape
    mask = g[f"{case}_mask"] if case == "mask" else None
    tmap = icp_port.scene(D, K, unit_per_m=1.0)
    valid, ntgt, src = icp_port.sources_and_targets(tmap, R, (0, 0, W, H), mask, np.float32(1.0))
    assert (ntgt, len(src)) == tuple(g[f"{case}_counts"])
    if case == "threshold":                         # the port's threshold rule equals the reference's compute_masks
        assert np.array_equal(valid, g["threshold_mask"] & (D > 0.2) & (D < 5))
    tgt, want = tmap.reshape(-1, 6)[valid.reshape(-1)], g[f"{case}_tgt"]
    assert np.array_equal(tgt[:, :3], want[:, :3])
    z = want[:, 2]
    bar = 4 * np.spacing(z) * max(K[0, 0], K[1, 1]) / (2 * z)
    assert (np.abs(tgt[:, 3:] - want[:, 3:]).max(1) <= bar).all()
    dbg = {}
    icp_port.refine(tmap, R, (0, 0, W, H), K, T0, mask=mask, debug=dbg, unit_per_m=1.0, num_levels=1, max_iters=1,
                    max_residual=1e9)
    shift = dbg["pose0"][:, 3]
    assert np.abs(icp_port.backproject(src, R, K, W) + shift - g[f"{case}_src"][:, :3]).max() < 1e-6
    assert np.abs(T0[:3, 3] + shift - g[f"{case}_pose_shifted"][:3, 3]).max() < 1e-6
    assert np.array_equal(g[f"{case}_pose_shifted"][:3, :3], T0[:3, :3])


def _bumpy_mesh(n_lat=20, n_lon=40):
    th = np.linspace(0, np.pi, n_lat)[:, None]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)[None]
    bump = 1 + 0.1 * np.sin(3 * th) * np.cos(2 * ph)
    V = np.stack([80 * np.sin(th) * np.cos(ph) * bump, 50 * np.sin(th) * np.sin(ph) * bump,
                  30 * np.cos(th) * bump + 0 * ph], -1).reshape(-1, 3).astype(np.float32)
    F = []
    for i in range(n_lat - 1):
        for j in range(n_lon):
            a, b = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            F += [[a, a + n_lon, b], [b, a + n_lon, b + n_lon]]
    return V, np.array(F, np.int32)


def test_port_icp_recovers_a_planted_transform_on_a_rendered_scene():
    """The whole of icp_port.refine: sets, centroid shift, projective association, median rejection and the level
    schedule.  A bumpy ellipsoid is rendered with oracle/render_port.py at T_true (the measurement, in front of an
    empty background) and at T0, 4 degrees and 6 mm off.  The pose ends within 0.2 mm / 0.1 degrees.  Both clouds are
    pixel samples of the surface, so the two sample grids never coincide and the result is not exact."""
    from oracle import render_port
    V, F = _bumpy_mesh()
    Kr = np.array([[500.0, 0, 80.0], [0, 500.0, 60.0], [0, 0, 1]], np.float32)
    T_true = np.eye(4, dtype=np.float32)
    T_true[:3, :3] = icp_port.rodrigues(np.array([0.3, 0.5, 0.1]))
    T_true[:3, 3] = (5.0, -3.0, 700.0)
    T0 = T_true.copy()
    T0[:3, :3] = (icp_port.rodrigues(np.deg2rad(4.0) * np.array([0.6, 0.0, 0.8])) @ T_true[:3, :3]).astype(np.float32)
    T0[:3, 3] += np.float32([4.0, -3.0, 3.0])
    D = render_port.render(V, F, T_true, Kr, 120, 160, 100.0)["depth"]
    r = render_port.render(V, F, T0, Kr, 120, 160, 100.0)
    out, st, res, fit = icp_port.refine(icp_port.scene(D, Kr), r["depth"], r["box"], Kr, T0, mask=D > 0, min_points=500)
    dR = out[:3, :3].astype(np.float64) @ T_true[:3, :3].T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    assert st == icp_port.OK
    assert np.linalg.norm(out[:3, 3] - T_true[:3, 3]) < 0.2 and ang < 0.1


def test_a_plane_is_degenerate():
    X, N = _surface()
    X[:, 2] = 700.0
    N = np.tile([0.0, 0.0, 1.0], (len(X), 1))
    A, b, _ = icp_port.normal_equations(X, X + [0, 0, 1.0], N, 1000.0)
    assert icp_port.solve(A, b) is None


def _plate_scene(n_pixels):
    """A fronto-parallel plate at 700 mm covering n_pixels pixels (rows of 40) in a 120 x 160 frame, rendered at the
    same pose: every plate pixel is a target and a source."""
    H, W = 120, 160
    D = np.zeros((H, W), np.float32)
    rows, rest = divmod(n_pixels, 40)
    D[30:30 + rows, 60:100] = 700.0
    D[30 + rows, 60:60 + rest] = 700.0
    ys, xs = np.nonzero(D)
    box = (xs.min(), ys.min(), xs.max() + 1, ys.max() + 1)
    return D, box


@pytest.mark.parametrize("n,status", [(999, icp_port.TOO_FEW_POINTS), (1000, icp_port.DEGENERATE)])
def test_too_few_points_at_999_not_at_1000_and_a_flat_plate_is_degenerate(n, status):
    D, box = _plate_scene(n)
    tmap = icp_port.scene(D, K)
    T0 = np.eye(4, dtype=np.float32)
    T0[:3, 3] = (1.0, 2.0, 3.0)
    dbg = {}
    out, st, _, _ = icp_port.refine(tmap, D, box, K, T0, mask=D > 0, debug=dbg)
    assert dbg["counts"] == (n, n)
    assert st == status and np.array_equal(out, T0)


def test_scene_points_are_exact_back_projections_and_normals_face_the_axis():
    D, _ = _plate_scene(1600)
    tmap = icp_port.scene(D, K)
    ys, xs = np.nonzero(D)
    assert np.array_equal(tmap[ys, xs, 2], D[ys, xs])
    assert np.array_equal(tmap[ys, xs, 0], ((xs.astype(np.float32) - K[0, 2]) * D[ys, xs]) / K[0, 0])
    inner = tmap[45:60, 70:90, 3:]
    assert np.abs(inner - [0, 0, 1]).max() < 1e-4
    assert (tmap[D == 0][:, 2] == 0).all()                   # holes and out-of-range depth are not targets


def test_icp_entry_points_reject_bad_arguments_before_touching_a_device(lib):
    ws = C.c_size_t()
    assert lib.gp_icp_query_sizes(1, 1, 480, 640, C.byref(ws)) == 0
    assert ws.value >= 480 * 640 * (36 + 12)
    assert lib.gp_icp_query_sizes(0, 1, 480, 640, C.byref(ws)) == -1 and b"n_frames" in lib.gp_last_error()
    assert lib.gp_icp_query_sizes(1, 1, 8, 640, C.byref(ws)) == -1 and b"image size" in lib.gp_last_error()
    assert lib.gp_icp_query_sizes(1, 1, 480, 640, None) == -1
    assert lib.gp_icp_prepare_scene(1, 480, 640, None, None, 1000.0, None, None) == -1
    assert lib.gp_icp_prepare_scene(1, 480, 640, 8, 8, 0.0, 8, None) == -1 and b"unit_per_m" in lib.gp_last_error()
    p = _lib.GpIcpParams(unit_per_m=1000.0, min_points=1000, num_levels=4, max_iters=100, rejection_scale=2.5,
                         max_residual=0.01, min_step_rad=1e-6, min_step_m=1e-6)
    args = [8] * 6

    def refine(params):
        return lib.gp_icp_refine(1, 1, 480, 640, *args, C.byref(params) if params is not None else None,
                                 8, 8, 8, 8, 8, None)
    assert refine(None) == -1 and b"params" in lib.gp_last_error()
    for field, bad in (("num_levels", 0), ("num_levels", 9), ("max_iters", 0), ("min_points", 0),
                       ("rejection_scale", float("nan")), ("max_residual", -1.0), ("unit_per_m", float("inf"))):
        q = _lib.GpIcpParams.from_buffer_copy(p)
        setattr(q, field, bad)
        assert refine(q) == -1, field
        assert field.encode() in lib.gp_last_error(), field
    assert lib.gp_icp_refine(1, 1, 480, 640, None, None, 8, 8, 8, 8, C.byref(p), 8, 8, 8, 8, 8, None) == -1
    assert b"null" in lib.gp_last_error()
