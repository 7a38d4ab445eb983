"""Row f17 without a GPU: the onboarding_static reader with depth and its refusals, the --reconstruct option checks,
write_ply / read_ply, the box from order statistics against numpy.partition (a planted outlier does not move it), the
fp64 evaluator's marching tetrahedra on an analytic sphere, and the argument checks of every new entry point."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import reconstruct_fp64 as ref
from gigapose_b200 import _lib, bop_run, build, onboarding, reconstruct, render
from gigapose_b200.onboarding import OnboardingError
from rgbd_static_tree import look_at_pose, write_scene

K = np.array([[50.0, 0.5, 16.0], [0.0, 52.0, 12.0], [0.0, 0.0, 1.0]])


def _frames(rng, n=3, H=24, W=32):
    out = []
    for k in range(n):
        P = look_at_pose(rng.normal(size=3), 300.0)
        mask = np.zeros((H, W), np.uint8)
        mask[8:16, 10:20] = 1
        depth = np.where(mask, 300 + k, 0).astype(np.uint16)
        out.append((rng.integers(0, 256, (H, W, 3)), mask, depth, P, K))
    return out


def test_reader_with_and_without_depth(tmp_path):
    rng = np.random.default_rng(1)
    ds = str(tmp_path)
    fr = _frames(rng)
    write_scene(ds, "obj_000001_up", 1, fr, depth_scale=0.1)
    write_scene(ds, "obj_000001_down", 1, _frames(rng, 2), depth_scale=0.1)
    plain = onboarding.read_onboarding_static(ds)[1]
    assert plain.depths is None and len(plain) == 5
    with pytest.raises(OnboardingError, match="no depth"):
        plain.load_depth(0)
    with_depth = onboarding.read_onboarding_static(ds, depth=True)[1]
    assert with_depth.images == plain.images and with_depth.masks == plain.masks
    assert np.array_equal(with_depth.K, plain.K) and np.array_equal(with_depth.poses, plain.poses)
    assert len(with_depth.depths) == 5 and with_depth.depths[0].endswith(os.path.join("depth", "000000.png"))
    d = with_depth.load_depth(3)                 # down scene, image 0: the down scenes come first
    assert d.dtype == np.float32
    want = (fr[0][2].astype(np.float64) * 0.1).astype(np.float32)
    assert np.array_equal(with_depth.load_depth(2 + 0), want)
    assert with_depth.depth_scale.tolist() == [0.1] * 5


def test_reader_refusals_name_the_depth_file_or_scale(tmp_path):
    rng = np.random.default_rng(2)
    ds = str(tmp_path / "a")
    d = write_scene(ds, "obj_000001_up", 1, _frames(rng), skip_depth=(1,))
    onboarding.read_onboarding_static(ds)                   # the default call does not look for depth
    with pytest.raises(OnboardingError, match=os.path.join(d, "depth", "000001.png").replace("\\", "\\\\")):
        onboarding.read_onboarding_static(ds, depth=True)
    ds = str(tmp_path / "b")
    d = write_scene(ds, "obj_000001_up", 1, _frames(rng), skip_scale=(2,))
    with pytest.raises(OnboardingError, match="scene_camera.json: image 2 has no depth_scale"):
        onboarding.read_onboarding_static(ds, depth=True)


def test_frames_depth_arguments():
    with pytest.raises(OnboardingError, match="depth images"):
        onboarding.Frames([0, 1], [0, 1], np.eye(3)[None].repeat(2, 0), np.eye(4)[None].repeat(2, 0), depths=[0])
    with pytest.raises(OnboardingError, match="depth_scale"):
        onboarding.Frames([0], [0], np.eye(3), np.eye(4), depths=[0], depth_scale=0.0)
    f = onboarding.Frames([0], [0], np.eye(3), np.eye(4), depths=[np.array([[1000, 0]], np.uint16)], depth_scale=0.25)
    assert f.load_depth(0).tolist() == [[250.0, 0.0]]


def test_reconstruct_options(capsys):
    base = ["--dataset-dir", "x", "--checkpoint", "y"]
    cases = [(["--reconstruct", "--refine-depth", "1"], bop_run.RECONSTRUCT_NEEDS_STATIC),
             (["--onboarding", "static", "--reconstruct"], bop_run.RECONSTRUCT_NEEDS_DEPTH),
             (["--onboarding", "static", "--refine-depth", "1"], bop_run.STATIC_NO_DEPTH)]
    for extra, msg in cases:
        with pytest.raises(SystemExit) as e:
            bop_run.main(base + extra)
        assert e.value.code == 2
        assert msg in capsys.readouterr().err
    # today's refusal, byte for byte
    assert bop_run.STATIC_NO_DEPTH == ("--onboarding static takes no --refine-depth: the depth refiners render the "
                                       "CAD model, which model-free onboarding does not read")
    for args, msg in ((("models", 1, True), bop_run.RECONSTRUCT_NEEDS_STATIC), (("static", 0, True),
                      bop_run.RECONSTRUCT_NEEDS_DEPTH), (("static", 2, False), bop_run.STATIC_NO_DEPTH)):
        with pytest.raises(bop_run.BopRunError) as e:
            bop_run.check_onboarding(*args)
        assert str(e.value) == msg
    bop_run.check_onboarding("static", 2, True)
    bop_run.check_onboarding("models", 2)
    assert bop_run.parser().parse_args(base).reconstruct is False


def test_write_ply_round_trips_bit_for_bit(tmp_path):
    rng = np.random.default_rng(3)
    V = rng.normal(size=(500, 3)).astype(np.float32) * np.float32(137.0)
    V[0] = [np.float32(1e-38), -0.0, np.float32(3.4e38)]
    F = rng.integers(0, 500, (900, 3)).astype(np.int32)
    path = str(tmp_path / "m.ply")
    render.write_ply(path, dict(vertices=V, faces=F))
    back = render.read_ply(path)
    assert back["vertices"].tobytes() == V.tobytes() and back["faces"].dtype == np.int32
    assert np.array_equal(back["faces"], F)
    render.write_ply(path, dict(vertices=np.zeros((0, 3), np.float32), faces=np.zeros((0, 3), np.int32)))
    assert render.read_ply(path)["vertices"].shape == (0, 3)
    with pytest.raises(render.PlyError, match="face indices"):
        render.write_ply(path, dict(vertices=V[:3], faces=[[0, 1, 3]]))


def test_bounds_are_order_statistics_and_ignore_a_planted_outlier():
    rng = np.random.default_rng(4)
    H, W = 200, 300
    Kf = np.array([[400.0, 1.5, 150.2], [0.0, 410.0, 99.7], [0.0, 0.0, 1.0]])
    P = look_at_pose([0.3, -0.5, 0.8], 500.0)
    mask = np.zeros((H, W), np.uint8)
    mask[40:160, 50:250] = 1                          # 24 000 pixels: q n = 24
    depth = (500.0 + rng.uniform(-40, 40, (H, W))).astype(np.float32)
    depth[60, 70] = 0.0                               # missing: not a point
    clean = depth.copy()
    clean[60, 70] = 0.0
    rows, cols = rng.integers(40, 160, 10), rng.integers(50, 250, 10)
    depth[rows, cols] = 1000.0                        # mixed pixels at the mask border, at 1 m
    clean[rows, cols] = 0.0
    pts = reconstruct.object_points(torch.as_tensor(depth), torch.as_tensor(mask), Kf, P).numpy()
    # against numpy in fp64
    v, u = np.nonzero((mask != 0) & (depth > 0))
    xc = (np.stack([u, v, np.ones_like(u)], 1).astype(np.float64) @ np.linalg.inv(Kf).T) * depth[v, u, None]
    want = (xc - P[:3, 3]) @ P[:3, :3]
    assert len(pts) == 120 * 200 - 1 and np.abs(pts - want).max() < 1e-9
    lo, hi = reconstruct.order_statistics(torch.as_tensor(pts))
    n = len(pts)
    k_lo, k_hi = int(np.floor(1e-3 * (n - 1))), int(np.ceil((1 - 1e-3) * (n - 1)))
    assert k_lo == 23 and k_hi == n - 1 - 23
    for a in range(3):
        assert lo[a] == np.partition(pts[:, a], k_lo)[k_lo] and hi[a] == np.partition(pts[:, a], k_hi)[k_hi]
    # the outliers lie ~500 mm beyond the object; the box stays within the clean points' extent, while q = 0 reaches them
    c = reconstruct.object_points(torch.as_tensor(clean), torch.as_tensor(mask), Kf, P).numpy()
    assert np.all(lo >= c.min(0)) and np.all(hi <= c.max(0))
    assert np.all(hi - lo > 0.9 * (c.max(0) - c.min(0)))
    lo0, hi0 = reconstruct.order_statistics(torch.as_tensor(pts), q=0.0)
    assert np.max((hi0 - lo0) - (c.max(0) - c.min(0))) > 300
    box = reconstruct.grid_box(lo, hi, resolution=64, trunc_voxels=4)
    s = float(box["voxel"])
    assert max(box["dims"]) == 64 and np.all(box["origin"] <= lo - 5 * s + 1e-3)
    top = box["origin"].astype(np.float64) + np.array(box["dims"]) * s
    assert np.all(top >= hi + 5 * s - 1e-3) and float(box["trunc"]) == np.float32(4 * s)


def _sphere_grid(n, r, s):
    o = -n * s / 2
    c = ref.centres((n, n, n), (o, o, o), s)
    d = np.linalg.norm(c, axis=-1) - r
    grid = np.stack([np.clip(d / (4 * s), -1, 1), np.ones_like(d)], -1).astype(np.float32)
    return grid, np.float32(o), s


def test_evaluator_extraction_of_an_analytic_sphere():
    for n, r, s in ((24, 7.3, 1.0), (40, 13.1, 0.75)):
        grid, o, s = _sphere_grid(n, r, s)
        mesh = ref.extract(grid, (o, o, o), s)
        topo = ref.topology(mesh["faces"], len(mesh["vertices"]))
        assert topo == dict(manifold=True, oriented=True, euler=2), topo
        assert ref.signed_volume(mesh["vertices"], mesh["faces"]) > 0
        assert len(np.unique(mesh["faces"])) == len(mesh["vertices"])        # no unreferenced vertex
        dist = np.abs(np.linalg.norm(mesh["vertices"], axis=1) - r)
        # linear interpolation of a sphere's distance along an edge of length <= sqrt(3) s: error <= 3 s^2 / (2 r)
        assert dist.max() <= 1.5 * s * s / r * 2, (dist.max(), s * s / r)
        vol = 4 / 3 * np.pi * r ** 3
        assert abs(ref.signed_volume(mesh["vertices"], mesh["faces"]) - vol) < 0.02 * vol


def test_evaluator_blocks_weight_zero_corners_and_truncation_steps():
    grid = np.zeros((2, 2, 2, 2), np.float32)
    grid[..., 1] = 1
    grid[..., 0] = 0.5
    grid[0, 0, 0, 0] = -0.5
    assert len(ref.extract(grid, (0, 0, 0), 1.0)["faces"]) == 6         # the corner is in every tetrahedron
    g = grid.copy()
    g[1, 1, 1, 1] = 0                                                    # weight 0 on the shared diagonal corner
    assert len(ref.extract(g, (0, 0, 0), 1.0)["faces"]) == 0
    g = grid.copy()
    g[0, 0, 0, 0], g[0, 0, 1, 0] = -1, 1                                 # a +1 / -1 edge of tetrahedra 0 and 1
    assert len(ref.extract(g, (0, 0, 0), 1.0)["faces"]) == 4


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_arguments_without_a_gpu(lib):
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first
    fp = C.POINTER(C.c_float)
    o = (C.c_float * 3)(0, 0, 0)
    Kok = (C.c_float * 9)(500, 0, 320, 0, 500, 240, 0, 0, 1)
    Kbad = (C.c_float * 9)(500, 0, 320, 0, 500, 240, 0, 0, 2)
    P = (C.c_float * 16)(1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 500, 0, 0, 0, 1)
    Pnan = (C.c_float * 16)(float("nan"), 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 500, 0, 0, 0, 1)
    o_nan = (C.c_float * 3)(0, float("inf"), 0)

    def fuse(nx=8, ny=8, nz=8, origin=o, voxel=1.0, trunc=4.0, n=1, H=48, W=64, K=Kok, pose=P, grid=fake, depth=fake):
        rc = lib.gp_tsdf_fuse(nx, ny, nz, C.cast(origin, fp) if origin is not None else None, voxel, trunc, n, H, W,
                              depth, fake, C.cast(K, fp), C.cast(pose, fp), grid, None)
        return rc, lib.gp_last_error()

    for kw, word in ((dict(nx=0), b"side"), (dict(nx=1 << 10, ny=1 << 10, nz=1 << 8), b"GP_TSDF_MAX_VOXELS"),
                     (dict(origin=None), b"origin"), (dict(origin=o_nan), b"origin[1]"), (dict(voxel=0.0), b"voxel"),
                     (dict(voxel=float("nan")), b"voxel"), (dict(trunc=-1.0), b"truncation"), (dict(n=-1), b"frame"),
                     (dict(H=0), b"frame"), (dict(K=Kbad), b"K must"), (dict(pose=Pnan), b"pose"),
                     (dict(grid=None), b"grid"), (dict(depth=None), b"null")):
        rc, msg = fuse(**kw)
        assert rc == -1 and word in msg, (kw, rc, msg)
    assert fuse(n=0)[0] == 0                          # nothing to do: no device touched
    ws = C.c_size_t()
    assert lib.gp_tsdf_extract_query_sizes(1, 8, 8, C.byref(ws)) == -1 and b"at least 2" in lib.gp_last_error()
    assert lib.gp_tsdf_extract_query_sizes(8, 8, 8, None) == -1
    assert lib.gp_tsdf_extract_query_sizes(64, 48, 32, C.byref(ws)) == 0
    assert ws.value >= 64 * 48 * 32 * 12
    assert lib.gp_tsdf_extract_count(8, 8, 8, None, fake, fake, None) == -1 and b"null" in lib.gp_last_error()
    assert lib.gp_tsdf_extract_count(8, 1, 8, fake, fake, fake, None) == -1
    assert lib.gp_tsdf_extract_emit(8, 8, 8, C.cast(o, fp), 1.0, fake, fake, None, fake, None) == -1
    assert lib.gp_tsdf_extract_emit(8, 8, 8, C.cast(o, fp), -1.0, fake, fake, fake, fake, None) == -1
    assert b"voxel" in lib.gp_last_error()


def test_python_entry_points_reject_bad_arguments_without_a_gpu():
    nodepth = onboarding.Frames([0], [0], np.eye(3), np.eye(4))
    with pytest.raises(reconstruct.ReconstructError, match="no depth"):
        reconstruct.reconstruct(nodepth)
    f = onboarding.Frames([0], [0], np.eye(3), np.eye(4), depths=[np.zeros((2, 2))])
    with pytest.raises(reconstruct.ReconstructError, match="resolution"):
        reconstruct.reconstruct(f, resolution=10, trunc_voxels=4)
    with pytest.raises(reconstruct.ReconstructError, match="trunc_voxels"):
        reconstruct.reconstruct(f, trunc_voxels=0)
    with pytest.raises(reconstruct.ReconstructError, match="bounds"):
        reconstruct.reconstruct(f, bounds=[[0, 0, 0], [1, -1, 1]])
    with pytest.raises(reconstruct.ReconstructError, match="no masked pixel"):
        reconstruct.order_statistics(torch.zeros(0, 3))
    with pytest.raises(reconstruct.ReconstructError, match="degenerate"):
        reconstruct.grid_box([0, 0, 0], [0, 0, 0])
    with pytest.raises(reconstruct.ReconstructError, match="voxels"):
        reconstruct.new_grid((1024, 1024, 1024), "cpu")
    with pytest.raises(_lib.GigaPoseNativeError):
        reconstruct.fuse(torch.zeros(2, 2, 2, 2), torch.zeros(1, 2, 2), torch.zeros(1, 2, 2, dtype=torch.uint8),
                         np.eye(3), np.eye(4), (0, 0, 0), 1.0, 4.0)
    with pytest.raises(_lib.GigaPoseNativeError):
        reconstruct.extract(torch.zeros(2, 2, 2, 2), (0, 0, 0), 1.0)
