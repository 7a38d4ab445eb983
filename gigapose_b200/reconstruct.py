"""Row f17: a mesh of an object from its onboarding RGB-D frames, so that model-free runs (row f16) can use the depth
refiners, which render a mesh at each hypothesis.  The frames' depth images are fused into a truncated signed
distance volume in the object frame and its zero surface is extracted by marching tetrahedra on the GPU
(csrc/reconstruct.cu, whose header comment states the contract).  The result is a `render.read_ply`-style dict in the
unit of the poses, which `GigaPose.attach_meshes` takes as it takes a CAD model.

`reconstruct(frames)` chooses the box from the frames themselves (`bounds`), decodes the frames on a thread pool a
chunk ahead of the one being uploaded, keeps them on the device while the box is found, then fuses and extracts."""
from __future__ import annotations

import concurrent.futures
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check

RESOLUTION = 256             # voxels along the longest side of the box
TRUNC_VOXELS = 4             # mu, in voxels
QUANTILE = 1e-3              # order statistics of the back-projected points that bound the box
DECODE_THREADS = 8
CHUNK = 16                   # frames decoded, uploaded and fused together


class ReconstructError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------- box
def object_points(depth, mask, K, pose):
    """The masked pixels with depth > 0 of one frame, back-projected into the object frame, f64 [n,3] on the tensors'
    device: x_c = D K^-1 (u, v, 1) with pixel (u, v) centred at (u, v), then R^T (x_c - t)."""
    depth = torch.as_tensor(depth)
    mask = torch.as_tensor(mask, device=depth.device)
    v, u = torch.nonzero((mask != 0) & (depth > 0), as_tuple=True)
    d = depth[v, u].double()
    Kinv = torch.as_tensor(np.linalg.inv(np.asarray(K, np.float64).reshape(3, 3)), device=depth.device)
    P = torch.as_tensor(np.asarray(pose, np.float64).reshape(4, 4), device=depth.device)
    pix = torch.stack([u.double(), v.double(), torch.ones_like(d)], 1)
    xc = (pix @ Kinv.T) * d[:, None]
    return (xc - P[:3, 3]) @ P[:3, :3]


def order_statistics(points, q=QUANTILE):
    """Per axis, the values of rank floor(q (n - 1)) and ceil((1 - q)(n - 1)) (0-based, ascending) of points [n,3]
    -> (lo f64 [3], hi f64 [3]).  A few stray points (mixed pixels at the mask border) do not move them."""
    n = points.shape[0]
    if n == 0:
        raise ReconstructError("no masked pixel has a depth: nothing to reconstruct")
    k_lo, k_hi = int(np.floor(q * (n - 1))), int(np.ceil((1.0 - q) * (n - 1)))
    lo = torch.kthvalue(points, k_lo + 1, dim=0).values
    hi = torch.kthvalue(points, k_hi + 1, dim=0).values
    return lo.double().cpu().numpy(), hi.double().cpu().numpy()


def grid_box(lo, hi, resolution=RESOLUTION, trunc_voxels=TRUNC_VOXELS):
    """The voxel grid of the box [lo, hi] widened by mu plus one voxel on every side, with `resolution` voxels along
    its longest side: s = (longest side of [lo, hi]) / (resolution - 2 (trunc_voxels + 1)), n_a = ceil(side_a / s) +
    2 (trunc_voxels + 1) -> dict(origin f32 [3], voxel f32, dims (nx, ny, nz), trunc f32 = trunc_voxels s)."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    pad = int(trunc_voxels) + 1
    inner = int(resolution) - 2 * pad
    if inner < 1:
        raise ReconstructError(f"resolution {resolution} leaves no voxel inside the {pad}-voxel margins")
    side = hi - lo
    if not np.all(np.isfinite(side)) or not side.max() > 0:
        raise ReconstructError(f"degenerate box {lo.tolist()} .. {hi.tolist()}")
    s = float(np.float32(side.max() / inner))
    # s is rounded to f32: a side may come out a few 1e-5 voxels over a whole count, which the margin absorbs
    dims = [max(1, int(np.ceil(side[a] / s - 1e-3))) + 2 * pad for a in range(3)]
    origin = (lo - pad * s).astype(np.float32)
    return dict(origin=origin, voxel=np.float32(s), dims=tuple(dims), trunc=np.float32(trunc_voxels * s))


def check_bounds(bounds):
    b = np.asarray(bounds, np.float64)
    if b.shape != (2, 3) or not np.all(np.isfinite(b)) or not np.all(b[1] > b[0]):
        raise ReconstructError(f"bounds must be [[x0, y0, z0], [x1, y1, z1]] with x1 > x0 etc., got {b.tolist()}")
    return b[0], b[1]


# ---------------------------------------------------------------------------------------------------- GPU launches
def _device_of(t, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise _lib.GigaPoseNativeError(f"{what} must be a CUDA tensor (no CPU fallback)")
    return t.device


def new_grid(dims, device):
    """A zeroed (tsdf, weight) grid f32 [nz,ny,nx,2] for `fuse`."""
    nx, ny, nz = (int(v) for v in dims)
    if min(nx, ny, nz) < 1 or nx * ny * nz > _lib.TSDF_MAX_VOXELS:
        raise ReconstructError(f"grid {nx} x {ny} x {nz} outside 1 .. {_lib.TSDF_MAX_VOXELS} voxels")
    return torch.zeros(nz, ny, nx, 2, device=device)


@torch.no_grad()
def fuse(grid, depth, mask, K, poses, origin, voxel, trunc):
    """gp_tsdf_fuse: frames depth f32 [n,H,W] (unit of the poses, 0 = missing) and mask u8 [n,H,W] on the grid's
    device, K [n,3,3] and poses [n,4,4] object -> camera on the host, into grid f32 [nz,ny,nx,2] in place."""
    dev = _device_of(grid, "grid")
    if grid.dtype != torch.float32 or grid.dim() != 4 or grid.shape[3] != 2 or not grid.is_contiguous():
        raise ValueError(f"grid must be a contiguous f32 [nz,ny,nx,2], got {grid.dtype} {tuple(grid.shape)}")
    if depth.dim() != 3 or depth.dtype != torch.float32:
        raise ValueError(f"depth must be f32 [n,H,W], got {depth.dtype} {tuple(depth.shape)}")
    n, H, W = depth.shape
    if tuple(mask.shape) != (n, H, W) or mask.dtype != torch.uint8:
        raise ValueError(f"mask must be u8 [{n},{H},{W}], got {mask.dtype} {tuple(mask.shape)}")
    Kf = np.ascontiguousarray(np.asarray(K, np.float32).reshape(n, 3, 3))
    Pf = np.ascontiguousarray(np.asarray(poses, np.float32).reshape(n, 4, 4))
    o = np.ascontiguousarray(np.asarray(origin, np.float32).reshape(3))
    nz, ny, nx, _ = grid.shape
    depth, mask = depth.to(dev).contiguous(), mask.to(dev).contiguous()
    fp = C.POINTER(C.c_float)
    with torch.cuda.device(dev):
        check(_lib.load().gp_tsdf_fuse(nx, ny, nz, o.ctypes.data_as(fp), float(voxel), float(trunc), n, H, W,
                                       depth.data_ptr(), mask.data_ptr(), Kf.ctypes.data_as(fp), Pf.ctypes.data_as(fp),
                                       grid.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return grid


@torch.no_grad()
def extract(grid, origin, voxel):
    """gp_tsdf_extract_count / _emit on grid f32 [nz,ny,nx,2] -> (vertices f32 [V,3], faces i32 [F,3]) on its
    device, the zero surface of the tsdf in the object frame."""
    dev = _device_of(grid, "grid")
    if grid.dtype != torch.float32 or grid.dim() != 4 or grid.shape[3] != 2 or not grid.is_contiguous():
        raise ValueError(f"grid must be a contiguous f32 [nz,ny,nx,2], got {grid.dtype} {tuple(grid.shape)}")
    nz, ny, nx, _ = grid.shape
    lib = _lib.load()
    ws = C.c_size_t()
    check(lib.gp_tsdf_extract_query_sizes(nx, ny, nz, C.byref(ws)))
    o = np.ascontiguousarray(np.asarray(origin, np.float32).reshape(3))
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _, workspace = _lib.aligned_buffer(ws.value, dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        check(lib.gp_tsdf_extract_count(nx, ny, nz, grid.data_ptr(), workspace.data_ptr(), counts.data_ptr(), stream))
        V, F = (int(v) for v in counts.tolist())
        vertices = torch.empty(V, 3, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
        if V and F:
            check(lib.gp_tsdf_extract_emit(nx, ny, nz, o.ctypes.data_as(C.POINTER(C.c_float)), float(voxel),
                                           grid.data_ptr(), workspace.data_ptr(), vertices.data_ptr(), faces.data_ptr(),
                                           stream))
    return vertices, faces


# ---------------------------------------------------------------------------------------------------- frames
def _load(frames, i):
    d = frames.load_depth(i)
    m = frames.mask(i)
    if d.shape != m.shape:
        raise ReconstructError(f"frame {i}: depth {d.shape} and mask {m.shape} differ in size")
    return d, m


def _chunks(frames, device, pool):
    """Yields (frame ids, depth f32 [c,H,W], mask u8 [c,H,W]) on the device, CHUNK frames at a time, the next chunk
    decoding on `pool` while the current one is used."""
    n = len(frames)
    submit = lambda c0: [pool.submit(_load, frames, i) for i in range(c0, min(n, c0 + CHUNK))]
    pending = submit(0)
    for c0 in range(0, n, CHUNK):
        loaded = [f.result() for f in pending]
        pending = submit(c0 + CHUNK) if c0 + CHUNK < n else []
        shapes = {d.shape for d, _ in loaded}
        if len(shapes) != 1:
            raise ReconstructError(f"frames {c0} .. {c0 + len(loaded) - 1} have different sizes {sorted(shapes)}")
        depth = torch.from_numpy(np.stack([d for d, _ in loaded])).pin_memory().to(device, non_blocking=True)
        mask = torch.from_numpy(np.stack([m for _, m in loaded])).pin_memory().to(device, non_blocking=True)
        yield list(range(c0, c0 + len(loaded))), depth, mask


@torch.no_grad()
def reconstruct(frames, resolution=RESOLUTION, trunc_voxels=TRUNC_VOXELS, bounds=None, device=None):
    """The mesh of one object from its onboarding frames (`onboarding.Frames` with depths): a `read_ply`-style dict
    (vertices f32 [V,3], faces i32 [F,3] on the host, in the unit of the poses, no colour or texture).

    The box is `bounds` ([[x0, y0, z0], [x1, y1, z1]] in the object frame) or, by default, the order statistics at
    1e-3 and 1 - 1e-3 of the masked depth pixels back-projected into the object frame (`order_statistics`); either is
    widened by mu plus one voxel (`grid_box`), with `resolution` voxels along its longest side and mu = trunc_voxels
    voxels."""
    if getattr(frames, "depths", None) is None:
        raise ReconstructError("the frames carry no depth images: reconstruction fuses the onboarding depth "
                               "(read_onboarding_static(..., depth=True))")
    if int(resolution) < 2 * (int(trunc_voxels) + 1) + 1 or int(trunc_voxels) < 1:
        raise ReconstructError(f"resolution {resolution} and trunc_voxels {trunc_voxels}: need trunc_voxels >= 1 and "
                               f"resolution > 2 (trunc_voxels + 1)")
    if bounds is not None:
        bounds = check_bounds(bounds)
    device = _lib.cuda_device(device if device is not None else "cuda", "reconstruct runs")
    pool = concurrent.futures.ThreadPoolExecutor(DECODE_THREADS)
    try:
        kept, points = [], []
        for ids, depth, mask in _chunks(frames, device, pool):
            kept.append((ids, depth, mask))
            if bounds is None:
                points += [object_points(depth[j], mask[j], frames.K[i], frames.poses[i]) for j, i in enumerate(ids)]
    finally:
        pool.shutdown(wait=True)
    lo, hi = bounds if bounds is not None else order_statistics(torch.cat(points))
    del points
    box = grid_box(lo, hi, resolution, trunc_voxels)
    grid = new_grid(box["dims"], device)
    for ids, depth, mask in kept:
        fuse(grid, depth, mask, frames.K[ids], frames.poses[ids], box["origin"], box["voxel"], box["trunc"])
    del kept
    vertices, faces = extract(grid, box["origin"], box["voxel"])
    if faces.shape[0] == 0:
        raise ReconstructError(f"the fused grid {box['dims']} has no surface: no frame saw the object inside the box")
    return dict(vertices=vertices.cpu().numpy(), faces=faces.cpu().numpy(), vertex_color=None, face_uv=None,
                texture=None)
