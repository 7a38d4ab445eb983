"""TEST INFRASTRUCTURE ONLY -- not part of the product path.

Row f12: gp_bop_add's arithmetic restated in numpy (the contract is the comment above add_kernel in
gigapose_b200/csrc/bop_eval.cu): fp32 per-vertex terms with every operation rounded once, the ADD-S min on the squared
terms' bits, one sqrt per point, fp64 sums left to right within each chunk of CHUNK vertices and then over the chunks,
one division by N.  It agrees with the kernel bit for bit (tests/test_gpu_add_eval.py).
"""
import numpy as np

F32 = np.float32
CHUNK = 1024                    # GP_BOP_ADD_CHUNK


def _affine32(A, P):
    A = np.asarray(A, F32).reshape(-1, 4)
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    return np.stack([((A[r, 0] * x + A[r, 1] * y) + A[r, 2] * z) + A[r, 3] for r in range(3)], 1).astype(F32)


def _project32(K, P):
    K = np.asarray(K, F32).reshape(3, 3)
    u = (K[0, 0] * P[:, 0] + K[0, 1] * P[:, 1]) / P[:, 2] + K[0, 2]
    v = (K[1, 1] * P[:, 1]) / P[:, 2] + K[1, 2]
    return u.astype(F32), v.astype(F32)


def _sq3(d):
    return ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)


NAN_BITS = 0x7FFFFFFF            # every NaN term ranks as this one: above +inf, whatever its sign bit


def _nn_sq_bits(g, e, block=2048, device=None):
    """min over the rows of e of the squared distance to each row of g, on the float bits (NaN above +inf).  With a
    torch `device` the same fp32 element-wise operations (each one rounding, no fusion in eager mode) run there, for
    objects too large for numpy's N^2."""
    if device is not None:
        return _nn_sq_bits_torch(g, e, device)
    out = np.full(len(g), 0xFFFFFFFF, np.uint32)
    for i0 in range(0, len(e), block):
        eb = e[i0:i0 + block]
        d = (eb[None, :, :] - g[:, None, :]).astype(F32)                  # e - g, [n_g, block, 3]
        sq = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F32)
        bits = np.where(np.isnan(sq), np.uint32(NAN_BITS), sq.view(np.uint32))
        out = np.minimum(out, bits.min(1))
    return out


def _nn_sq_bits_torch(g, e, device, elems=1 << 28):
    import torch
    G = torch.as_tensor(np.asarray(g, F32), device=device)
    E = torch.as_tensor(np.asarray(e, F32), device=device)
    out = torch.full((len(g),), NAN_BITS + 1, dtype=torch.int64, device=device)  # above every term
    block = max(1, elems // max(len(g), 1))
    for i0 in range(0, len(e), block):
        eb = E[i0:i0 + block]
        dx, dy, dz = (eb[None, :, c] - G[:, None, c] for c in range(3))
        sq = (dx * dx + dy * dy) + dz * dz
        bits = sq.view(torch.int32).to(torch.int64)                 # >= 0 for every non-negative float
        bits = torch.where(torch.isnan(sq), torch.full_like(bits, NAN_BITS), bits)
        out = torch.minimum(out, bits.min(1).values)
    return out.cpu().numpy().astype(np.uint32)


def chunked_mean(dist):
    """The kernel's fp64 mean of per-point fp32 distances: sequential sums per CHUNK, then over the chunks."""
    d = np.asarray(dist, F32).astype(np.float64)
    partial = np.array([np.cumsum(d[c:c + CHUNK])[-1] for c in range(0, len(d), CHUNK)])
    return float(np.cumsum(partial)[-1] / np.float64(len(d)))


def add_terms(vertices, pose_est, pose_gt, K, device=None):
    """Per-vertex fp32 distances (add, adds, proj) [N] each, in the kernel's order (`device`: see _nn_sq_bits)."""
    V = np.asarray(vertices, F32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        e = _affine32(pose_est, V)
        g = _affine32(pose_gt, V)
        ue, ve = _project32(K, e)
        ug, vg = _project32(K, g)
        add = np.sqrt(_sq3((e - g).astype(F32))).astype(F32)
        du, dv = (ue - ug).astype(F32), (ve - vg).astype(F32)
        proj = np.sqrt((du * du + dv * dv).astype(F32)).astype(F32)
        adds = np.sqrt(_nn_sq_bits(g, e, device=device).view(F32)).astype(F32)
    return add, adds, proj


def add_errors(vertices, pose_est, pose_gt, K, device=None):
    """-> (ADD, ADD-S, proj) as the kernel computes them, fp64."""
    with np.errstate(all="ignore"):
        return tuple(chunked_mean(t) for t in add_terms(vertices, pose_est, pose_gt, K, device))


def add_errors_pairs(vertices, vertex_offsets, obj_idx, K, frame_idx, pose_est, pose_gt, device=None):
    """gp_bop_add's output [n, 3] for the same arguments (NaN for an index out of range)."""
    n_obj, n_f = len(vertex_offsets) - 1, len(K)
    out = np.full((len(obj_idx), 3), np.nan)
    for p, (o, f) in enumerate(zip(obj_idx, frame_idx)):
        if 0 <= o < n_obj and 0 <= f < n_f:
            V = np.asarray(vertices, F32)[vertex_offsets[o]:vertex_offsets[o + 1]]
            out[p] = add_errors(V, pose_est[p], pose_gt[p], K[f], device)
    return out
