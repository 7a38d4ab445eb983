"""CPU restatement of the template renderer (gigapose_b200/csrc/render.cu) in numpy float32: the same 1/256 px snapping,
64-bit integer edge functions with the top-left rule, per-sample depth formula and operation order, depth keys and
resolve.  Every float32 operation below rounds once, as the kernel's __fmul_rn / __fadd_rn / __fdiv_rn / __frcp_rn do,
so the outputs are meant to be bit-identical.  Test infrastructure, like oracle/port.py."""
from __future__ import annotations

import numpy as np

F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
SAMPLE_DX = np.array([-32, 96, -96, 32], dtype=np.int64)        # 1/256 px
SAMPLE_DY = np.array([-96, -32, 32, 96], dtype=np.int64)
GUARD_PX = F32(4194304.0)


def _setup(vertices, faces, pose, K, z_near):
    """Per face: snapped x, y [F,3] (int64), 1/z [F,3], corner order [F,3], doubled area [F], valid [F]."""
    V = np.asarray(vertices, F32)
    P = np.asarray(pose, F32).reshape(4, 4)
    K = np.asarray(K, F32).reshape(3, 3)
    X, Y, Z = V[:, 0], V[:, 1], V[:, 2]
    cam = [((P[r, 0] * X + P[r, 1] * Y) + P[r, 2] * Z) + P[r, 3] for r in range(3)]
    x, y, z = cam
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = (K[0, 0] * x + K[0, 1] * y) / z + K[0, 2]
        v = (K[1, 1] * y) / z + K[1, 2]
        iz = F32(1) / z
        ok_v = (z > F32(z_near)) & (np.abs(u) < GUARD_PX) & (np.abs(v) < GUARD_PX)
        sx = np.where(ok_v, np.rint(u * F32(256)), 0).astype(np.int64)
        sy = np.where(ok_v, np.rint(v * F32(256)), 0).astype(np.int64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    inb = (f >= 0) & (f < len(V))
    fi = np.where(inb, f, 0)
    valid = inb.all(1) & ok_v[fi].all(1)
    fx, fy, fz = sx[fi], sy[fi], iz[fi]
    area = (fx[:, 1] - fx[:, 0]) * (fy[:, 2] - fy[:, 0]) - (fy[:, 1] - fy[:, 0]) * (fx[:, 2] - fx[:, 0])
    corner = np.tile(np.arange(3), (len(f), 1))
    flip = area < 0
    for a in (fx, fy, fz, corner):
        a[flip, 1], a[flip, 2] = a[flip, 2].copy(), a[flip, 1].copy()
    area = np.abs(area)
    valid &= area != 0
    # rotate to start at the smallest (y, x)
    r = np.argmin((fy << 32) + (fx + (1 << 31)), axis=1)
    rot = (np.arange(3)[None] + r[:, None]) % 3
    fx, fy, fz, corner = [np.take_along_axis(a, rot, 1) for a in (fx, fy, fz, corner)]
    return dict(x=fx, y=fy, iz=fz, corner=corner, area=area, valid=valid)


def _edge(ax, ay, bx, by, px, py):
    """Edge value, or -1 where the sample is outside (top-left rule on the edge itself)."""
    dx, dy = bx - ax, by - ay
    e = dx * (py - ay) - dy * (px - ax)
    top_left = (dy < 0) | ((dy == 0) & (dx > 0))
    return np.where((e > 0) | ((e == 0) & top_left), e, -1)


def _weights(t, f, sx, sy):
    """lambda_i / z_i [n,3] of samples (sx, sy) against faces f, and the inside mask."""
    x, y = t["x"][f], t["y"][f]
    w0 = _edge(x[:, 1], y[:, 1], x[:, 2], y[:, 2], sx, sy)
    w1 = _edge(x[:, 2], y[:, 2], x[:, 0], y[:, 0], sx, sy)
    w2 = _edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], sx, sy)
    inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
    a = t["area"][f].astype(F32)
    iz = t["iz"][f]
    b = np.stack([(w.astype(F32) / a) * iz[:, i] for i, w in enumerate((w0, w1, w2))], 1)
    return b, inside


def _depth(b):
    return F32(1) / ((b[:, 0] + b[:, 1]) + b[:, 2])


def rasterize(vertices, faces, pose, K, H, W, z_near):
    """Key buffer uint64 [H,W,4]: min over covering faces of (float bits of z) << 32 | face id."""
    t = _setup(vertices, faces, pose, K, z_near)
    keys = np.full(H * W * 4, EMPTY, dtype=np.uint64)
    fid = np.nonzero(t["valid"])[0]
    if not len(fid):
        return keys.reshape(H, W, 4), t
    x, y = t["x"][fid], t["y"][fid]
    px0 = np.maximum(-((96 - x.min(1)) >> 8), 0)
    px1 = np.minimum((x.max(1) + 96) >> 8, W - 1)
    py0 = np.maximum(-((96 - y.min(1)) >> 8), 0)
    py1 = np.minimum((y.max(1) + 96) >> 8, H - 1)
    bw, bh = px1 - px0 + 1, py1 - py0 + 1
    keep = (bw > 0) & (bh > 0)
    fid, px0, py0, bw, bh = fid[keep], px0[keep], py0[keep], bw[keep], bh[keep]
    n = bw * bh
    # every (face, pixel of its bounding box) pair, processed in slices to bound memory
    starts = np.concatenate([[0], np.cumsum(n)])
    step = 1 << 22
    for lo in range(0, int(starts[-1]), step):
        idx = np.arange(lo, min(lo + step, int(starts[-1])))
        k = np.searchsorted(starts, idx, side="right") - 1
        p = idx - starts[k]
        px, py = px0[k] + p % bw[k], py0[k] + p // bw[k]
        f = fid[k]
        for s in range(4):
            b, inside = _weights(t, f, px * 256 + SAMPLE_DX[s], py * 256 + SAMPLE_DY[s])
            z = _depth(b[inside])
            key = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | f[inside].astype(np.uint64)
            np.minimum.at(keys, ((py[inside] * W + px[inside]) * 4 + s), key)
    return keys.reshape(H, W, 4), t


def _sample_texture(tex, u, v):
    th, tw = tex.shape[:2]
    fx = u * F32(tw) - F32(0.5)
    fy = v * F32(th) - F32(0.5)
    fx = np.where(np.isfinite(fx), fx, F32(0))
    fy = np.where(np.isfinite(fy), fy, F32(0))
    x0, y0 = np.floor(fx), np.floor(fy)
    ax, ay = fx - x0, fy - y0

    def wrap(i, n):
        m = np.fmod(i, F32(n))
        m = np.where(m < 0, m + F32(n), m).astype(np.int64)
        return np.where(m >= n, 0, m)

    c0 = wrap(x0, tw)
    c1 = np.where(c0 + 1 == tw, 0, c0 + 1)
    b0 = wrap(y0, th)
    b1 = np.where(b0 + 1 == th, 0, b0 + 1)
    r0, r1 = th - 1 - b0, th - 1 - b1

    def lerp(a, b, w):
        return (F32(1) - w)[:, None] * a + w[:, None] * b

    lo = lerp(tex[r0, c0], tex[r0, c1], ax)
    hi = lerp(tex[r1, c0], tex[r1, c1], ax)
    return lerp(lo, hi, ay)


def _interp(b, z, a):
    """a [n,3 corners] -> [n]"""
    return ((b[:, 0] * a[:, 0] + b[:, 1] * a[:, 1]) + b[:, 2] * a[:, 2]) * z


def render(vertices, faces, pose, K, H, W, z_near, vertex_color=None, face_uv=None, texture=None, constant_color=None):
    """One view -> dict(rgba [4,H,W], depth [H,W], box [4], keys [H,W,4]), all numpy."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    keys, t = rasterize(vertices, faces, pose, K, H, W, z_near)
    flat = keys.reshape(-1, 4)
    covered = flat != EMPTY
    summ = np.zeros((H * W, 3), F32)
    zmin = np.full(H * W, np.inf, F32)
    pix = np.arange(H * W)
    ccol = np.ones(3, F32) if constant_color is None else np.asarray(constant_color, F32)
    for s in range(4):
        m = covered[:, s]
        p, key = pix[m], flat[m, s]
        f = (key & np.uint64(0xFFFFFFFF)).astype(np.int64)
        zs = (key >> np.uint64(32)).astype(np.uint32).view(F32)
        zmin[p] = np.minimum(zmin[p], zs)
        b, _ = _weights(t, f, (p % W) * 256 + SAMPLE_DX[s], (p // W) * 256 + SAMPLE_DY[s])
        z = _depth(b)
        corner = t["corner"][f]
        if texture is not None:
            uv = np.asarray(face_uv, F32).reshape(-1, 3, 2)[f[:, None], corner]       # [n,3,2]
            c = _sample_texture(np.asarray(texture, F32), _interp(b, z, uv[..., 0]), _interp(b, z, uv[..., 1]))
        elif vertex_color is not None:
            col = np.asarray(vertex_color, F32)[faces[f[:, None], corner]]              # [n,3 corners,3]
            c = np.stack([_interp(b, z, col[..., ch]) for ch in range(3)], 1)
        else:
            c = np.broadcast_to(ccol, (len(p), 3))
        summ[p] = summ[p] + c
    q = np.clip(np.rint((summ * F32(0.25)) * F32(255)), 0, 255).astype(F32)
    rgb = (q / F32(255)).T.reshape(3, H, W)
    alpha = covered.any(1).astype(F32).reshape(1, H, W)
    depth = np.where(covered.any(1), zmin, F32(0)).reshape(H, W)
    ys, xs = np.nonzero(alpha[0])
    box = np.array([xs.min(), ys.min(), xs.max() + 1, ys.max() + 1] if len(xs) else [0, 0, W, H], np.int64)
    return dict(rgba=np.concatenate([rgb, alpha]), depth=depth, box=box, keys=keys)
