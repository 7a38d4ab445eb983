"""CPU restatement of the depth refiner (gigapose_b200/csrc/depth_icp.cu, row f6) in numpy: float32 where the kernel
computes in float32, with the same operation order, and fp64 for the centroids and the normal equations.  The
integer decisions (target and source sets, associations, rejections) follow the header comment of the .cu exactly;
the fp64 sums are taken in numpy's order, so poses agree with the kernel to fp64 rounding of those sums.  Test
infrastructure, like oracle/port.py."""
from __future__ import annotations

import numpy as np

F32 = np.float32
RADIUS = 8
OK, TOO_FEW_POINTS, DEGENERATE, RESIDUAL, LOST = 0, 1, 2, 3, 5
DEFAULTS = dict(unit_per_m=1000.0, min_points=1000, num_levels=4, max_iters=100, rejection_scale=2.5,
                max_residual=0.01, min_step_rad=1e-6, min_step_m=1e-6)


def gauss_weights():
    """scipy.ndimage's _gaussian_kernel1d(sigma=2, order=0, radius=8), rounded once to float32."""
    x = np.arange(-RADIUS, RADIUS + 1, dtype=np.float64)
    e = np.exp(-0.5 * x * x / 4.0)
    return (e / e.sum()).astype(F32)


def _reflect(i, n):
    return np.where(i < 0, -i - 1, np.where(i >= n, 2 * n - i - 1, i))


def smooth(depth):
    """Normalised Gaussian convolution: pixels with D <= 0 have weight 0; vertical pass, then horizontal."""
    D = np.asarray(depth, F32)
    H, W = D.shape
    w = gauss_weights()
    valid = D > 0
    num = np.zeros_like(D)
    den = np.zeros_like(D)
    rows = np.arange(H)
    for k in range(-RADIUS, RADIUS + 1):
        r = _reflect(rows + k, H)
        ok = valid[r]
        num = np.where(ok, num + w[k + RADIUS] * D[r], num).astype(F32)
        den = np.where(ok, den + w[k + RADIUS], den).astype(F32)
    cols = np.arange(W)
    sn = np.zeros_like(D)
    sd = np.zeros_like(D)
    for k in range(-RADIUS, RADIUS + 1):
        c = _reflect(cols + k, W)
        sn = (sn + w[k + RADIUS] * num[:, c]).astype(F32)
        sd = (sd + w[k + RADIUS] * den[:, c]).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(sd > 0, sn / sd, F32(0)).astype(F32)


def gradient2(S, axis):
    """np.gradient(S, 2, edge_order=2) along `axis`, in the kernel's float32 operation order."""
    x = np.moveaxis(S, axis, 0)
    g = np.empty_like(x)
    g[1:-1] = (x[2:] - x[:-2]) / F32(4)
    g[0] = (F32(-0.75) * x[0] + x[1]) + F32(-0.25) * x[2]
    g[-1] = (F32(0.25) * x[-3] + (-x[-2])) + F32(0.75) * x[-1]
    return np.moveaxis(g, 0, axis)


def scene(depth, K, unit_per_m=1000.0):
    """Target map f32 [H,W,6] = (x, y, z, normal) of one frame; z = 0 where D is outside (0.2, 5) m."""
    D = np.asarray(depth, F32)
    K = np.asarray(K, F32)
    fx, cx, fy, cy = K[0, 0], K[0, 2], K[1, 1], K[1, 2]
    H, W = D.shape
    S = smooth(D)
    gv, gu = gradient2(S, 0), gradient2(S, 1)
    a = (np.arange(W, dtype=F32) - cx)[None, :]
    b = (np.arange(H, dtype=F32) - cy)[:, None]
    ix, iy = F32(1) / fx, F32(1) / fy
    tux = S * ix + (a * ix) * gu
    tuy = (b * iy) * gu
    tuz = gu
    tvx = (a * ix) * gv
    tvy = S * iy + (b * iy) * gv
    tvz = gv
    nx = tuy * tvz - tuz * tvy
    ny = tuz * tvx - tux * tvz
    nz = tux * tvy - tuy * tvx
    nn = np.sqrt((nx * nx + ny * ny) + nz * nz)
    with np.errstate(divide="ignore", invalid="ignore"):
        n = np.where(nn[..., None] > 0, np.stack([nx, ny, nz], -1) / nn[..., None], F32(0)).astype(F32)
    ok = (D > F32(0.2) * F32(unit_per_m)) & (D < F32(5) * F32(unit_per_m))
    x = np.where(ok, (a * D) / fx, F32(0))
    y = np.where(ok, (b * D) / fy, F32(0))
    z = np.where(ok, D, F32(0))
    return np.concatenate([np.stack([x, y, z], -1), n], -1).astype(F32)


def target_mask(tmap, rendered, mask, unit_per_m):
    d = tmap[..., 2]
    if mask is not None:
        return (d > 0) & (np.asarray(mask) != 0)
    R = np.asarray(rendered, F32)
    return (d > 0) & (R > 0) & (np.abs(d - R) <= F32(0.1) * F32(unit_per_m))


def backproject(pix, R, K, W):
    K = np.asarray(K, F32)
    fx, cx, fy, cy = K[0, 0], K[0, 2], K[1, 1], K[1, 2]
    v, u = pix // W, pix % W
    z = R.reshape(-1)[pix]
    return np.stack([((u.astype(F32) - cx) * z) / fx, ((v.astype(F32) - cy) * z) / fy, z], -1).astype(F32)


def transform(T, p):
    """((T0 x + T1 y) + T2 z) + T3 per row, float32."""
    T = np.asarray(T, F32)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], -1)


def associate(s, tmap, valid, K, rad):
    """Per transformed source point: (target pixel index or -1, distance float32 or +inf)."""
    K = np.asarray(K, F32)
    fx, cx, fy, cy = K[0, 0], K[0, 2], K[1, 1], K[1, 2]
    H, W = valid.shape
    n = len(s)
    best_i = np.full(n, -1, np.int64)
    best_d = np.zeros(n, F32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        front = s[:, 2] > 0
        pu = (fx * s[:, 0]) / s[:, 2] + cx
        pv = (fy * s[:, 1]) / s[:, 2] + cy
        ok = front & (np.abs(pu) < F32(1e7)) & (np.abs(pv) < F32(1e7))
        cu = np.where(ok, np.rint(pu), 0).astype(np.int64)
        cv = np.where(ok, np.rint(pv), 0).astype(np.int64)
    flat = tmap.reshape(-1, 6)
    vflat = valid.reshape(-1)
    for dv in range(-rad, rad + 1):
        for du in range(-rad, rad + 1):
            uu, vv = cu + du, cv + dv
            inside = ok & (uu >= 0) & (uu < W) & (vv >= 0) & (vv < H)
            t = np.where(inside, vv * W + uu, 0)
            cand = inside & vflat[t]
            q = flat[t]
            dx, dy, dz = q[:, 0] - s[:, 0], q[:, 1] - s[:, 1], q[:, 2] - s[:, 2]
            d2 = (dx * dx + dy * dy) + dz * dz
            better = cand & ((best_i < 0) | (d2 < best_d))
            best_i = np.where(better, t, best_i)
            best_d = np.where(better, d2, best_d)
    with np.errstate(invalid="ignore"):
        dist = np.sqrt(best_d).astype(F32)
        best_i = np.where(dist < F32(np.inf), best_i, -1)     # an overflowed (or NaN) distance is no pair
    dist = np.where(best_i >= 0, dist, F32(np.inf)).astype(F32)
    return best_i, dist


def normal_equations(s, q, n, L):
    """fp64 point-to-plane system of kept pairs: A^T A [6,6], A^T r [6], sum r^2."""
    s, q, n = s.astype(np.float64), q.astype(np.float64), n.astype(np.float64)
    r = ((s[:, 0] - q[:, 0]) * n[:, 0] + (s[:, 1] - q[:, 1]) * n[:, 1]) + (s[:, 2] - q[:, 2]) * n[:, 2]
    c = np.cross(s, n) / L
    J = np.concatenate([c, n], 1)
    return J.T @ J, J.T @ r, float(r @ r)


def solve(A, b):
    """Cholesky of the kernel (pivot <= 1e-8 x max diagonal: singular) -> xi or None."""
    A = np.array(A, np.float64)
    dmax = max(A[c, c] for c in range(6))
    Lm = np.zeros((6, 6))
    for c in range(6):
        d = A[c, c] - sum(Lm[c, e] ** 2 for e in range(c))
        if not d > 1e-8 * dmax:
            return None
        Lm[c, c] = np.sqrt(d)
        for r in range(c + 1, 6):
            Lm[r, c] = (A[r, c] - sum(Lm[r, e] * Lm[c, e] for e in range(c))) / Lm[c, c]
    y = np.zeros(6)
    for c in range(6):
        y[c] = (-b[c] - sum(Lm[c, e] * y[e] for e in range(c))) / Lm[c, c]
    x = np.zeros(6)
    for c in range(5, -1, -1):
        x[c] = (y[c] - sum(Lm[e, c] * x[e] for e in range(c + 1, 6))) / Lm[c, c]
    return x


def rodrigues(w):
    th = float(np.sqrt(w @ w))
    if th < 1e-8:
        A, B = 1.0 - th * th / 6.0, 0.5 - th * th / 24.0
    else:
        A, B = np.sin(th) / th, (1.0 - np.cos(th)) / (th * th)
    Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    return np.eye(3) + A * Wx + B * (Wx @ Wx)


def apply_step(dT, xi, L):
    """dT [3,4] fp64 <- [Rodrigues(omega) | v] dT; returns (dT, |omega|, |v|)."""
    w = np.asarray(xi[:3], np.float64) / L
    Rw = rodrigues(w)
    out = Rw @ dT
    out[:, 3] += xi[3:]
    return out, float(np.sqrt(w @ w)), float(np.sqrt(xi[3:] @ xi[3:]))


def sources_and_targets(tmap, rendered, box, mask, unit_per_m):
    """Target set [H,W] bool, target count, compacted source pixel indices (row-major inside the box)."""
    R = np.asarray(rendered, F32)
    H, W = R.shape
    valid = target_mask(tmap, R, mask, unit_per_m)
    x0, y0, x1, y1 = [int(v) for v in box]
    x0, x1 = max(0, min(W, x0)), max(0, min(W, x1))
    y0, y1 = max(0, min(H, y0)), max(0, min(H, y1))
    inbox = np.zeros((H, W), bool)
    inbox[y0:y1, x0:x1] = True
    counted = valid if mask is not None else valid & inbox
    src = np.flatnonzero((valid & (R > 0) & inbox).reshape(-1))
    return valid, int(counted.sum()), src


def refine(tmap, rendered, box, K, T0, mask=None, debug=None, **params):
    """Stages 2-6 for one hypothesis -> (pose f32 [4,4], status, residual, fitness).  `debug`, a dict, receives
    counts, sources, pose0 (the correction after the centroid shift), assoc (last level-0 iteration) and iterations."""
    p = dict(DEFAULTS, **params)
    upm = float(p["unit_per_m"])
    L = upm
    T0 = np.asarray(T0, F32)
    R = np.asarray(rendered, F32)
    H, W = R.shape
    valid, ntgt, src = sources_and_targets(tmap, R, box, mask, F32(upm))
    dbg = debug if debug is not None else {}
    dbg.update(counts=(ntgt, len(src)), sources=src)
    if ntgt < p["min_points"] or len(src) < p["min_points"]:
        return T0.copy(), TOO_FEW_POINTS, -1.0, 0.0
    flat = tmap.reshape(-1, 6)
    vt = valid.reshape(-1)
    tgt_mean = flat[vt, :3].astype(np.float64).mean(0)
    S0 = backproject(src, R, K, W)
    dT = np.zeros((3, 4))
    dT[:, :3] = np.eye(3)
    dT[:, 3] = tgt_mean - S0.astype(np.float64).mean(0)
    dbg["pose0"] = dT.astype(F32)
    residual, fitness, status = -1.0, 0.0, OK
    iters = {}
    step_t = float(F32(p["min_step_m"]) * F32(upm))
    for level in range(p["num_levels"] - 1, -1, -1):
        stride, rad = 1 << level, 2 << level
        s_lvl = S0[::stride]
        it = 0
        while it < p["max_iters"]:
            s = transform(dT.astype(F32), s_lvl)
            t, d = associate(s, tmap, valid, K, rad)
            found = t >= 0
            m = int(found.sum())
            if m == 0:
                status = LOST
                break
            med = np.sort(d[found])[(m - 1) // 2]
            kept = found & (d <= F32(p["rejection_scale"]) * med)
            if level == 0:
                dbg["assoc"] = np.where(~found, -1, np.where(kept, t, -2 - t))
            A, b, rr = normal_equations(s[kept], flat[t[kept], :3], flat[t[kept], 3:], L)
            nk = int(kept.sum())
            if level == 0:
                residual, fitness = (np.sqrt(rr / nk) if nk else -1.0), nk / len(s_lvl)
            if nk < 6:
                status = LOST
                break
            xi = solve(A, b)
            if xi is None:
                status = DEGENERATE
                break
            dT, wn, vn = apply_step(dT, xi, L)
            it += 1
            if wn < p["min_step_rad"] and vn < step_t:
                break
        iters[level] = it
        if status != OK:
            break
    dbg["iterations"] = iters
    if status == OK and not (0 <= residual <= float(F32(p["max_residual"]) * F32(upm))):
        status = RESIDUAL
    if status != OK:
        return T0.copy(), status, residual, fitness
    out = T0.copy()
    out[:3] = (dT[:, :3] @ T0[:3].astype(np.float64) + np.concatenate([np.zeros((3, 3)), dT[:, 3:]], 1)).astype(F32)
    return out, OK, residual, fitness
