"""numpy restatement of gp_teaser_refine (gigapose_b200/csrc/depth_teaser.cu, row f13), operation for operation: the
compaction, sampling, graph, clique, statuses and inlier counts are reproduced exactly, and the rotation and
translation bit for bit where the kernel's fp64 order is restated (every elementwise numpy op rounds once, as the
kernel does under -fmad=false).  `mutate` switches on one altered definition at a time, for the tests that show each
one is caught:  fps_start=i, inlier_le=True, edge_scale=1.0, compose_right=True, pad_copies=True."""
from __future__ import annotations

import math

import numpy as np

OK, TOO_FEW_POINTS, CLIQUE_TOO_SMALL, CLIQUE_BUDGET, TOO_FEW_INLIERS, INVALID = 0, 1, 2, 3, 4, 5
DEFAULTS = dict(unit_per_m=1000.0, min_points=100, n_points=1000, noise_bound=0.01, cbar2=1.0, min_inliers=50,
                gnc_factor=1.4, gnc_max_iters=100, gnc_cost_threshold=1e-12, clique_budget=20000)
SWEEPS = 8


def f32(x):
    return float(np.float32(x))


def points(depth, rendered, box, K):
    """-> src, tgt f32 [N,3]: the masked pixels of the render box in row-major order, back-projected."""
    H, W = depth.shape
    x0, y0, x1, y1 = (int(min(max(v, 0), lim)) for v, lim in zip(box, (W, H, W, H)))
    if x1 <= x0 or y1 <= y0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32)
    r, m = rendered[y0:y1, x0:x1].astype(np.float32), depth[y0:y1, x0:x1].astype(np.float32)
    mask = (m > 0) & (r > 0)
    vs, us = np.nonzero(mask)
    du = (us + x0).astype(np.float64) - np.float64(np.float32(K[0, 2]))
    dv = (vs + y0).astype(np.float64) - np.float64(np.float32(K[1, 2]))
    fx, fy = np.float32(K[0, 0]), np.float32(K[1, 1])

    def back(d):
        return np.stack([(du * (d / fx).astype(np.float64)).astype(np.float32),
                         (dv * (d / fy).astype(np.float64)).astype(np.float32), d], 1)
    return back(r[mask]), back(m[mask])


def fps(src, M, start=0):
    """Farthest-point sampling of M indices, fp32 ((dx dx + dy dy) + dz dz), the lowest index on a tie."""
    N = len(src)
    mind = np.full(N, np.inf, np.float32)
    idx = [start]
    for _ in range(1, M):
        d = src - src[idx[-1]]
        mind = np.minimum(mind, (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        idx.append(int(np.argmax(mind)))
    return np.asarray(idx, np.int64)


def graph(s, t, noise, cbar2, edge_scale=2.0):
    """Boolean adjacency [M,M] of the sampled correspondences (fp64, no diagonal)."""
    s, t = s.astype(np.float64), t.astype(np.float64)
    a, b = s[None] - s[:, None], t[None] - t[:, None]
    ls = np.sqrt((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2])
    lt = np.sqrt((b[..., 0] * b[..., 0] + b[..., 1] * b[..., 1]) + b[..., 2] * b[..., 2])
    adj = np.abs(lt - ls) <= (edge_scale * noise) * math.sqrt(cbar2)
    np.fill_diagonal(adj, False)
    return adj


def pack(adj):
    """[M,M] bool -> the kernel's rows, u32 [M,32] (bit b of word w = column 32 w + b)."""
    M = adj.shape[0]
    full = np.zeros((M, 1024), bool)
    full[:, :M] = adj
    return np.packbits(full, axis=1, bitorder="little").view("<u4")


def max_clique(adj, budget):
    """-> (members ascending, size, nodes, over budget): the kernel's search, with Python ints as bit sets over
    positions (degree descending, the lower index first)."""
    M = adj.shape[0]
    deg = adj.sum(1)
    vert = sorted(range(M), key=lambda i: (-int(deg[i]), i))
    sub = adj[np.ix_(vert, vert)]
    nbr = [int.from_bytes(np.packbits(row, bitorder="little").tobytes(), "little") for row in sub]
    first = lambda P: (P & -P).bit_length() - 1                       # noqa: E731
    full = (1 << M) - 1
    best, P = [], full
    while P:
        v = first(P)
        best.append(v)
        P &= nbr[v]
    bs = len(best)
    stack, cur = [full] + [0] * M, [0] * (M + 1)
    d, nodes, over, P = 0, 0, False, full
    while True:
        nodes += 1
        if nodes > budget:
            over = True
            break
        Q, k, last = P, 0, -1
        while Q:
            k += 1
            R = Q
            while R:
                v = first(R)
                R &= ~nbr[v] & ~(1 << v)
                Q &= ~(1 << v)
                last = v
        if k == 0 or d + k <= bs:
            if d == 0:
                break
            d -= 1
            P = stack[d] & ~(1 << cur[d])
            stack[d] = P
            continue
        v = last
        cur[d] = v
        NP = P & nbr[v]
        if not NP:
            if d + 1 > bs:
                bs, best = d + 1, cur[:d + 1]
            P &= ~(1 << v)
            stack[d] = P
            continue
        stack[d] = P
        d += 1
        P = NP
        stack[d] = P
    return np.sort(np.asarray([vert[p] for p in best], np.int64)), bs, nodes, over


def lane_sum(vals):
    """The kernel's warp sum: lane l adds k = l, l + 32, .. in order, then an xor butterfly 16, 8, 4, 2, 1."""
    vals = np.asarray(vals, np.float64)
    acc = np.zeros((32,) + vals.shape[1:])
    for r in range(0, len(vals), 32):
        c = vals[r:r + 32]
        acc[:len(c)] = acc[:len(c)] + c
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[lanes ^ o]
    return acc[0]


def horn(S):
    """The kernel's `horn`: rotation (row-major list of 9) of Horn's quaternion of S (S[3a+b] = sum s_a t_b)."""
    xx, xy, xz, yx, yy, yz, zx, zy, zz = (float(v) for v in S)
    A = [[(xx + yy) + zz, yz - zy, zx - xz, xy - yx],
         [yz - zy, (xx - yy) - zz, xy + yx, zx + xz],
         [zx - xz, xy + yx, (yy - xx) - zz, yz + zy],
         [xy - yx, zx + xz, yz + zy, (zz - xx) - yy]]
    V = [[1.0 if i == j else 0.0 for j in range(4)] for i in range(4)]
    for _ in range(SWEEPS):
        for p in range(3):
            for q in range(p + 1, 4):
                apq = A[p][q]
                if apq == 0.0:
                    continue
                th = (A[q][q] - A[p][p]) / (2.0 * apq)
                tt = (1.0 if th >= 0.0 else -1.0) / (abs(th) + math.sqrt(th * th + 1.0))
                c = 1.0 / math.sqrt(tt * tt + 1.0)
                s = tt * c
                for k in range(4):
                    akp, akq = A[k][p], A[k][q]
                    A[k][p], A[k][q] = c * akp - s * akq, s * akp + c * akq
                for k in range(4):
                    apk, aqk = A[p][k], A[q][k]
                    A[p][k], A[q][k] = c * apk - s * aqk, s * apk + c * aqk
                for k in range(4):
                    vkp, vkq = V[k][p], V[k][q]
                    V[k][p], V[k][q] = c * vkp - s * vkq, s * vkp + c * vkq
    e = 0
    for k in range(1, 4):
        if A[k][k] > A[e][e]:
            e = k
    qw, qx, qy, qz = V[0][e], V[1][e], V[2][e], V[3][e]
    nq = math.sqrt(((qw * qw + qx * qx) + qy * qy) + qz * qz)
    qw, qx, qy, qz = qw / nq, qx / nq, qy / nq, qz / nq
    return [((qw * qw + qx * qx) - qy * qy) - qz * qz, 2.0 * (qx * qy - qw * qz), 2.0 * (qx * qz + qw * qy),
            2.0 * (qx * qy + qw * qz), ((qw * qw - qx * qx) + qy * qy) - qz * qz, 2.0 * (qy * qz - qw * qx),
            2.0 * (qx * qz - qw * qy), 2.0 * (qy * qz + qw * qx), ((qw * qw - qx * qx) - qy * qy) + qz * qz]


def chain_tims(s, t, members):
    a, b = members, np.roll(members, -1)
    return s[b].astype(np.float64) - s[a].astype(np.float64), t[b].astype(np.float64) - t[a].astype(np.float64)


def residuals(R, s, t):
    R = np.asarray(R, np.float64)
    e = [t[:, a] - ((R[3 * a] * s[:, 0] + R[3 * a + 1] * s[:, 1]) + R[3 * a + 2] * s[:, 2]) for a in range(3)]
    return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]


def weighted_S(w, s, t):
    ws = w[:, None] * s
    return lane_sum((ws[:, :, None] * t[:, None, :]).reshape(-1, 9))


def gnc_tls(s, t, eps2, factor, max_iters, thr):
    """-> R (list of 9), trace [dict(weights, R, mu, cost, max_residual, stopped)]."""
    m = len(s)
    w = np.ones(m)
    prev, mu, trace, R = math.inf, 0.0, [], None
    for it in range(max_iters):
        R = horn(weighted_S(w, s, t))
        r = residuals(R, s, t)
        maxr = float(r.max())
        rec = dict(weights=w.copy(), R=np.asarray(R), max_residual=maxr, stopped=False, cost=0.0)
        stop = False
        if it == 0:
            mu = 1.0 / ((2.0 * maxr) / eps2 - 1.0)
            stop = not mu > 0.0 or math.isinf(mu)
        rec["mu"] = mu
        if stop:
            rec["stopped"] = True
            trace.append(rec)
            break
        th1, th2 = ((mu + 1.0) / mu) * eps2, (mu / (mu + 1.0)) * eps2
        with np.errstate(divide="ignore", invalid="ignore"):
            mid = np.sqrt(((eps2 * mu) * (mu + 1.0)) / r) - mu
        w = np.where(r >= th1, 0.0, np.where(r <= th2, 1.0, mid))
        cost = float(lane_sum(w * r))
        rec["cost"] = cost
        trace.append(rec)
        diff = abs(cost - prev)
        mu = mu * factor
        prev = cost
        if diff < thr:
            break
    return R, trace


def vote(x, r, upm):
    """The kernel's adaptive voting on one axis -> the estimate."""
    m = len(x)
    val = np.concatenate([x - r, x + r])
    sec = np.concatenate([np.arange(1, m + 1), -np.arange(1, m + 1)])
    order = np.lexsort((sec, val))
    cnt, sx, sxx, rs, best, est = 0, 0.0, 0.0, 0.0, math.inf, 0.0
    for _ in range(m):
        rs = rs + r
    for e in order:
        i = int(e % m)
        xi = float(x[i])
        if e >= m:
            cnt, sx, sxx, rs = cnt - 1, sx - xi, sxx - xi * xi, rs + r
        else:
            cnt, sx, sxx, rs = cnt + 1, sx + xi, sxx + xi * xi, rs - r
        if cnt > 0:
            mean = sx / float(cnt)
            cost = (((float(cnt) * mean) * mean + sxx) - (2.0 * sx) * mean) + upm * rs
            if cost < best:
                best, est = cost, mean
    return est


def inliers(R, tv, s, t, noise, le=False):
    """Samples with ||R s + t - t_i|| < noise (the kernel's order; `le` counts <= instead, a mutation)."""
    R = np.asarray(R, np.float64).reshape(-1)
    sd, td = s.astype(np.float64), t.astype(np.float64)
    e = [(((R[3 * a] * sd[:, 0] + R[3 * a + 1] * sd[:, 1]) + R[3 * a + 2] * sd[:, 2]) + tv[a]) - td[:, a]
         for a in range(3)]
    dist = np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
    return int(np.count_nonzero(dist <= noise if le else dist < noise))


def compose(T, T0, right=False):
    """fp32 of [R | t] T0 in fp64, rows ((T_a0 T0_0b + T_a1 T0_1b) + T_a2 T0_2b) + T_a3 T0_3b; the last row is T0's.
    `right` composes T0 T instead (a mutation)."""
    T0 = np.asarray(T0, np.float32)
    A, B = (T0.astype(np.float64), T) if right else (T, T0.astype(np.float64))
    pose = T0.copy()
    for a in range(3):
        for b in range(4):
            pose[a, b] = np.float32(((A[a, 0] * B[0, b] + A[a, 1] * B[1, b]) + A[a, 2] * B[2, b]) + A[a, 3] * B[3, b])
    return pose


def refine_one(depth, rendered, box, K, T0, frame_ok=True, mutate=None, **params):
    """One hypothesis -> dict(status, pose f32 [4,4], inliers, clique, and every intermediate)."""
    mutate = mutate or {}
    p = dict(DEFAULTS, **params)
    upm = f32(p["unit_per_m"])
    noise = f32(p["noise_bound"]) * upm
    eps2 = noise * noise
    cbar2 = f32(p["cbar2"])
    T0 = np.asarray(T0, np.float32)
    out = dict(status=OK, pose=T0.copy(), inliers=0, clique=0, N=0, M=0)
    if not frame_ok:
        out.update(status=INVALID, N=-1)
        return out
    src, tgt = points(depth, rendered, box, K)
    N = len(src)
    out.update(src=src, tgt=tgt, N=N)
    if N < p["min_points"] or N < 1:
        out["status"] = TOO_FEW_POINTS
        return out
    n_points = int(p["n_points"])
    M = min(n_points, N)
    idx = fps(src, M, mutate.get("fps_start", 0))
    if mutate.get("pad_copies") and N < n_points:
        idx = np.concatenate([idx, np.full(n_points - N, N - 1)])
        M = n_points
    s, t = src[idx], tgt[idx]
    adj = graph(s, t, noise, cbar2, mutate.get("edge_scale", 2.0))
    members, size, nodes, over = max_clique(adj, int(p["clique_budget"]))
    out.update(M=M, samples=idx, adjacency=pack(adj), clique=size, nodes=nodes, members=members)
    if over:
        out["status"] = CLIQUE_BUDGET
        return out
    if size < 3:
        out["status"] = CLIQUE_TOO_SMALL
        return out
    ts, tt = chain_tims(s, t, members)
    R, trace = gnc_tls(ts, tt, eps2, f32(p["gnc_factor"]), int(p["gnc_max_iters"]),
                       float(p["gnc_cost_threshold"]) * (upm * upm))
    R = np.asarray(R)
    sm, tm = s[members].astype(np.float64), t[members].astype(np.float64)
    r = noise * math.sqrt(cbar2)
    tv = np.array([vote(tm[:, a] - ((R[3 * a] * sm[:, 0] + R[3 * a + 1] * sm[:, 1]) + R[3 * a + 2] * sm[:, 2]), r, upm)
                   for a in range(3)])
    inl = inliers(R, tv, s, t, noise, mutate.get("inlier_le", False))
    out.update(R=R.reshape(3, 3), t=tv, gnc=trace, inliers=inl)
    if inl < p["min_inliers"]:
        out["status"] = TOO_FEW_INLIERS
        return out
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R.reshape(3, 3), tv
    pose = compose(T, T0, mutate.get("compose_right", False))
    out["pose"] = pose
    return out


def refine(depth, K, frame_idx, rendered, boxes, T0, mutate=None, **params):
    """Every hypothesis; depth [F,H,W], K [F,3,3], frame_idx [n], rendered [n,H,W], boxes [n,4], T0 [n,4,4]."""
    F = depth.shape[0]
    return [refine_one(depth[f] if 0 <= f < F else depth[0], rendered[i], boxes[i], K[f] if 0 <= f < F else K[0],
                       T0[i], 0 <= f < F, mutate, **params) for i, f in enumerate(np.asarray(frame_idx).tolist())]
