"""CPU restatement of the BOP 2019 pose errors (gigapose_b200/csrc/bop_eval.cu) and of the matching into recalls, from
the published definitions: VSD (Hodan et al., BOP, ECCV 2018), MSSD / MSPD and the average recall (Hodan et al.,
BOP Challenge 2020 report).  Two forms of each error:
  *_fp32  the kernels' float32 arithmetic in their stated operation order, every operation rounded once, so that the
          kernels' outputs are meant to be bit-identical;
  *_fp64  the plain definitions in float64, to bound the fp32 error.
Depth maps come from `render_depth` below, the one-sample restatement of gp_render_depth built on the setup and
barycentric helpers of oracle/render_port.py.  Test infrastructure, like oracle/port.py."""
from __future__ import annotations

import numpy as np

from oracle import render_port as rp

F32 = np.float32


# ---------------------------------------------------------------------------------------------------- depth renders
def render_depth(vertices, faces, pose, K, H, W, z_near):
    """gp_render_depth for one view: the same setup, 64-bit edge functions and per-sample depth as
    render_port.rasterize, with ONE sample per pixel at the pixel centre (offset 0, so a face reaches the pixels whose
    centre its snapped box contains); key = (float bits of z) << 32 | face id, the minimum wins.
    -> dict(depth f32 [H,W] (0 = background), box i64 [4] of depth > 0, (0, 0, W, H) when empty)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    t = rp._setup(vertices, faces, pose, K, z_near)
    keys = np.full(H * W, rp.EMPTY, dtype=np.uint64)
    fid = np.nonzero(t["valid"])[0]
    if len(fid):
        x, y = t["x"][fid], t["y"][fid]
        px0 = np.maximum(-((0 - x.min(1)) >> 8), 0)
        px1 = np.minimum(x.max(1) >> 8, W - 1)
        py0 = np.maximum(-((0 - y.min(1)) >> 8), 0)
        py1 = np.minimum(y.max(1) >> 8, H - 1)
        bw, bh = px1 - px0 + 1, py1 - py0 + 1
        keep = (bw > 0) & (bh > 0)
        fid, px0, py0, bw, bh = fid[keep], px0[keep], py0[keep], bw[keep], bh[keep]
        starts = np.concatenate([[0], np.cumsum(bw * bh)])
        step = 1 << 22
        for lo in range(0, int(starts[-1]), step):
            idx = np.arange(lo, min(lo + step, int(starts[-1])))
            k = np.searchsorted(starts, idx, side="right") - 1
            p = idx - starts[k]
            px, py, f = px0[k] + p % bw[k], py0[k] + p // bw[k], fid[k]
            b, inside = rp._weights(t, f, px * 256, py * 256)
            z = rp._depth(b[inside])
            key = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | f[inside].astype(np.uint64)
            np.minimum.at(keys, py[inside] * W + px[inside], key)
    covered = keys != rp.EMPTY
    depth = np.where(covered, (keys >> np.uint64(32)).astype(np.uint32).view(F32), F32(0)).reshape(H, W)
    ys, xs = np.nonzero(depth > 0)
    box = np.array([xs.min(), ys.min(), xs.max() + 1, ys.max() + 1] if len(xs) else [0, 0, W, H], np.int64)
    return dict(depth=depth, box=box)


# ---------------------------------------------------------------------------------------------------- VSD
def _union_box(box_a, box_b, H, W):
    x0, y0 = max(min(box_a[0], box_b[0]), 0), max(min(box_a[1], box_b[1]), 0)
    x1, y1 = min(max(box_a[2], box_b[2]), W), min(max(box_a[3], box_b[3]), H)
    return int(x0), int(y0), int(max(x1, x0)), int(max(y1, y0))


def dist_fp32(z, K, x0, y0):
    """Distance from the camera centre of depth z [h,w] whose top-left pixel is (x0, y0), kernel order."""
    z = np.asarray(z, F32)
    K = np.asarray(K, F32).reshape(3, 3)
    h, w = z.shape
    u = np.arange(x0, x0 + w, dtype=F32)[None]
    v = np.arange(y0, y0 + h, dtype=F32)[:, None]
    X = ((u - K[0, 2]) * z) / K[0, 0]
    Y = ((v - K[1, 2]) * z) / K[1, 1]
    return np.sqrt((X * X + Y * Y) + z * z).astype(F32)


def dist_fp64(z, K):
    z = np.asarray(z, np.float64)
    K = np.asarray(K, np.float64).reshape(3, 3)
    h, w = z.shape
    u, v = np.arange(w)[None], np.arange(h)[:, None]
    return np.sqrt(((u - K[0, 2]) * z / K[0, 0]) ** 2 + ((v - K[1, 2]) * z / K[1, 1]) ** 2 + z ** 2)


def _masks(d_test, d_gt, d_est, delta):
    vis = lambda d: (d > 0) & (((d - d_test) <= delta) | (d_test == 0))
    visib_gt = vis(d_gt)
    visib_est = vis(d_est) | (visib_gt & (d_est > 0))
    return visib_gt, visib_est


def vsd_fp32(depth_test, K, est_depth, est_box, gt_depth, gt_box, diameter, delta, taus):
    """One pair -> (counts int64 [2 + n_tau] = (inter, union, cost per tau), errors f32 [n_tau]), kernel order."""
    H, W = depth_test.shape
    x0, y0, x1, y1 = _union_box(est_box, gt_box, H, W)
    sl = (slice(y0, y1), slice(x0, x1))
    d_test, d_gt, d_est = (dist_fp32(np.asarray(d, F32)[sl], K, x0, y0) for d in (depth_test, gt_depth, est_depth))
    visib_gt, visib_est = _masks(d_test, d_gt, d_est, F32(delta))
    inter, union = visib_gt & visib_est, visib_gt | visib_est
    c = np.abs(d_gt - d_est) / F32(diameter)
    costs = [int(np.count_nonzero(inter & (c >= F32(t)))) for t in taus]
    ni, nu = int(inter.sum()), int(union.sum())
    err = [F32(1) if nu == 0 else F32(F32(ct + nu - ni) / F32(nu)) for ct in costs]
    return np.array([ni, nu] + costs, np.int64), np.array(err, F32)


def vsd_fp64(depth_test, K, est_depth, gt_depth, diameter, delta, taus):
    """The definition over the whole image in float64 -> (counts, errors)."""
    d_test, d_gt, d_est = (dist_fp64(d, K) for d in (depth_test, gt_depth, est_depth))
    visib_gt, visib_est = _masks(d_test, d_gt, d_est, float(delta))
    inter, union = visib_gt & visib_est, visib_gt | visib_est
    c = np.abs(d_gt - d_est) / float(diameter)
    costs = [int(np.count_nonzero(inter & (c >= t))) for t in taus]
    ni, nu = int(inter.sum()), int(union.sum())
    err = [1.0 if nu == 0 else (ct + nu - ni) / nu for ct in costs]
    return np.array([ni, nu] + costs, np.int64), np.array(err)


# ---------------------------------------------------------------------------------------------------- MSSD / MSPD
def _affine32(A, P):
    A = np.asarray(A, F32).reshape(-1, 4)
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    return np.stack([((A[r, 0] * x + A[r, 1] * y) + A[r, 2] * z) + A[r, 3] for r in range(3)], 1).astype(F32)


def _project32(K, P):
    K = np.asarray(K, F32).reshape(3, 3)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = (K[0, 0] * P[:, 0] + K[0, 1] * P[:, 1]) / P[:, 2] + K[0, 2]
        v = (K[1, 1] * P[:, 1]) / P[:, 2] + K[1, 2]
    return u.astype(F32), v.astype(F32)


def _bits_max(x):
    return np.asarray(x, F32).view(np.uint32).max()


def mssd_mspd_fp32(vertices, syms, pose_est, pose_gt, K):
    """-> (mssd, mspd) float32, kernel order: squared terms, max over vertices and min over transforms on the float
    bits (NaN last), one sqrt."""
    V = np.asarray(vertices, F32)
    e = _affine32(pose_est, V)
    ue, ve = _project32(K, e)
    best_d = best_p = np.uint32(0xFFFFFFFF)
    with np.errstate(over="ignore", invalid="ignore"):
        for S in np.asarray(syms, F32).reshape(-1, 4, 4):
            g = _affine32(pose_gt, _affine32(S, V))
            ug, vg = _project32(K, g)
            d = e - g
            dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            du, dv = ue - ug, ve - vg
            pp = du * du + dv * dv
            for val, which in ((dd, 0), (pp, 1)):
                m = np.sqrt(np.uint32(_bits_max(val)).view(F32)).astype(F32).view(np.uint32)
                if which == 0:
                    best_d = min(best_d, m)
                else:
                    best_p = min(best_p, m)
    return np.uint32(best_d).view(F32), np.uint32(best_p).view(F32)


def mssd_mspd_fp64(vertices, syms, pose_est, pose_gt, K):
    V = np.asarray(vertices, np.float64)
    Pe, Pg = np.asarray(pose_est, np.float64).reshape(4, 4), np.asarray(pose_gt, np.float64).reshape(4, 4)
    K = np.asarray(K, np.float64).reshape(3, 3)
    e = V @ Pe[:3, :3].T + Pe[:3, 3]
    proj = lambda P: np.stack([(K[0, 0] * P[:, 0] + K[0, 1] * P[:, 1]) / P[:, 2] + K[0, 2],
                               K[1, 1] * P[:, 1] / P[:, 2] + K[1, 2]], 1)
    pe = proj(e)
    mssd = mspd = np.inf
    for S in np.asarray(syms, np.float64).reshape(-1, 4, 4):
        g = (V @ S[:3, :3].T + S[:3, 3]) @ Pg[:3, :3].T + Pg[:3, 3]
        mssd = min(mssd, np.linalg.norm(e - g, axis=1).max())
        mspd = min(mspd, np.linalg.norm(pe - proj(g), axis=1).max())
    return mssd, mspd


# ---------------------------------------------------------------------------------------------------- matching
def average_recalls(pairs, targets, taus, theta_vsd, theta_mssd, theta_mspd, r):
    """pairs: dicts (target, rank, gt, vsd [n_tau], mssd, mspd), rank = position of the estimate in its target's
    descending score order; targets: dicts (valid {gt: bool}, diameter).  Greedy matching per target and threshold:
    estimates by rank, each takes the unmatched valid gt with the smallest error strictly below the threshold (the
    first in gt order on a tie).  -> dict(ar, ar_vsd, ar_mssd, ar_mspd, recall_vsd [n_tau, n_theta], recall_mssd,
    recall_mspd)."""
    n_targets = sum(sum(1 for v in t["valid"].values() if v) for t in targets)
    by_target = {}
    for p in pairs:
        by_target.setdefault(p["target"], []).append(p)

    def matched(err_of, th_of):
        total = 0
        for ti, ps in by_target.items():
            valid, th = targets[ti]["valid"], th_of(targets[ti])
            taken = set()
            for rank in sorted({p["rank"] for p in ps}):
                best, best_e = None, None
                for p in sorted((p for p in ps if p["rank"] == rank), key=lambda p: p["gt"]):
                    e = float(err_of(p))
                    if not valid[p["gt"]] or p["gt"] in taken or not e < th:
                        continue
                    if best is None or e < best_e:
                        best, best_e = p["gt"], e
                if best is not None:
                    taken.add(best)
                    total += 1
        return total

    n = max(n_targets, 1)
    rv = np.array([[matched(lambda p, t=t: p["vsd"][t], lambda _, th=th: th) / n for th in theta_vsd]
                   for t in range(len(taus))])
    rs = np.array([matched(lambda p: p["mssd"], lambda tg, th=th: th * tg["diameter"]) / n for th in theta_mssd])
    rp = np.array([matched(lambda p: p["mspd"], lambda _, th=th: th * r) / n for th in theta_mspd])
    a = (float(rv.mean()), float(rs.mean()), float(rp.mean()))
    return dict(ar=sum(a) / 3, ar_vsd=a[0], ar_mssd=a[1], ar_mspd=a[2], recall_vsd=rv, recall_mssd=rs, recall_mspd=rp)
