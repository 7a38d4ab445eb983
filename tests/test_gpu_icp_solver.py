"""Row f6 inside the kernel: the depth refiner's (csrc/depth_icp.cu) median select, and every ICP iteration it traces,
against exact and fp64 references computed from the kernel's own state for that step (so one step's error cannot hide
another's, and the rounding drift of a whole trajectory does not blur the bars); the status paths with their traces,
batch and trace invariance, and the scene kernels at their edges.

Bars (u = 2^-53):
- normal equations: |got - want| <= G_SUMS u sum|term| per entry, want = the exactly rounded sum of the longdouble terms,
  sum|term| from the absolute values of every operand (so cancellation inside a term counts, see _terms);
- solve: ||A xi + b||inf <= C_BACK u (||A||inf ||xi||inf + ||b||inf), and xi within cond(A) C_FWD u of np.linalg.solve;
- step: dT within STEP_ULPS ulps of icp_port.apply_step(dT_prev, xi), relative to 1 + |t|.
Each test prints the largest measured value of its bars and the ratio by which fp32 arithmetic misses them."""
import math

import numpy as np
import pytest
import torch

from gigapose_b200 import _lib, icp
from icp_scenes import (DEV, H, K, T_ASM, T_ELL, W, assembly, ellipsoid, noisy_occluded_scene, perturb, plate, pose,
                        rot, scene)
from oracle import icp_port

pytestmark = pytest.mark.gpu

NO_PAIR = 0x7F800000
U = 2.0 ** -53
TRACE = np.dtype(_lib.GpIcpTrace)
CAP = 512
# Per-thread chains of ceil(n / 256) additions, 5 shuffle levels and 8 warps, plus ~6 roundings inside a term, bound the
# sums' error by (n / 256 + 19) u sum|term|, 47 at the 7 000 level-0 sources of these scenes.  On an H100 the largest
# values were 3.58 (sums), 0.99 (backward), 0.38 (forward) and 1.72 ulp (step); the bars are about 4x those
# (DESIGN.md §6).
G_SUMS = 15.0
C_BACK = 4.0
C_FWD = 1.5
STEP_ULPS = 8


# --- median select --------------------------------------------------------------------------------------------------

def _select(bits, rank):
    lib = _lib.load()
    d = torch.as_tensor(bits.view(np.int32)).to(DEV)
    out = torch.zeros(2, dtype=torch.int32, device=DEV)
    _lib.check(lib.gp_debug_icp_select(d.data_ptr(), len(bits), rank, out.data_ptr(), None))
    m, v = out.cpu().numpy().view(np.uint32)
    return int(m), int(v)


def _check_select(bits, ranks=None):
    bits = np.ascontiguousarray(bits, np.uint32)
    valid = np.sort(bits[bits != NO_PAIR])
    m = len(valid)
    if ranks is None:
        ranks = {0, (m - 1) // 2, m - 1} if m else {0}
    for r in sorted(ranks):
        got_m, got = _select(bits, r)
        want = int(valid[r]) if r < m else NO_PAIR
        assert (got_m, got) == (m, want), (len(bits), m, r, hex(got), hex(want))
    return len(ranks)


def _boundary(pass_, k, total, rng):
    """`total` values sharing the bytes above `pass_`, byte `pass_` = 0x40 for the first k and 0x41 for the rest,
    random bytes below, shuffled: rank k is the first of bucket 0x41 at that pass (count before it == rank), rank k - 1
    the last of bucket 0x40 (count before 0x41 == rank + 1)."""
    hi = np.uint32(0x3F123456) & ~np.uint32((1 << (8 * (pass_ + 1))) - 1) if pass_ < 3 else np.uint32(0)
    byte = np.where(np.arange(total) < k, 0x40, 0x41).astype(np.uint32) << np.uint32(8 * pass_)
    low = rng.integers(0, 1 << (8 * pass_), total, dtype=np.uint64).astype(np.uint32) if pass_ else np.uint32(0)
    return rng.permutation(hi | byte | low)


def test_median_select_is_exact():
    rng = np.random.default_rng(0)
    checked = 0
    for n in (1, 2, 3, 255, 256, 257, 4097, 307200):
        d = rng.uniform(0, 40, n).astype(np.float32).view(np.uint32)
        checked += _check_select(d)                                       # m = n
        d = d.copy()
        d[rng.integers(0, n)] = NO_PAIR                                    # m = n - 1: the other parity
        checked += _check_select(d)
    for n in (1, 2, 257, 4097):
        checked += _check_select(np.full(n, np.float32(3.25)).view(np.uint32))    # every value equal
        checked += _check_select(np.zeros(n, np.uint32))                           # every value +0.0
    checked += _check_select(np.uint32(0x42C80000) | rng.integers(0, 256, 3001).astype(np.uint32))  # lowest byte
    checked += _check_select((rng.integers(0, 0x80, 3001).astype(np.uint32) << np.uint32(24)) | np.uint32(0x123456))
    for pass_ in range(4):                                                 # rank on a histogram-bucket boundary
        for k, total in ((1, 2), (37, 100), (128, 1000), (300, 301)):
            b = _boundary(pass_, k, total, rng)
            checked += _check_select(b, {k - 1, k, 0, total - 1})
    top = np.array([0x3FFFFFFF, 0x3FFFFF00, 0x3FFF00FF, 0x3F00FFFF, 0x3FFFFFFE, 0x7F7FFFFF, 0x7F7FFF00], np.uint32)
    checked += _check_select(rng.permutation(np.concatenate([top, rng.integers(0, 0x3F000000, 50).astype(np.uint32)])),
                             set(range(57)))                               # bucket 255 at every pass, and FLT_MAX
    checked += _check_select(rng.integers(1, 0x00800000, 2049).astype(np.uint32))          # denormals
    checked += _check_select(np.array([0x7F7FFFFF, 0x7F7FFFFF, 0, 1], np.uint32), {0, 1, 2, 3})
    d = rng.uniform(0, 40, 5000).astype(np.float32).view(np.uint32)
    d[rng.random(5000) < 0.6] = NO_PAIR                                    # kNoPair interleaved
    checked += _check_select(d)
    for n, keep in ((1000, 137), (300, 299), (4096, None)):                # all but one entry kNoPair, and none left
        d = np.full(n, NO_PAIR, np.uint32)
        if keep is not None:
            d[keep] = 0x3F800000
        checked += _check_select(d, {0, 1, n - 1})
    print(f"median select: {checked} (array, rank) cases exact")


# --- traced runs -----------------------------------------------------------------------------------------------------

def _traced(depth, Ks, fidx, R, boxes, T0, masks, trace=True, **params):
    """gp_icp_refine over the given renders with the trace (and counts, sources, pose0, iterations) on."""
    F = depth.shape[0]
    n = T0.shape[0]
    L = params.get("num_levels", 4)
    ws = torch.empty(icp.workspace_bytes(F, n, H, W), dtype=torch.uint8, device=DEV)
    icp.prepare_scene(depth, Ks, ws, params.get("unit_per_m", 1000.0))
    dbg = dict(counts=torch.zeros(n, 2, dtype=torch.int32, device=DEV),
               sources=torch.full((n, H * W), -7, dtype=torch.int32, device=DEV),
               pose0=torch.zeros(n, 3, 4, device=DEV),
               iterations=torch.full((n, L), -1, dtype=torch.int32, device=DEV))
    if trace:
        dbg.update(trace=torch.zeros(n * CAP * TRACE.itemsize, dtype=torch.uint8, device=DEV), trace_capacity=CAP,
                   trace_count=torch.full((n,), -7, dtype=torch.int32, device=DEV))
    out = icp.refine_rendered(depth, Ks, fidx, R, boxes, T0, masks, ws, debug=dbg, **params)
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in dbg.items() if isinstance(v, torch.Tensor)}
    if trace:
        res["trace"] = res["trace"].view(TRACE).reshape(n, CAP)
    tmap = ws[:F * H * W * 24].view(torch.float32).reshape(F, H, W, 6).cpu().numpy()
    return [x.cpu().numpy() for x in out], res, tmap


def _one(mesh, T0, depth, mask, **params):
    dm = icp.device_meshes([mesh], DEV)
    T0t = torch.as_tensor(T0).reshape(1, 4, 4).to(DEV)
    Kt = torch.as_tensor(K).reshape(1, 3, 3).to(DEV)
    R, boxes = icp.render_hypotheses(dm, torch.tensor([0]), T0t, Kt, torch.tensor([0]), H, W)
    m = None if mask is None else mask.reshape(1, H, W).to(torch.uint8).contiguous()
    out, dbg, tmap = _traced(depth.reshape(1, H, W).contiguous(), Kt, torch.zeros(1, dtype=torch.int32, device=DEV),
                             R, boxes, T0t, m, **params)
    return out, dbg, tmap[0], R[0].cpu().numpy(), boxes[0].cpu().numpy(), m


def _pivots(S):
    """The kernel's Cholesky order on traced sums, in fp64: (pivots reached, threshold)."""
    A = np.zeros((6, 6))
    iu = np.triu_indices(6)
    A[iu] = S[:21]
    A = A + np.triu(A, 1).T
    thr = 1e-8 * max(A[c, c] for c in range(6))
    Lm = np.zeros((6, 6))
    piv = []
    for c in range(6):
        d = A[c, c]
        for e in range(c):
            d -= Lm[c, e] * Lm[c, e]
        piv.append(d)
        if not d > thr:
            break
        Lm[c, c] = math.sqrt(d)
        for r in range(c + 1, 6):
            s = A[r, c]
            for e in range(c):
                s -= Lm[r, e] * Lm[c, e]
            Lm[r, c] = s / Lm[c, c]
    return piv, thr


def _system(S, dtype=np.float64):
    A = np.zeros((6, 6), dtype)
    A[np.triu_indices(6)] = S[:21]
    return A + np.triu(A, 1).T, np.asarray(S[21:27], dtype)


def _chol_solve32(A, b):
    """The kernel's Cholesky solve of A xi = -b in float32 (the sensitivity check of the backward bar)."""
    A, b = A.astype(np.float32), b.astype(np.float32)
    Lm = np.zeros((6, 6), np.float32)
    for c in range(6):
        d = A[c, c] - np.float32(sum(Lm[c, :c] * Lm[c, :c]))
        Lm[c, c] = np.sqrt(max(d, np.float32(1e-30)))
        for r in range(c + 1, 6):
            Lm[r, c] = (A[r, c] - np.float32(sum(Lm[r, :c] * Lm[c, :c]))) / Lm[c, c]
    y = np.zeros(6, np.float32)
    for c in range(6):
        y[c] = (-b[c] - np.float32(sum(Lm[c, :c] * y[:c]))) / Lm[c, c]
    x = np.zeros(6, np.float32)
    for c in range(5, -1, -1):
        x[c] = (y[c] - np.float32(sum(Lm[c + 1:, c] * x[c + 1:]))) / Lm[c, c]
    return x


def _terms(s, q, nrm, L):
    """The 29 per-pair terms in longdouble from the fp32 s, q, n, and the magnitudes of their operands (what the
    rounding errors of the kernel's fp64 evaluation scale with)."""
    ld = np.longdouble
    s, q, nrm = s.astype(ld), q.astype(ld), nrm.astype(ld)
    d = s - q
    r = (d[:, 0] * nrm[:, 0] + d[:, 1] * nrm[:, 1]) + d[:, 2] * nrm[:, 2]
    rb = np.abs(d[:, 0] * nrm[:, 0]) + np.abs(d[:, 1] * nrm[:, 1]) + np.abs(d[:, 2] * nrm[:, 2])
    j, jb = [], []
    for a, b in ((1, 2), (2, 0), (0, 1)):
        j.append((s[:, a] * nrm[:, b] - s[:, b] * nrm[:, a]) / ld(L))
        jb.append((np.abs(s[:, a] * nrm[:, b]) + np.abs(s[:, b] * nrm[:, a])) / ld(L))
    for c in range(3):
        j.append(nrm[:, c])
        jb.append(np.abs(nrm[:, c]))
    t, tb = [], []
    for c in range(6):
        for e in range(c, 6):
            t.append(j[c] * j[e])
            tb.append(jb[c] * jb[e])
    for c in range(6):
        t.append(j[c] * r)
        tb.append(jb[c] * rb)
    t += [r * r, np.ones_like(r)]
    tb += [rb * rb, np.ones_like(r)]
    return t, tb


def _exact_sum(x):
    """The correctly rounded fp64 sum of longdouble values: each split exactly into two doubles, then math.fsum."""
    hi = x.astype(np.float64)
    lo = (x - hi.astype(np.longdouble)).astype(np.float64)
    return math.fsum(np.concatenate([hi, lo]).tolist())


def _check_trajectory(name, out, dbg, tmap, R, box, T0, mask, stats, h=0, Km=K, **params):
    """Every traced iteration of hypothesis h against references started from the record's own state."""
    p = dict(icp_port.DEFAULTS, **params)
    upm = np.float32(p["unit_per_m"])
    L = float(upm)
    pose_out, status, residual, fitness = (x[h] for x in out)
    count = int(dbg["trace_count"][h])
    assert 0 < count <= CAP, count
    rec = dbg["trace"][h, :count]
    m = None if mask is None else mask
    valid, ntgt, src = icp_port.sources_and_targets(tmap, R, box, m, upm)
    assert tuple(dbg["counts"][h]) == (ntgt, len(src))
    assert np.array_equal(dbg["sources"][h, :len(src)], src)
    S0 = icp_port.backproject(src, R, Km, W)
    flat = tmap.reshape(-1, 6)
    # chaining: Tf of record 0 is the fp32 centroid-shift pose, then fp32 of the previous record's dT, bit for bit
    assert np.array_equal(rec[0]["Tf"], dbg["pose0"][h].reshape(12))
    for a, b in zip(rec[:-1], rec[1:]):
        assert np.array_equal(b["Tf"], a["dT"].astype(np.float32))
    # levels: L-1 .. 0 in order, n = ceil(nsrc / 2^l), each completed level ends on done == 1 or after max_iters steps
    levels = rec["level"]
    assert (np.diff(levels) <= 0).all() and levels[0] == p["num_levels"] - 1
    for lv in np.unique(levels):
        r = rec[levels == lv]
        assert (r["iteration"] == np.arange(len(r))).all()
        assert (r["n"] == -(-len(src) // (1 << lv))).all()
        assert (r["done"][:-1] == 0).all()
        steps = int(((r["done"] == 0) | (r["done"] == 1)).sum())
        assert dbg["iterations"][h, lv] == steps
        last = r["done"][-1]
        if last in (2, 3):
            assert lv == levels[-1], "no level after one that ended the refinement"
        else:
            assert last == 1 or (last == 0 and len(r) == p["max_iters"]), (lv, last, len(r))
    if rec["done"][-1] in (0, 1):
        assert levels[-1] == 0
    gate_t = float(np.float32(p["min_step_m"]) * upm)
    dT_prev = None
    skipped = 0
    for j, t in enumerate(rec):
        lv, n = int(t["level"]), int(t["n"])
        s = icp_port.transform(t["Tf"].reshape(3, 4), S0[::1 << lv])
        assert len(s) == n
        tg, dist = icp_port.associate(s, tmap, valid, Km, 2 << lv)
        found = tg >= 0
        assert int(t["found"]) == int(found.sum()), (name, j)
        S = t["sums"]
        if t["found"] == 0:
            assert t["done"] == 3 and t["median_bits"] == NO_PAIR and t["kept"] == 0
            continue
        med = np.sort(dist[found])[(int(found.sum()) - 1) // 2]
        assert int(t["median_bits"]) == int(med.view(np.uint32)), (name, j)
        kept = found & (dist <= np.float32(p["rejection_scale"]) * med)
        assert int(t["kept"]) == int(kept.sum()) == S[28], (name, j)
        # normal equations: 29 sums against the exactly rounded longdouble sums
        terms, mags = _terms(s[kept], flat[tg[kept], :3], flat[tg[kept], 3:], L)
        miss32 = 0.0
        for k in range(29):
            want = _exact_sum(terms[k])
            scale = U * float(mags[k].astype(np.float64).sum())
            if scale == 0:
                assert S[k] == want, (name, j, k)
                continue
            stats["sums"] = max(stats["sums"], abs(S[k] - want) / scale)
            f32 = float(np.cumsum(terms[k].astype(np.float32), dtype=np.float32)[-1])
            miss32 = max(miss32, abs(f32 - want) / scale / G_SUMS)
            assert abs(S[k] - want) <= G_SUMS * scale, (name, j, k, S[k], want, scale)
        stats["sums32"] = min(stats["sums32"], miss32)
        if t["done"] == 3:
            assert S[28] < 6
            assert np.array_equal(t["xi"], np.zeros(6))
            assert dT_prev is None or np.array_equal(t["dT"], dT_prev)
            continue
        # degeneracy: the kernel's pivot test, in fp64 from the traced sums
        piv, thr = _pivots(S)
        near = [d for d in piv if abs(d - thr) <= 1e-6 * abs(thr)]
        skipped += len(near)
        if not near:
            if t["done"] == 2:
                assert not piv[-1] > thr, (name, j, piv, thr)
            else:
                assert len(piv) == 6 and all(d > thr for d in piv), (name, j, piv, thr)
        if t["done"] == 2:
            assert np.array_equal(t["xi"], np.zeros(6))
            assert dT_prev is None or np.array_equal(t["dT"], dT_prev)
            continue
        # solve: backward error in longdouble, forward error against np.linalg.solve
        A, b = _system(S)
        xi = t["xi"]
        ld = np.longdouble
        back = float(np.abs(A.astype(ld) @ xi.astype(ld) + b.astype(ld)).max())
        bscale = U * (np.abs(A).sum(1).max() * np.abs(xi).max() + np.abs(b).max())
        x_np = np.linalg.solve(A, -b)
        if bscale == 0:                                    # b = 0 (every residual 0): xi is 0 exactly
            assert back == 0 and not xi.any() and not x_np.any()
        else:
            stats["back"] = max(stats["back"], back / bscale)
            x32 = _chol_solve32(A, b).astype(ld)
            back32 = float(np.abs(A.astype(ld) @ x32 + b.astype(ld)).max()) / bscale / C_BACK
            stats["back32"] = min(stats["back32"], back32)
            assert back <= C_BACK * bscale, (name, j, back / bscale)
            fwd = np.abs(xi - x_np).max() / (np.linalg.cond(A, np.inf) * U * np.abs(x_np).max())
            stats["fwd"] = max(stats["fwd"], float(fwd))
            assert fwd <= C_FWD, (name, j, fwd)
        # step: Rodrigues and the left-multiplied composition, from the previous record's dT
        if dT_prev is None:
            # the fp64 centroid shift is not traced: record 0 starts from identity and the port's shift
            shift = np.zeros((3, 4))
            shift[:, :3] = np.eye(3)
            tgt_mean = flat[valid.reshape(-1), :3].astype(np.float64).mean(0)
            shift[:, 3] = tgt_mean - S0.astype(np.float64).mean(0)
            want, wn, vn = icp_port.apply_step(shift, xi, L)
            tb = 1e-9 * (1 + np.abs(want[:, 3]).max())
            assert np.abs(t["dT"].reshape(3, 4)[:, :3] - want[:, :3]).max() <= STEP_ULPS * 2.0 ** -52
            assert np.abs(t["dT"].reshape(3, 4)[:, 3] - want[:, 3]).max() <= tb
        else:
            want, wn, vn = icp_port.apply_step(dT_prev.reshape(3, 4), xi, L)
            err = np.abs(t["dT"].reshape(3, 4) - want).max() / (2.0 ** -52 * (1 + np.abs(want[:, 3]).max()))
            stats["step"] = max(stats["step"], float(err))
            assert err <= STEP_ULPS, (name, j, err)
        assert bool(t["done"] == 1) == (wn < float(np.float32(p["min_step_rad"])) and vn < gate_t), (name, j)
        dT_prev = t["dT"]
    stats["pivots_skipped"] += skipped
    stats["records"] += count
    # outputs: residual and fitness of the last level-0 record, bit for bit; the pose; the status decision
    lvl0 = rec[rec["level"] == 0]
    if len(lvl0):
        S = lvl0[-1]["sums"]
        want_res = np.float32(math.sqrt(S[27] / S[28])) if S[28] > 0 else np.float32(-1)
        assert residual.view(np.uint32) == want_res.view(np.uint32), (name, residual, want_res)
        assert fitness.view(np.uint32) == np.float32(S[28] / lvl0[-1]["n"]).view(np.uint32)
    last = rec[-1]["done"]
    if last in (0, 1):
        ok = 0 <= float(residual) <= float(np.float32(p["max_residual"]) * upm)
        assert status == (icp_port.OK if ok else icp_port.RESIDUAL)
    else:
        assert status == (icp_port.DEGENERATE if last == 2 else icp_port.LOST)
    if status == icp_port.OK:
        dT = rec[-1]["dT"].reshape(3, 4)
        want = (dT[:, :3] @ T0[:3].astype(np.float64) + np.c_[np.zeros((3, 3)), dT[:, 3]]).astype(np.float32)
        ulps = np.abs(pose_out[:3].view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)).max()
        stats["pose_ulps"] = max(stats["pose_ulps"], int(ulps))
        assert ulps <= 1 and np.array_equal(pose_out[3], T0[3])
    else:
        assert np.array_equal(pose_out, T0)
    return rec


def _new_stats():
    return dict(sums=0.0, sums32=np.inf, back=0.0, back32=np.inf, fwd=0.0, step=0.0, pose_ulps=0, pivots_skipped=0,
                records=0)


def _report(stats):
    print(f"{stats['records']} records: sums {stats['sums']:.2f} (bar {G_SUMS}), fp32 sums miss it by "
          f">= {stats['sums32']:.3g}x; backward {stats['back']:.3f} (bar {C_BACK}), fp32 Cholesky misses it by "
          f">= {stats['back32']:.3g}x; forward {stats['fwd']:.3g} (bar {C_FWD}); step {stats['step']:.2f} ulp (bar {STEP_ULPS}); "
          f"pose {stats['pose_ulps']} ulp; pivots within 1e-6 of the threshold skipped: {stats['pivots_skipped']}")


def _scene_iii():
    return noisy_occluded_scene(ellipsoid(), T_ELL)


@pytest.mark.parametrize("case", ["ellipsoid_mask", "assembly_threshold", "noisy_occluded", "at_the_truth"])
def test_every_traced_iteration_matches_the_fp64_reference(case):
    if case == "ellipsoid_mask":
        mesh, Tt = ellipsoid(), T_ELL
        d, mask = scene(mesh, Tt)
        T0 = perturb(Tt, [0.2, 1, 0.4], 8.0, [9.0, -8.0, 9.0])
    elif case == "assembly_threshold":
        mesh, Tt = assembly(), T_ASM
        d, _ = scene(mesh, Tt)
        mask = None
        T0 = perturb(Tt, [1, 0.3, -0.5], 7.0, [-10.0, 6.0, 10.0])
    elif case == "noisy_occluded":
        mesh, Tt = ellipsoid(), T_ELL
        d, mask = _scene_iii()
        T0 = perturb(Tt, [0.2, 1, 0.4], 8.0, [9.0, -8.0, 9.0])
    else:
        mesh, Tt = ellipsoid(), T_ELL
        d, mask = scene(mesh, Tt, background=None)
        T0 = Tt
    out, dbg, tmap, R, box, m = _one(mesh, T0, d, mask)
    stats = _new_stats()
    mk = None if m is None else m[0].cpu().numpy()
    rec = _check_trajectory(case, out, dbg, tmap, R, box, T0, mk, stats)
    counts = [int((rec["level"] == lv).sum()) for lv in (3, 2, 1, 0)]
    print(f"{case}: status {int(out[1][0])}, records per level 3/2/1/0 {counts}")
    _report(stats)
    assert stats["pivots_skipped"] == 0
    assert stats["sums32"] >= 100 and (case == "at_the_truth" or stats["back32"] >= 100)
    if case == "noisy_occluded":
        assert counts[0] == 100 and (rec[rec["level"] == 3]["done"] == 0).all()     # level 3 runs into max_iters
        assert (rec["kept"] < rec["found"]).any()                                    # the median gate rejects pairs
    if case == "at_the_truth":
        assert counts == [1, 1, 1, 1]
        assert (rec["median_bits"] == 0).all() and (rec["xi"] == 0).all() and (rec["done"] == 1).all()
        assert np.array_equal(out[0][0], T0) and int(out[1][0]) == _lib.ICP_OK and out[2][0] == 0


def test_status_paths_with_their_traces():
    stats = _new_stats()
    # DEGENERATE: a planar object, alone in the frame
    Tp = pose(np.eye(3), [10.0, 5.0, 700.0])
    dp, mp = scene(plate(), Tp, background=None)
    T0p = perturb(Tp, [0, 0, 1], 3.0, [4.0, 3.0, 2.0])
    out, dbg, tmap, R, box, m = _one(plate(), T0p, dp, mp)
    rec = _check_trajectory("plate", out, dbg, tmap, R, box, T0p, m[0].cpu().numpy(), stats)
    assert int(out[1][0]) == _lib.ICP_DEGENERATE and rec[-1]["done"] == 2
    piv, thr = _pivots(rec[-1]["sums"])
    assert not piv[-1] > thr
    print(f"plate: degenerate after {len(rec)} records, pivot {piv[-1]:.3e} <= {thr:.3e}")
    # LOST: a mask of 4 object pixels, so that level 3 has one source
    mesh = ellipsoid()
    d, mask = scene(mesh, T_ELL)
    ys, xs = torch.nonzero(mask, as_tuple=True)
    y, x = int(ys.float().mean()), int(xs.float().mean())
    m4 = torch.zeros_like(mask)
    m4[y:y + 2, x:x + 2] = True
    assert bool(mask[y:y + 2, x:x + 2].all())
    T0 = perturb(T_ELL, [0.2, 1, 0.4], 3.0, [3.0, -2.0, 4.0])
    out, dbg, tmap, R, box, m = _one(mesh, T0, d, m4, min_points=1)
    assert tuple(dbg["counts"][0]) == (4, 4)
    rec = _check_trajectory("lost", out, dbg, tmap, R, box, T0, m[0].cpu().numpy(), stats, min_points=1)
    assert int(out[1][0]) == _lib.ICP_LOST and len(rec) == 1 and rec[0]["done"] == 3 and rec[0]["n"] == 1
    # TOO_FEW_POINTS: min_points at min(targets, sources) runs, one more does not
    out, dbg, *_ = _one(mesh, T0, d, mask)
    lo = int(dbg["counts"][0].min())
    out, dbg, *_ = _one(mesh, T0, d, mask, min_points=lo)
    assert int(out[1][0]) != _lib.ICP_TOO_FEW_POINTS and dbg["trace_count"][0] > 0
    out, dbg, *_ = _one(mesh, T0, d, mask, min_points=lo + 1)
    assert int(out[1][0]) == _lib.ICP_TOO_FEW_POINTS and np.array_equal(out[0][0], T0)
    assert dbg["trace_count"][0] == 0 and out[2][0] == -1 and out[3][0] == 0
    # INVALID: frame indices -1 and n_frames
    dm = icp.device_meshes([mesh], DEV)
    T0t = torch.as_tensor(np.stack([T0, T0])).to(DEV)
    Kt = torch.as_tensor(K).reshape(1, 3, 3).to(DEV)
    R2, b2 = icp.render_hypotheses(dm, torch.tensor([0, 0]), T0t, Kt, torch.tensor([0, 0]), H, W)
    out, dbg, _ = _traced(d.reshape(1, H, W).contiguous(), Kt, torch.tensor([-1, 1], dtype=torch.int32, device=DEV),
                          R2, b2, T0t, None)
    assert (out[1] == _lib.ICP_INVALID).all() and np.array_equal(out[0], np.stack([T0, T0]))
    assert (out[2] == -1).all() and (out[3] == 0).all() and (dbg["trace_count"] == 0).all()
    _report(stats)


def test_batch_over_frames_with_their_own_K_and_trace_invariance():
    meshes = [ellipsoid(), assembly()]
    Ks = np.stack([K, K * np.float32([[1.1, 1, 0.97], [1, 1.05, 1.02], [1, 1, 1]]),
                   K * np.float32([[0.9, 1, 1.03], [1, 0.93, 0.96], [1, 1, 1]])]).astype(np.float32)
    frames = [(0, T_ELL), (1, T_ASM), (0, pose(rot([0, 1, 0], -20), [-60.0, 40.0, 650.0]))]
    depth = torch.stack([scene(meshes[o], T, Km=Ks[f])[0] for f, (o, T) in enumerate(frames)]).contiguous()
    rng = np.random.default_rng(5)
    T0, labels, fidx = [], [], []
    for i in range(12):
        f = i % 3
        o, Tt = frames[f]
        T0.append(perturb(Tt, rng.normal(size=3), rng.uniform(1, 6), rng.uniform(-8, 8, 3)))
        labels.append(o)
        fidx.append(f)
    T0 = np.stack(T0)
    dm = icp.device_meshes(meshes, DEV)
    Kt = torch.as_tensor(Ks).to(DEV)
    T0t = torch.as_tensor(T0).to(DEV)
    R, boxes = icp.render_hypotheses(dm, torch.tensor(labels), T0t, Kt, torch.tensor(fidx), H, W)
    fi = torch.tensor(fidx, dtype=torch.int32, device=DEV)
    out, dbg, tmaps = _traced(depth, Kt, fi, R, boxes, T0t, None)
    plain, plain_dbg, _ = _traced(depth, Kt, fi, R, boxes, T0t, None, trace=False)
    for a, b in zip(out, plain):
        assert np.array_equal(a, b)
    for k in plain_dbg:
        assert np.array_equal(dbg[k], plain_dbg[k]), k
    stats = _new_stats()
    Rn, bn = R.cpu().numpy(), boxes.cpu().numpy()
    for i in (0, 5, 11):
        alone, adbg, _ = _traced(depth, Kt, fi[i:i + 1].contiguous(), R[i:i + 1].contiguous(),
                                 boxes[i:i + 1].contiguous(), T0t[i:i + 1].contiguous(), None)
        c = int(dbg["trace_count"][i])
        assert adbg["trace_count"][0] == c
        assert dbg["trace"][i, :c].tobytes() == adbg["trace"][0, :c].tobytes()
        for a, b in zip(alone, out):
            assert np.array_equal(a[0], b[i])
        f = fidx[i]
        _check_trajectory(f"batch {i}", out, dbg, tmaps[f], Rn[i], bn[i], T0[i], None, stats, h=i, Km=Ks[f])
    print("statuses of the batch of 12:", np.bincount(out[1], minlength=6).tolist())
    _report(stats)


@pytest.mark.parametrize("size", [(17, 17), (17, 45), (33, 17)])
def test_scene_kernels_at_their_edges(size):
    """Three frames with their own K in one gp_icp_prepare_scene call: the reflect border of a radius-8 window on a
    17-pixel side, depth exactly at the excluded bounds and one ulp inside, zero and negative depth, border holes, and
    an all-zero frame (denominator 0, normal 0)."""
    h, w = size
    upm = np.float32(1000)
    lo, hi = np.float32(0.2) * upm, np.float32(5) * upm
    rng = np.random.default_rng(h * 100 + w)
    D = rng.uniform(300, 4000, (3, h, w)).astype(np.float32)
    D[0, 0, :] = 0                                                      # border holes
    D[0, :, -1] = 0
    D[1, -1, :] = 0
    D[1, :, 0] = -5.0
    specials = [lo, hi, np.nextafter(lo, np.float32(np.inf)), np.nextafter(hi, np.float32(0)), np.float32(0),
                np.float32(-1), np.float32(-0.0)]
    for f in (0, 1):
        for k, v in enumerate(specials):
            D[f, 1 + k % (h - 2), 2 + (3 * k) % (w - 3)] = v
    D[2] = 0                                                            # all-zero frame
    Ks = np.stack([[[572.4, 0, w / 2 - 0.3], [0, 573.6, h / 2 + 0.2], [0, 0, 1]],
                   [[300.0, 0, 1.5], [0, 310.0, h - 2.0], [0, 0, 1]],
                   [[800.0, 0, w * 0.7], [0, 790.0, 4.0], [0, 0, 1]]]).astype(np.float32)
    ws = torch.empty(icp.workspace_bytes(3, 0, h, w), dtype=torch.uint8, device=DEV)
    Dt = torch.as_tensor(D).to(DEV)
    _lib.check(_lib.load().gp_icp_prepare_scene(3, h, w, Dt.data_ptr(), torch.as_tensor(Ks).to(DEV).data_ptr(),
                                                float(upm), ws.data_ptr(), None))
    torch.cuda.synchronize()
    tmap = ws[:3 * h * w * 24].view(torch.float32).reshape(3, h, w, 6).cpu().numpy()
    worst = 0.0
    for f in range(3):
        want = icp_port.scene(D[f], Ks[f], unit_per_m=float(upm))
        assert np.array_equal(tmap[f, ..., :3].view(np.uint32), want[..., :3].view(np.uint32)), f
        worst = max(worst, float(np.abs(tmap[f, ..., 3:] - want[..., 3:]).max()))
        for v in (lo, hi):
            assert (tmap[f][D[f] == v][:, :3] == 0).all()
        inside = (D[f] == specials[2]) | (D[f] == specials[3])
        if f < 2:
            assert inside.sum() == 2 and (tmap[f][inside][:, 2] == D[f][inside]).all()
        assert (tmap[f][D[f] <= 0][:, :3] == 0).all()
    assert (tmap[2] == 0).all()
    print(f"scene {h}x{w}: normals max |kernel - port| = {worst:.3e}")
    assert worst < 4e-6
