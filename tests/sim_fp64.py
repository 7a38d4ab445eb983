"""An independent numpy restatement of the similarity search's epilogue (row a4), applied to fp32 similarity tiles.

Written from the reference, src/models/matching.py:231-278 (LocalSimilarity.test, tar2src direction) and :80-113
(find_consistency_patches); it does not use oracle/port.py or gigapose_b200.  Input: one raw fp32 tile or a batch of
them, [..., 256 t, 256 s], with the 16x16 template mask (over s) and query mask (over t).  Every decision is made in
fp32, in the reference's order:

- v = (raw * sm) * tm, each product rounded to fp32 (matching.py:234-235);
- v < thr -> +0.0 (:236);
- row and column maxima with torch.max's tie rule: the first index wins, and -0.0 equals +0.0 (:240-241);
- mask_sim = score >= thr (:247);
- the cycle test sqrt(dx^2 + dy^2) <= patch_threshold in fp32, together with score_src2tar[idx] >= thr (:95-113);
- mask_non_zero = tm * sm[idx] * (idx_src2tar != 0) * (idx_tar2src != 0), where `idx_src2tar != 0` is indexed by the
  query patch t, not by s: the reference multiplies the [.., s] tensor position-wise with the [.., t] ones (:263-268).

The per-template score sim_avg (:274-278) is summed in fp64 from the fp32 scores and masks, with a bar that holds for
any fp32 summation order: each product score * mask_all rounds once (u = 2^-24) and a sum of 256 terms in any order
errs by at most 255 u sum |x| (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 4.4), so
|fp32 result - fp64| <= 257 u sum_t |score_t mask_all_t| / 256.  Dividing by 256 is exact.

Note on the cycle test's similarity condition: score_src2tar[idx] is the maximum of a column that contains score
itself, so score >= thr implies it.  It can change mask_cycle (on rows whose score is below thr) but never mask_all;
`mask_cycle` is returned so that the condition can still be checked.

`mutation` names one deliberate error, so that a test can show its cases would catch it."""
from __future__ import annotations

import numpy as np

G = 16
P = G * G
U32 = 2.0 ** -24

MUTATIONS = ("thr_le", "tie_high", "mask_assoc", "quirk_s", "avg_by_count", "cycle_no_sim", "chebyshev")


def _argmax(v, axis, high):
    """First index of the maximum along `axis` (numpy compares -0.0 == +0.0, like torch.max); `high`: the last."""
    if not high:
        return np.argmax(v, axis=axis)
    return v.shape[axis] - 1 - np.argmax(np.flip(v, axis=axis), axis=axis)


def epilogue(tiles, smask, tmask, sim_threshold, patch_threshold, mutation=None):
    """tiles [..., 256 t, 256 s] fp32; smask [..., 256 s] and tmask [..., 256 t] broadcast against the leading dims.
    Returns per query patch t: score (fp32 score_tar2src), idx (idx_tar2src), valid (mask_all != 0), mask_all,
    mask_cycle; per column s: score_src2tar, idx_src2tar; per tile: sim_avg (fp64) and its bar sim_avg_bar."""
    assert mutation is None or mutation in MUTATIONS, mutation
    f32 = np.float32
    tiles = np.asarray(tiles, dtype=f32)
    lead = tiles.shape[:-2]
    sm = np.broadcast_to(np.asarray(smask, dtype=f32), lead + (P,))
    tm = np.broadcast_to(np.asarray(tmask, dtype=f32), lead + (P,))
    thr, pthr = f32(sim_threshold), f32(patch_threshold)
    high = mutation == "tie_high"

    if mutation == "mask_assoc":
        v = tiles * (sm[..., None, :] * tm[..., :, None])
    else:
        v = (tiles * sm[..., None, :]) * tm[..., :, None]
    below = (v <= thr) if mutation == "thr_le" else (v < thr)
    v[below] = f32(0.0)

    idx = _argmax(v, -1, high)                                                  # idx_tar2src [..., t]
    score = np.take_along_axis(v, idx[..., None], -1)[..., 0]
    idx_s2t = _argmax(v, -2, high)                                              # idx_src2tar [..., s]
    score_s2t = np.take_along_axis(v, idx_s2t[..., None, :], -2)[..., 0, :]
    del v, below

    mask_sim = score >= thr
    t = np.arange(P)
    back = np.take_along_axis(idx_s2t, idx, -1)                                 # idx_src2src
    dx = (back % G).astype(f32) - (t % G).astype(f32)
    dy = (back // G).astype(f32) - (t // G).astype(f32)
    if mutation == "chebyshev":
        dist = np.maximum(np.abs(dx), np.abs(dy))
    else:
        dist = np.sqrt(dx * dx + dy * dy)
    mask_cycle = dist <= pthr
    if mutation != "cycle_no_sim":
        mask_cycle &= np.take_along_axis(score_s2t, idx, -1) >= thr

    quirk = np.take_along_axis(idx_s2t, idx, -1) if mutation == "quirk_s" else idx_s2t
    mnz = tm * np.take_along_axis(sm, idx, -1)
    mnz = mnz * (quirk != 0).astype(f32)
    mnz = mnz * (idx != 0).astype(f32)
    mask_all = np.where(mask_sim & mask_cycle, mnz, f32(0.0))

    x = score.astype(np.float64) * mask_all.astype(np.float64)
    msum = mask_all.astype(np.float64).sum(-1)
    has = msum > 0
    denom = np.where(has, msum, 1.0) if mutation == "avg_by_count" else float(P)
    sim_avg = np.where(has, x.sum(-1) / denom, 0.0)
    bar = np.where(has, 257 * U32 * np.abs(x).sum(-1) / P, 0.0)
    return dict(score=score, idx=idx, valid=mask_all != 0, mask_all=mask_all, mask_cycle=mask_cycle,
                score_src2tar=score_s2t, idx_src2tar=idx_s2t, sim_avg=sim_avg, sim_avg_bar=bar)


def topk_consistent(order, sim_avg, bar):
    """Positions where a returned top-k order (template ids, best first) contradicts the restated sim_avg by more than
    the two templates' bars: a template ranked ahead of another must not score below it by more than bar_a + bar_b.
    Templates not returned count as ranked behind all returned ones.  `sim_avg`, `bar`: [T] fp64."""
    order = np.asarray(order)
    rest = np.setdiff1d(np.arange(len(sim_avg)), order)
    bad = []
    for i, a in enumerate(order):
        behind = np.concatenate([order[i + 1:], rest])
        if behind.size and np.any(sim_avg[behind] - sim_avg[a] > bar[behind] + bar[a]):
            bad.append(i)
    return bad


def ulp_neighbours(values, thr):
    """Counts of values equal to fp32 thr, one ulp below and one ulp above it."""
    thr = np.float32(thr)
    lo, hi = np.nextafter(thr, np.float32(-np.inf)), np.nextafter(thr, np.float32(np.inf))
    return int((values == thr).sum()), int((values == lo).sum()), int((values == hi).sum())
