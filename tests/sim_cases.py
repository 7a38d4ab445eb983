"""Inputs for the similarity-epilogue tests (test_sim_fp64_cpu.py, test_gpu_sim_epilogue.py): synthetic FeatureCases
whose decisions sit where a kernel epilogue goes wrong, and the CPU tiles that LocalSimilarity.test computes on them.

- `realistic`: a shared low-rank component makes most masked products fall in 0.3-0.7 (median ~0.5), so a
  threshold of 0.5 cuts through the bulk of them instead of sitting far below planted ~0.99 matches.
- `plant_ties`: exact row and column ties, planted by duplicated rows (the same descriptor in two template patches, or
  in two query patches) and placed across the kernel's lanes, warpgroups and the second t-half.
- `frac_masks` / `edge_masks`: alpha masks in {0.25, 0.5, 0.75, 1}; all-zero, single-patch and border masks.
- `plant_cycle_pairs`: duplicated query rows at grid distance 1, sqrt(2) and 3, so that the cycle test's back
  match lands on the other row of the pair: `pick_knife` then puts sim_threshold and patch_threshold exactly on one of
  these decisions."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from gigapose_b200 import synth

import sim_fp64

G, P, C = 16, 256, synth.C_AE

# (s_lo, s_hi, t): template patches s_lo and s_hi carry one descriptor, query patch t matches it.  In the kernel's
# accumulator fragment column s sits in lane 4 k + (s % 8) // 2, register pair s % 2, loop step s // 8:
# 4 / 5 one lane and register pair, 2 / 10 one lane in two loop steps, 1 / 202 two lanes
ROW_TIES = ((4, 5, 5), (2, 10, 40), (1, 202, 202))
# (t_lo, t_hi): query patches with one descriptor, both matching template patch s = t_lo.  Rows t0 / t0 + 8 of a lane
# (3 / 11), two lanes (16 / 17), two warpgroups (20 / 100), both in the second t-half (130 / 250)
COL_TIES = ((3, 11), (16, 17), (20, 100), (130, 250))
# (t', t, s): query rows t' < t duplicated, template patches s < t and t match them; t's cycle lands on t'.  Template
# patch t carries the match too, so that at a threshold as high as the match column t keeps a nonzero arg-max (the
# reference reads idx_src2tar at t)
CYCLE_PAIRS = ((57, 74, 60), (88, 89, 72), (150, 153, 151))     # distances sqrt(2), 1, 3


def _unit(x):
    return F.normalize(x, dim=-1)


def realistic(B, O, T, seed, labels=None, device="cpu", shared=0.7, spread=0.35):
    """make_feature_case's geometry and planted matches, mixed with one shared component c = m + spread * (rank-4 term):
    f <- normalize(sqrt(shared) c + sqrt(1 - shared) f)."""
    case = synth.make_feature_case(B=B, O=O, T=T, seed=seed, labels=labels, device=device)
    g = torch.Generator(device=device).manual_seed(seed + 1000)
    m = _unit(torch.randn(C, generator=g, device=device))
    basis = torch.randn(4, C, generator=g, device=device) / math.sqrt(C)

    def mix(f):
        for i in range(f.shape[0]):                      # one object / query at a time: bounded temporaries
            w = torch.randn(*f.shape[1:-1], 4, generator=g, device=device)
            c = _unit(m + spread * (w @ basis))
            f[i] = _unit(math.sqrt(shared) * c + math.sqrt(1 - shared) * f[i])

    mix(case.bank_feat)
    mix(case.q_feat)
    return case


def _plant(case, g, rows_q, rows_t, strength=0.1):
    """One random direction u per object: the query rows `rows_q` and template rows `rows_t` (all templates) get u plus
    noise; the template copies are identical across the rows of `rows_t`, the query copies across `rows_q`."""
    dev = case.q_feat.device
    o = (case.q_label - 1).to(dev)
    u = _unit(torch.randn(case.O, C, generator=g).to(dev))
    sig = (0.05 + 0.1 * torch.arange(case.T, device=dev) / case.T)[None, :, None]
    q = _unit(u[o] + strength * torch.randn(case.B, C, generator=g).to(dev) / 32)
    tm = _unit(u[:, None] + sig * torch.randn(case.O, case.T, C, generator=g).to(dev) / 32)
    for t in rows_q:
        case.q_feat[:, t] = q
        case.q_mask16[:, t] = 1
    for s in rows_t:
        case.bank_feat[:, :, s] = tm
        case.bank_mask16[:, :, s] = 1


def plant_ties(case, seed):
    g = torch.Generator().manual_seed(seed)
    for s_lo, s_hi, t in ROW_TIES:
        _plant(case, g, [t], [s_lo, s_hi])
        case.bank_mask16[:, :, t] = 1
    for t_lo, t_hi in COL_TIES:
        _plant(case, g, [t_lo, t_hi], [t_lo])
        case.bank_mask16[:, :, t_hi] = 1
    return case


def plant_cycle_pairs(case, seed):
    g = torch.Generator().manual_seed(seed)
    for t0, t1, s in CYCLE_PAIRS:
        _plant(case, g, [t0, t1], [s, t1])
    return case


def frac_masks(case, seed):
    """Every nonzero mask value replaced by one of 0.25, 0.5, 0.75, 1 (0.75 x 0.75 is where (raw sm) tm and
    raw (sm tm) round differently)."""
    g = torch.Generator().manual_seed(seed)
    levels = torch.tensor([0.25, 0.5, 0.75, 1.0])
    for m in (case.q_mask16, case.bank_mask16):
        pick = levels[torch.randint(0, 4, m.shape, generator=g)].to(m.device)
        m.copy_(torch.where(m != 0, pick, m))
    return case


def edge_masks(case):
    """Needs B >= 5 and T >= 4.  Query 0 and template 0 (every object) all zero; query 1 and template 1 only patch 0;
    query 2 only patch 137; query 3 all ones (every border patch); query 4 and template 2 a disc around the corner
    (0, 0); template 3 the border ring alone."""
    ys, xs = torch.meshgrid(torch.arange(G), torch.arange(G), indexing="ij")
    ys, xs = ys.reshape(-1), xs.reshape(-1)
    corner = ((xs ** 2 + ys ** 2) <= 49).float()
    ring = ((xs == 0) | (ys == 0) | (xs == G - 1) | (ys == G - 1)).float()
    one = lambda i: torch.nn.functional.one_hot(torch.tensor(i), P).float()
    qm, bm = case.q_mask16, case.bank_mask16
    dev = qm.device
    qm[0] = 0
    qm[1] = one(0).to(dev)
    qm[2] = one(137).to(dev)
    qm[3] = 1
    qm[4] = corner.to(dev)
    bm[:, 0] = 0
    bm[:, 1] = one(0).to(dev)
    bm[:, 2] = corner.to(dev)
    bm[:, 3] = ring.to(dev)
    return case


def unsorted_labels(B, O, seed):
    """Every object in turn, shuffled: the batch is not grouped by object."""
    lab = torch.arange(B) % O + 1
    return lab[torch.randperm(B, generator=torch.Generator().manual_seed(seed))]


def masks_of(case, shard_rank=0, shard_world=1):
    """Per query b and local template n: smask [B, T_local, 256] and tmask [B, 1, 256] (fp32 numpy)."""
    lab = (case.q_label - 1).cpu()
    sel = torch.arange(shard_rank, case.T, shard_world)
    sm = case.bank_mask16.cpu()[lab][:, sel]
    return sm.numpy().astype(np.float32), case.q_mask16.cpu()[:, None].numpy().astype(np.float32)


def cpu_tiles(case, chunk=32):
    """[B, T, 256 t, 256 s] fp32 tiles exactly as LocalSimilarity.test (matching.py:222-233) computes them on the CPU:
    the reference layout, a second F.normalize over channels, and one einsum per chunk of `chunk` queries."""
    ri = synth.to_reference_layout(case)
    out = []
    for b0 in range(0, case.B, chunk):
        tf = F.normalize(ri["tar_feat"][b0:b0 + chunk], dim=1)
        sf = F.normalize(ri["src_feats"][b0:b0 + chunk], dim=2)
        n, c = tf.shape[:2]
        tf = tf.reshape(n, c, P)
        sf = sf.reshape(n, sf.shape[1], c, P)
        out.append(torch.einsum("b c t, b n c s -> b n t s", tf, sf))
    return torch.cat(out).numpy()


def pick_knife(tiles, sm, tm, thr0, pthr, cycle=False, max_try=256):
    """A sim_threshold (and, with `cycle`, a patch_threshold) placed exactly on decisions of these tiles, which must be
    the tiles a second run with that threshold will see.  tiles [N, 256, 256], sm / tm [N, 256] (fp32 numpy).

    Candidates are the scores of records valid at (thr0, pthr).  Without `cycle` a candidate with masked products one
    ulp either side of it is preferred, then one with products on one side, then one with other products equal to it; with `cycle`, a record of a CYCLE_PAIRS row t whose back match
    is t', with patch_threshold set to that distance in fp32.  Either way the candidate is kept only if the restatement
    flips a decision at it: `<=` instead of `<` (and, for the cycle, patch_threshold one ulp lower) must change a valid
    flag.  Returns (sim_threshold, patch_threshold, populations)."""
    f32 = np.float32
    r = sim_fp64.epilogue(tiles, sm, tm, thr0, pthr)
    live = (sm[:, None, :] * tm[:, :, None]) != 0
    pop = np.sort(((tiles * sm[:, None, :]) * tm[:, :, None])[live])
    count = lambda x: np.searchsorted(pop, x, "right") - np.searchsorted(pop, x, "left")
    if cycle:
        cands = []
        for t0, t1, s in CYCLE_PAIRS:
            ok = r["valid"][:, t1] & (r["idx"][:, t1] == s)
            for i in np.nonzero(ok)[0]:
                dx, dy = f32(t0 % G - t1 % G), f32(t0 // G - t1 // G)
                cands.append((i, r["score"][i, t1], np.sqrt(dx * dx + dy * dy)))
    else:
        vals = np.unique(r["score"][r["valid"]])
        lo, hi = np.nextafter(vals, f32(-np.inf)), np.nextafter(vals, f32(np.inf))
        ne, nl, nh = count(vals), count(lo), count(hi)
        key = 4 * (np.minimum(nl, nh) > 0) + 2 * (nl + nh > 0) + (ne > 1)   # both sides, one side, duplicates
        order = np.argsort(-key, kind="stable")
        cands = [(None, vals[i], f32(pthr)) for i in order]
    for i, thr, pt in cands[:max_try]:
        sel = np.nonzero((r["score"] == thr).any(-1))[0] if i is None else np.array([i])
        a = sim_fp64.epilogue(tiles[sel], sm[sel], tm[sel], thr, pt)
        flips = [sim_fp64.epilogue(tiles[sel], sm[sel], tm[sel], thr, pt, mutation="thr_le")]
        if cycle:
            flips.append(sim_fp64.epilogue(tiles[sel], sm[sel], tm[sel], thr, np.nextafter(pt, f32(0))))
        if all((a["valid"] != b["valid"]).any() for b in flips):
            eq, dn, up = sim_fp64.ulp_neighbours(pop, thr)
            return float(thr), float(pt), dict(products_equal=eq, products_ulp_below=dn, products_ulp_above=up)
    raise AssertionError("no candidate threshold flips a decision: the planted population is not live")
