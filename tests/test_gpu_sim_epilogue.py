"""-m gpu: every decision of sim_search_kernel against the numpy restatement (tests/sim_fp64.py) applied to the
kernel's own fp32 tiles.

An engine with k = T returns every template's record through sim_candidates (the production kernel, kDebug = false);
debug_sim_tiles returns the raw tiles of the same search ([T, B sorted by object, 256, 256], the kDebug = true
instantiation).  On those tiles:
- rec_idx and rec_valid equal the restatement exactly and rec_score bit for bit, for every (query, template, patch);
- the kernel's sim_avg lies within the restatement's order-independent bar, and the top-k order equals the sort of the
  restated sim_avg wherever two templates are further apart than their bars;
- the tiles themselves stay within the fp64 tile bars (BAR_TILES of test_gpu_kernels.py for fp32_split, 2e-2 as in
  test_gpu_retrieval.py::test_similarity_tiles_against_fp64 for bf16).
Each case asserts that the population it was built for is present in the tiles.  Populations, worst sim_avg ratio to
its bar and the record differences go to $GIGAPOSE_REPORT_DIR/sim_epilogue_<case>_<precision>.json and to stdout."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gigapose_b200 import synth

import sim_cases
import sim_fp64
from helpers import engine_from_case, write_report
from test_gpu_kernels import BAR_TILES

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
BAR_TILES_BF16 = 2e-2            # one bf16 pass: test_gpu_retrieval.py::test_similarity_tiles_against_fp64
SQRT2 = float(np.sqrt(np.float32(2.0)))


def _case(B, O, T, seed, labels=None, plain=False, ties=True, mod=None, device="cpu"):
    def make():
        lab = sim_cases.unsorted_labels(B, O, seed) if labels is None else labels
        if plain:
            case = synth.make_feature_case(B=B, O=O, T=T, seed=seed, labels=lab, device=device)
        else:
            case = sim_cases.realistic(B, O, T, seed, labels=lab, device=device)
        if ties:
            sim_cases.plant_ties(case, seed + 1)
        if mod is not None:
            mod(case)
        return case
    return make


# name: (case, sim_threshold, patch_threshold, (shard rank, world), k or None for k = T, populations that must be live)
CASES = {
    "realistic_ties": (_case(9, 3, 12, 51), 0.5, 3.0, (0, 1), None, ("bulk_03_07", "row_ties", "col_ties", "invalid")),
    "b1": (_case(1, 1, 8, 52), 0.5, 3.0, (0, 1), None, ("valid", "row_ties", "col_ties")),
    "b33": (_case(33, 2, 32, 53), 0.5, 3.0, (0, 1), None, ("valid", "row_ties", "col_ties")),
    "one_query_per_object": (_case(64, 64, 4, 54, labels=torch.randperm(64, generator=torch.Generator().manual_seed(1)) + 1,
                                   device="cuda"), 0.5, 3.0, (0, 1), None, ("valid",)),
    "empty_objects": (_case(7, 5, 10, 55, labels=torch.tensor([4, 2, 4, 4, 2, 4, 2])), 0.5, 3.0, (0, 1), None, ("valid",)),
    "frac_masks": (_case(6, 2, 8, 56, mod=lambda c: sim_cases.frac_masks(c, 3)), 0.5, 3.0, (0, 1), None,
                   ("mask_075_pairs", "valid")),
    "edge_masks": (_case(6, 2, 8, 57, mod=sim_cases.edge_masks), 0.5, 3.0, (0, 1), None, ("valid",)),
    "thr_0": (_case(6, 2, 8, 58, plain=True), 0.0, 3.0, (0, 1), None, ("neg_zero", "valid")),
    "thr_neg": (_case(6, 2, 8, 58, plain=True), -0.05, 3.0, (0, 1), None, ("neg_kept", "neg_zero", "valid")),
    "thr_high": (_case(4, 2, 6, 59), 1.01, 3.0, (0, 1), None, ()),
    "pthr_0.5": (_case(6, 2, 8, 60), 0.5, 0.5, (0, 1), None, ("valid", "cycle_far")),
    "pthr_1": (_case(6, 2, 8, 60), 0.5, 1.0, (0, 1), None, ("cycle_at_pthr", "cycle_far")),
    "pthr_sqrt2": (_case(6, 2, 8, 60), 0.5, SQRT2, (0, 1), None, ("cycle_at_pthr", "cycle_far")),
    "pthr_3": (_case(6, 2, 8, 60), 0.5, 3.0, (0, 1), None, ("cycle_at_pthr", "cycle_far")),
    "pthr_30": (_case(6, 2, 8, 60), 0.5, 30.0, (0, 1), None, ("valid",)),
    "knife_thr": (_case(16, 2, 16, 61), 0.5, 3.0, (0, 1), None, ("thr_equal",)),
    "knife_cycle": (_case(8, 2, 8, 62, mod=lambda c: sim_cases.plant_cycle_pairs(c, 5)), 0.5, 3.0, (0, 1), None,
                    ("thr_equal", "cycle_at_pthr")),
    "shard_1_of_2": (_case(5, 2, 20, 63), 0.5, 3.0, (1, 2), None, ("valid", "row_ties")),
    "t576": (_case(2, 1, 576, 64, device="cuda"), 0.5, 3.0, (0, 1), 32, ("valid",)),
}


def _search(case, precision, thr, pthr, shard, k):
    """(candidate records on the CPU, tiles [B in query order, T_local, 256, 256] fp32 on the GPU)."""
    r, w = shard
    t_local = len(range(r, case.T, w))
    eng = engine_from_case(case, precision=precision, k=k or t_local, sim_threshold=thr, patch_threshold=pthr,
                           shard_rank=r, shard_world=w)
    eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1)
    cand = {n: v[0].cpu() for n, v in eng.sim_candidates().items()}          # kDebug = false
    tiles = eng.debug_sim_tiles()                                             # kDebug = true
    order = torch.argsort(case.q_label.cpu(), stable=True)
    inv = torch.empty_like(order)
    inv[order] = torch.arange(case.B)
    tiles = tiles[:, inv.to(DEV)].transpose(0, 1).contiguous()
    torch.cuda.synchronize()
    del eng
    return cand, tiles


def _tile_error(case, tiles, shard):
    """max |tile - fp64 einsum of the normalised descriptors| over every tile."""
    r, w = shard
    lab = (case.q_label - 1).to(DEV)
    q = F.normalize(case.q_feat.to(DEV, torch.float64), dim=-1)
    err = 0.0
    for i, n in enumerate(range(r, case.T, w)):
        bank = F.normalize(case.bank_feat[:, n].to(DEV, torch.float64), dim=-1)[lab]
        err = max(err, float((tiles[:, i].double() - torch.einsum("btc,bsc->bts", q, bank)).abs().max()))
    return err


def _populations(tiles, sm, tm, thr, pthr, r):
    """Counts of the inputs each case is built to exercise (tiles [N,256,256], sm/tm [N,256], r: the restatement)."""
    f32 = np.float32
    live = (sm[:, None, :] * tm[:, :, None]) != 0
    v = (tiles * sm[:, None, :]) * tm[:, :, None]
    kept = np.where(v < f32(thr), f32(0), v)
    vals = v[live]
    eq, dn, up = sim_fp64.ulp_neighbours(vals, thr)
    out = dict(products=int(vals.size), bulk_03_07=int(((vals > 0.3) & (vals < 0.7)).sum()),
               valid=int(r["valid"].sum()),
               invalid=int((~r["valid"] & (np.take_along_axis(sm, r["idx"], -1) * tm != 0)).sum()),
               neg_kept=int(((kept < 0) & live).sum()), neg_zero=int((kept.view(np.int32) == np.int32(-2 ** 31)).sum()),
               thr_equal=eq, thr_ulp_below=dn, thr_ulp_above=up,
               mask_075_pairs=int(((sm[:, None, :] == 0.75) & (tm[:, :, None] == 0.75)).sum()))
    # exact ties and near-ties (the two largest values within 4 ulps, not equal) of nonzero row / column maxima
    for name, ax in (("row", -1), ("col", -2)):
        top2 = -np.partition(-kept, 1, axis=ax).take([0, 1], axis=ax)
        a, b = top2.take(0, axis=ax), top2.take(1, axis=ax)
        nz = a != 0
        ulps = np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))
        out[name + "_ties"] = int((nz & (a == b)).sum())
        out[name + "_near_ties"] = int((nz & (ulps > 0) & (ulps <= 4)).sum())
    t = np.arange(256)
    back = np.take_along_axis(r["idx_src2tar"], r["idx"], -1)
    dx, dy = (back % 16 - t % 16).astype(f32), (back // 16 - t // 16).astype(f32)
    dist = np.sqrt(dx * dx + dy * dy)
    decided = (r["score"] >= f32(thr)) & (np.take_along_axis(sm, r["idx"], -1) * tm != 0)
    out["cycle_at_pthr"] = int((decided & (dist == f32(pthr))).sum())
    out["cycle_far"] = int((decided & (dist > f32(pthr))).sum())
    return out


def _check(name, precision, case, cand, tiles, thr, pthr, shard, need, extra=None):
    r_, w = shard
    B, k = cand["id"].shape
    t_local = tiles.shape[1]
    sm, tm = sim_cases.masks_of(case, r_, w)
    tile_err = _tile_error(case, tiles, shard)
    ids = cand["id"].numpy().astype(np.int64)
    scores = cand["score"].numpy()
    local = (ids - r_) // w
    assert np.all((ids - r_) % w == 0) and np.all((local >= 0) & (local < t_local)), "global template ids"
    diff = dict(idx=0, valid=0, score=0)
    pops, worst, order_bad = None, 0.0, 0
    for b0 in range(0, B, 8):                                      # a few queries at a time: bounded host memory
        tl = tiles[b0:b0 + 8].cpu().numpy()
        n_q = tl.shape[0]
        r = sim_fp64.epilogue(tl, sm[b0:b0 + 8], tm[b0:b0 + 8], thr, pthr)
        flat = lambda x: x.reshape(n_q * t_local, *x.shape[2:])
        p = _populations(flat(tl), flat(np.broadcast_to(sm[b0:b0 + 8], (n_q, t_local, 256))),
                         flat(np.broadcast_to(tm[b0:b0 + 8], (n_q, t_local, 256))), thr, pthr,
                         {key: flat(v) for key, v in r.items() if v.ndim == 3})
        pops = p if pops is None else {key: pops[key] + v for key, v in p.items()}
        del tl
        for j in range(n_q):
            b = b0 + j
            n = local[b]
            # sim_topk's own order: score descending, then template id ascending
            s = scores[b]
            assert np.all((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (ids[b, :-1] < ids[b, 1:]))), f"query {b}: order"
            diff["idx"] += int((cand["idx"][b].numpy() != r["idx"][j, n]).sum())
            diff["valid"] += int((cand["valid"][b].numpy().astype(bool) != r["valid"][j, n]).sum())
            diff["score"] += int((cand["pts_score"][b].numpy().view(np.int32) !=
                                  r["score"][j, n].astype(np.float32).view(np.int32)).sum())
            bar = r["sim_avg_bar"][j, n]
            err = np.abs(s.astype(np.float64) - r["sim_avg"][j, n])
            assert np.all(err <= bar), f"query {b}: sim_avg outside its bar: {err.max():.3e} vs {bar[np.argmax(err - bar)]:.3e}"
            worst = max(worst, float(np.max(np.where(bar > 0, err / np.where(bar > 0, bar, 1), 0))))
            order_bad += len(sim_fp64.topk_consistent(n, r["sim_avg"][j], r["sim_avg_bar"][j]))
    report = dict(case=name, precision=precision, B=B, T=t_local, k=k, sim_threshold=thr, patch_threshold=pthr,
                  shard=list(shard), record_differences=diff, sim_avg_worst_ratio_to_bar=worst,
                  topk_order_violations=order_bad, tile_err_fp64=tile_err, populations=pops, **(extra or {}))
    write_report(f"sim_epilogue_{name}_{precision}.json", report)
    print(f"\n{name} {precision}: differences {diff}, sim_avg/bar {worst:.3f}, tile err {tile_err:.2e}\n  {pops}")
    assert diff == dict(idx=0, valid=0, score=0), f"{name} {precision}: kernel records differ from the restatement: {diff}"
    assert order_bad == 0, f"{name} {precision}: top-k order contradicts the restated sim_avg at {order_bad} places"
    assert tile_err < (BAR_TILES if precision == "fp32_split" else BAR_TILES_BF16), f"tiles vs fp64: {tile_err:.3e}"
    for key in need:
        assert pops[key] > 0, f"{name} {precision}: planted population {key} is empty: {pops}"
    return pops


@pytest.mark.parametrize("precision", ["fp32_split", "bf16"])
@pytest.mark.parametrize("name", list(CASES))
def test_epilogue_matches_restatement(name, precision):
    make, thr, pthr, shard, k, need = CASES[name]
    case = make()
    cand, tiles = _search(case, precision, thr, pthr, shard, k)
    extra = None
    if name.startswith("knife"):
        # thresholds placed on this precision's own tiles, then the same case searched again with them
        flat = tiles.reshape(-1, 256, 256).cpu().numpy()
        sm, tm = sim_cases.masks_of(case, *shard)
        thr, pthr, picked = sim_cases.pick_knife(flat, sm.reshape(-1, 256),
                                                 np.broadcast_to(tm, sm.shape).reshape(-1, 256), thr, pthr,
                                                 cycle=name == "knife_cycle")
        del flat
        first = tiles
        cand, tiles = _search(case, precision, thr, pthr, shard, k)
        assert torch.equal(first.view(torch.int32), tiles.view(torch.int32)), "the second search's tiles differ"
        del first
        extra = dict(picked=picked)
    pops = _check(name, precision, case, cand, tiles, thr, pthr, shard, need, extra)
    if name == "thr_high":
        assert pops["valid"] == 0 and bool((cand["score"] == 0).all())
    if name == "edge_masks":
        assert bool((cand["score"][0] == 0).all()) and not bool(cand["valid"][0].any()), "all-zero query mask"
