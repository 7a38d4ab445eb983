"""The similarity-epilogue restatement (tests/sim_fp64.py) pinned on the CPU: it equals oracle/port.py's
similarity_search and the unmodified reference LocalSimilarity given the same fp32 einsum, and each of its named
mutations changes an output on these cases, so the GPU test that applies it to the kernel's tiles would notice them."""
import functools

import numpy as np
import pytest
import torch

from gigapose_b200 import synth
from oracle import port, ref_import

import sim_cases
import sim_fp64
from helpers import write_report

SQRT2 = float(np.sqrt(np.float32(2.0)))


def _golden(seed, B, O, T):
    return lambda: (synth.make_feature_case(B=B, O=O, T=T, seed=seed), 0.5, 3.0)


def _real(B=5, O=2, T=6, seed=41, thr=0.5, pthr=3.0, plain=False, mod=None):
    def make():
        labels = sim_cases.unsorted_labels(B, O, seed)
        if plain:
            case = synth.make_feature_case(B=B, O=O, T=T, seed=seed, labels=labels)
        else:
            case = sim_cases.realistic(B, O, T, seed, labels=labels)
        sim_cases.plant_ties(case, seed + 1)
        if mod is not None:
            mod(case)
        return case, thr, pthr
    return make


CASES = {
    # the retrieval golden fixtures' inputs (oracle/make_golden.py RETRIEVAL_CASES)
    "golden_c1": _golden(11, 1, 1, 16),
    "golden_small": _golden(12, 6, 3, 24),
    "realistic_ties": _real(),
    "frac_masks": _real(B=4, T=5, seed=43, mod=lambda c: sim_cases.frac_masks(c, 7)),
    "edge_masks": _real(B=6, T=5, seed=44, mod=sim_cases.edge_masks),
    "thr_0": _real(B=4, T=4, seed=45, thr=0.0, plain=True),
    "thr_neg": _real(B=4, T=4, seed=45, thr=-0.05, plain=True),
    "thr_high": _real(B=3, T=4, seed=46, thr=1.01),
    "pthr_half": _real(B=3, T=4, seed=47, pthr=0.5),
    "pthr_1": _real(B=3, T=4, seed=47, pthr=1.0),
    "pthr_sqrt2": _real(B=3, T=4, seed=47, pthr=SQRT2),
    "pthr_30": _real(B=3, T=4, seed=47, pthr=30.0),
    "knife_thr": _real(B=6, T=8, seed=48),
    "knife_cycle": _real(B=4, T=6, seed=49, mod=lambda c: sim_cases.plant_cycle_pairs(c, 9)),
}


@functools.lru_cache(maxsize=None)
def prepared(name):
    """(case, tiles [B,T,256,256], smask [B,T,256], tmask [B,1,256], sim_threshold, patch_threshold, populations)."""
    case, thr, pthr = CASES[name]()
    tiles = sim_cases.cpu_tiles(case)
    sm, tm = sim_cases.masks_of(case)
    pops = {}
    if name.startswith("knife"):
        flat = tiles.reshape(-1, 256, 256)
        sm_f = sm.reshape(-1, 256)
        tm_f = np.broadcast_to(tm, sm.shape).reshape(-1, 256)
        thr, pthr, pops = sim_cases.pick_knife(flat, sm_f, tm_f, thr, pthr, cycle=name == "knife_cycle")
    return case, tiles, sm, tm, thr, pthr, pops


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_equals_port(name):
    """Every per-patch output bit for bit, mask_all exactly, sim_avg within its bar of port's fp32 sum."""
    case, tiles, sm, tm, thr, pthr, _ = prepared(name)
    ri = synth.to_reference_layout(case)
    ref = port.similarity_search(ri["src_feats"], ri["tar_feat"], ri["src_masks"], ri["tar_mask"], k=min(5, case.T),
                                 sim_threshold=thr, patch_threshold=pthr, return_intermediates=True)
    r = sim_fp64.epilogue(tiles, sm, tm, thr, pthr)
    assert np.array_equal(r["idx"], ref["idx_tar2src"].numpy())
    assert np.array_equal(r["idx_src2tar"], ref["idx_src2tar"].numpy())
    assert np.array_equal(_bits(r["score"]), _bits(ref["score_tar2src"].numpy()))
    assert np.array_equal(_bits(r["score_src2tar"]), _bits(ref["score_src2tar"].numpy()))
    assert np.array_equal(r["mask_all"], ref["mask_all"].numpy())
    err = np.abs(ref["sim_avg"].numpy().astype(np.float64) - r["sim_avg"])
    assert np.all(err <= r["sim_avg_bar"]), float((err / np.maximum(r["sim_avg_bar"], 1e-300)).max())


def _ref_module(thr, pthr, k):
    if not ref_import.available():
        pytest.skip("reference tree not present")
    return ref_import.load().LocalSimilarity(k=k, sim_threshold=thr, patch_threshold=pthr)


@pytest.mark.parametrize("name", ["golden_small", "realistic_ties", "frac_masks", "edge_masks", "thr_neg",
                                  "knife_thr", "knife_cycle"])
def test_restatement_equals_reference_live(name):
    """LocalSimilarity.test with k = T returns every template's record: each one equals the restatement (score_pts bit
    for bit, the -1 pattern of tar_pts / src_pts and the matched patch exactly), score_src is within the bar and the
    order agrees within the bars.  find_consistency_patches on the restated maxima equals mask_cycle."""
    case, tiles, sm, tm, thr, pthr, _ = prepared(name)
    mod = _ref_module(thr, pthr, case.T)
    ri = synth.to_reference_layout(case)
    with torch.no_grad():
        out = mod.test(ri["src_feats"], ri["tar_feat"], ri["src_masks"], ri["tar_mask"])
    r = sim_fp64.epilogue(tiles, sm, tm, thr, pthr)
    ids = out.id_src.numpy()
    for b in range(case.B):
        assert not sim_fp64.topk_consistent(ids[b], r["sim_avg"][b], r["sim_avg_bar"][b])
        err = np.abs(out.score_src[b].numpy() - r["sim_avg"][b, ids[b]])
        assert np.all(err <= r["sim_avg_bar"][b, ids[b]])
        assert np.array_equal(_bits(out.score_pts[b].numpy()), _bits(r["score"][b, ids[b]]))
        valid = r["valid"][b, ids[b]]
        src = out.src_pts[b].numpy()
        assert np.array_equal(src[..., 0] >= 0, valid) and np.array_equal(out.tar_pts[b].numpy()[..., 0] >= 0, valid)
        idx = r["idx"][b, ids[b]]
        assert np.array_equal(src[..., 0][valid], (idx % 16)[valid]) and np.array_equal(src[..., 1][valid], (idx // 16)[valid])
    cyc = mod.find_consistency_patches(sim_src2tar=torch.from_numpy(r["score_src2tar"]),
                                       idx_src2tar=torch.from_numpy(r["idx_src2tar"]), idx_tar2src=torch.from_numpy(r["idx"]))
    assert np.array_equal(cyc.numpy(), r["mask_cycle"])


def _differences(a, b):
    """Output entries of restatement b that differ from a: records, scores, sim_avg beyond the two bars, mask_cycle."""
    over = np.abs(a["sim_avg"] - b["sim_avg"]) > a["sim_avg_bar"] + b["sim_avg_bar"]
    return dict(idx=int((a["idx"] != b["idx"]).sum()), valid=int((a["valid"] != b["valid"]).sum()),
                score=int((_bits(a["score"]) != _bits(b["score"])).sum()), sim_avg=int(over.sum()),
                mask_cycle=int((a["mask_cycle"] != b["mask_cycle"]).sum()))


@pytest.mark.parametrize("mutation", sim_fp64.MUTATIONS)
def test_every_mutation_changes_an_output(mutation):
    """Each mutation changes a record (idx, valid, score bits) or a sim_avg by more than the bars on these cases; the
    counts per case are printed.  `cycle_no_sim` can only change mask_cycle: score_src2tar[idx] >= score, so
    score >= thr already implies it and mask_all cannot move (see sim_fp64)."""
    total = dict(idx=0, valid=0, score=0, sim_avg=0, mask_cycle=0)
    per_case = {}
    for name in CASES:
        _, tiles, sm, tm, thr, pthr, _ = prepared(name)
        a = sim_fp64.epilogue(tiles, sm, tm, thr, pthr)
        b = sim_fp64.epilogue(tiles, sm, tm, thr, pthr, mutation=mutation)
        d = _differences(a, b)
        if any(d.values()):
            print(f"{mutation:13s} {name:15s} {d}")
            per_case[name] = d
        for k, v in d.items():
            total[k] += v
    write_report(f"sim_fp64_mutation_{mutation}.json", dict(total=total, cases=per_case))
    if mutation == "cycle_no_sim":
        assert total["mask_cycle"] > 0 and total["idx"] + total["valid"] + total["score"] + total["sim_avg"] == 0, total
    else:
        assert total["idx"] + total["valid"] + total["score"] + total["sim_avg"] > 0, total


def test_knife_cases_are_live():
    """The knife-edge thresholds sit on products of the tiles: some equal thr, some one ulp from it."""
    for name in ("knife_thr", "knife_cycle"):
        *_, thr, pthr, pops = prepared(name)
        print(name, thr, pthr, pops)
        assert pops["products_equal"] >= 1
    assert prepared("knife_thr")[-1]["products_ulp_below"] + prepared("knife_thr")[-1]["products_ulp_above"] >= 1


def test_bar_covers_any_summation_order():
    """The sim_avg bar against fp32 sums of one record in forward, reverse, pairwise and strided orders."""
    _, tiles, sm, tm, thr, pthr, _ = prepared("frac_masks")
    r = sim_fp64.epilogue(tiles, sm, tm, thr, pthr)
    x = (r["score"] * r["mask_all"]).reshape(-1, 256).astype(np.float32)
    want, bar = r["sim_avg"].reshape(-1), r["sim_avg_bar"].reshape(-1)
    has = r["mask_all"].reshape(-1, 256).astype(np.float64).sum(-1) > 0

    def seq(v):
        s = np.float32(0)
        for e in v:
            s = np.float32(s + e)
        return s

    def pairwise(v):
        while len(v) > 1:
            v = (v[0::2] + v[1::2]).astype(np.float32)
        return v[0]

    for order in (lambda v: v, lambda v: v[::-1], lambda v: v.reshape(8, 32).T.reshape(-1)):
        got = np.array([seq(order(v)) for v in x], dtype=np.float32) / np.float32(256)
        assert np.all(np.abs(np.where(has, got, 0) - want) <= bar)
    got = np.array([pairwise(v) for v in x], dtype=np.float32) / np.float32(256)
    assert np.all(np.abs(np.where(has, got, 0) - want) <= bar)
