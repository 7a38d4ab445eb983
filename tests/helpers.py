"""Shared helpers for the GPU parity tests: load a synthetic FeatureCase into an Engine, run the oracle."""
from __future__ import annotations

import torch

from gigapose_b200 import synth
from gigapose_b200.engine import Engine

INT_KEYS = ["id_src", "tar_pts", "src_pts", "idx_failed", "ransac_scores", "ransac_src_pts", "ransac_tar_pts"]
FLOAT_KEYS = ["score_src", "score_pts", "relScale", "relInplane", "M", "scores", "pred_poses"]


def engine_from_case(case: synth.FeatureCase, device="cuda:0", precision="fp32_split", regressor=None,
                     shard_rank=0, shard_world=1, max_batch=None, **cfg) -> Engine:
    """Loads the (already unit-norm, patch-major) synthetic bank; the kernel applies the matching-time
    normalisation (matching.py:229), i.e. norm_passes=1, exactly like the oracle does on the same tensors.
    `cfg`: further Engine settings (sim_threshold, ...)."""
    local = list(range(shard_rank, case.T, shard_world))
    eng = Engine(case.O, len(local), max_batch or case.B, device=device, precision=precision,
                 shard_rank=shard_rank, shard_world=shard_world, num_templates_global=case.T, **cfg)
    sel = torch.tensor(local)
    for o in range(case.O):
        eng.bank_write(o, 0, case.bank_feat[o, sel], case.bank_mask16[o, sel].reshape(-1, 16, 16),
                       ist_feat=case.bank_ist[o, sel], norm_passes=1)
    eng.set_poses(case.bank_K, case.bank_M, case.bank_poses)
    if regressor is not None:
        eng.set_ist_weights(regressor)
    return eng


def run_engine(eng: Engine, case: synth.FeatureCase):
    return eng.retrieve(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1, case.q_ist, case.q_K,
                        case.q_M, norm_passes=1)


def cpu(d):
    return {k: v.detach().cpu() for k, v in d.items()}


def reference_slice(case: synth.FeatureCase, sel):
    """`synth.to_reference_layout` for the queries `sel` only (the full layout gathers 170 MB per query, so the
    BASELINE-sized cases are checked on slices).  Works for cases generated on the GPU: the slice is moved to the CPU."""
    sel = torch.as_tensor(sel, dtype=torch.long)
    lab = (case.q_label.cpu()[sel] - 1)
    dev = case.bank_feat.device
    n, T = len(sel), case.T
    src_feats = case.bank_feat[lab.to(dev)].cpu().permute(0, 1, 3, 2).reshape(n, T, synth.C_AE, 16, 16).contiguous()
    tar_feat = case.q_feat[sel.to(dev)].cpu().permute(0, 2, 1).reshape(n, synth.C_AE, 16, 16).contiguous()
    c = lambda t: t.cpu()
    return dict(
        src_feats=src_feats, tar_feat=tar_feat,
        src_masks=synth.mask16_to_224(c(case.bank_mask16)[lab]), tar_mask=synth.mask16_to_224(c(case.q_mask16)[sel]),
        src_ist=case.bank_ist[lab.to(dev)].cpu(), tar_ist=case.q_ist[sel.to(dev)].cpu(),
        tar_label=c(case.q_label)[sel], tar_K=c(case.q_K)[sel], tar_M=c(case.q_M)[sel],
        template_K=c(case.bank_K), template_Ms=c(case.bank_M), template_poses=c(case.bank_poses),
    )


def assert_chain_equal(out, ref, sel=None, pose_tol=1e-3, tag=""):
    """Every output of rows a4-a9: integer tensors bit-exact, floats within the stated tolerances, pose <= 1e-3
    (BASELINE.json north_star; translation error relative to max(|t|, 1))."""
    pick = (lambda v: v) if sel is None else (lambda v: v[torch.as_tensor(sel, dtype=torch.long)])
    for k in INT_KEYS:
        got = pick(out[k])
        assert torch.equal(got.to(ref[k].dtype), ref[k]), f"{tag}{k}: {(got.to(ref[k].dtype) != ref[k]).sum().item()} entries differ"
    assert torch.allclose(pick(out["score_src"]), ref["score_src"], atol=2e-6), tag + "score_src"
    assert torch.allclose(pick(out["score_pts"]), ref["score_pts"], atol=5e-6), tag + "score_pts"
    assert torch.allclose(pick(out["relScale"]), ref["relScale"], atol=1e-4, rtol=1e-5), tag + "relScale"
    assert torch.allclose(pick(out["relInplane"]), ref["relInplane"], atol=1e-4, rtol=1e-5), tag + "relInplane"
    assert torch.allclose(pick(out["M"]), ref["M"], atol=2e-3, rtol=1e-5), tag + "M"
    assert torch.equal(pick(out["scores"]), ref["scores"]), tag + "scores"
    err = (pick(out["pred_poses"]) - ref["pred_poses"]).abs()
    err[..., :3, 3] /= ref["pred_poses"][..., :3, 3].abs().clamp(min=1.0)
    assert float(err.max()) < pose_tol, f"{tag}pose error {float(err.max()):.3e}"


def write_report(name, payload):
    """Parity reports (flip counts etc.) as JSON under $GIGAPOSE_REPORT_DIR; nothing is written when it is unset."""
    import json
    import os
    out = os.environ.get("GIGAPOSE_REPORT_DIR")
    if not out:
        return
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, name), "w") as f:
        json.dump(payload, f, indent=1, sort_keys=True)
