"""-m gpu parity of the native ViT forward (row a1) against the fp32 CPU restatement (oracle/port.py::DinoV2Port,
itself pinned by tests/golden/backbones.npz and cross-checked against transformers' Dinov2).  Tolerances are
floating-point: measured block by block against fp64 (tests/test_gpu_vit_fp64.py, H100 80GB HBM3 at 700 W), each ViT
block is within 4.1e-6 of the magnitude sum of its output, the 24-block x_prenorm within 8.1e-4 of the last block's
sum, and the unit-norm descriptors within 2.7e-6 absolute.  These weights have every LayerScale at 1, so the
LayerScale wiring is checked there, not here."""
import pytest
import torch

from gigapose_b200 import synth
from gigapose_b200.vit import DinoVisionTransformer
from gigapose_b200.vit_engine import NativeViT
from oracle import port

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pair(depth, seed):
    ref = port.DinoV2Port(depth=depth, seed=seed)
    mine = DinoVisionTransformer(depth=depth)
    mine.load_state_dict(ref.state_dict())
    return ref, mine.to(DEV)


@pytest.mark.parametrize("depth,tol", [(1, 2e-4), (4, 5e-4)])
def test_native_vit_blocks_match_oracle(depth, tol):
    ref, mine = _pair(depth, seed=5)
    rgb, _ = synth.make_crops(3, seed=9)
    want = ref.forward_features(rgb)["x_prenorm"]
    got = NativeViT(mine, DEV, max_crops=4).forward(rgb.to(DEV)).cpu()
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert err < tol * max(1.0, scale), f"depth {depth}: max err {err:.3e} (|x| up to {scale:.1f})"


def test_native_vit_l14_features_match_oracle_and_golden(golden_dir):
    """Full 24-block ViT-L/14 -> unit-norm patch features (ae_net.py:55-69) vs oracle and reference golden."""
    import os
    import numpy as np
    from src.models.network.ae_net import AENet
    ref, mine = _pair(24, seed=7)
    ae = AENet("dinov2_vitl14", dinov2_model=mine, descriptor_size=1024, max_batch_size=64).to(DEV)
    rgb, _ = synth.make_crops(2, seed=31)
    feat = ae(rgb.to(DEV)).cpu()                      # [2,1024,16,16]
    assert feat.shape == (2, 1024, 16, 16)
    g = np.load(os.path.join(golden_dir, "backbones.npz"))
    err = np.abs(feat[:, ::8].numpy() - g["ae_feat_sub"]).max()
    assert err < 5e-4, f"max |feature - reference golden| = {err:.3e} on unit-norm descriptors"
    assert torch.allclose(feat.norm(dim=1), torch.ones(2, 16, 16), atol=1e-5)


def test_native_vit_bf16_mode_is_close():
    ref, mine = _pair(2, seed=5)
    rgb, _ = synth.make_crops(2, seed=9)
    want = ref.forward_features(rgb)["x_prenorm"]
    got = NativeViT(mine, DEV, max_crops=2, precision="bf16").forward(rgb.to(DEV)).cpu()
    rel = ((got - want).norm() / want.norm()).item()
    assert rel < 2e-2, rel


def test_persistent_attention_over_many_crops_is_batch_invariant():
    """20 crops = 320 (crop, head) items, one attention CTA per item: more CTAs than SMs, so they run in several waves.
    The result of a crop must not depend on what else is in the batch
    (bit-identical to a 2-crop call) and must match the oracle."""
    ref, mine = _pair(2, seed=11)
    rgb, _ = synth.make_crops(20, seed=13)
    eng = NativeViT(mine, DEV, max_crops=32)
    big = eng.forward(rgb.to(DEV)).cpu()
    for i in (0, 9, 18):
        small = eng.forward(rgb[i:i + 2].to(DEV)).cpu()
        assert torch.equal(big[i:i + 2], small), i
    want = ref.forward_features(rgb[:6])["x_prenorm"]
    err = (big[:6] - want).abs().max().item()
    assert err < 3e-4 * max(1.0, want.abs().max().item()), err
