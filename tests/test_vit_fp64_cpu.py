"""The fp64 ViT evaluator (tests/vit_fp64.py) on the CPU: it agrees with the fp32 restatement `port.DinoV2Port` block
by block on `realistic_weights`, every named mutation of the block moves its output far beyond that agreement, and
`_params_in_abi_order` puts each block's LayerScales where gp_vit_create reads them.

Errors are normalised per element by the magnitude sum of `vit_fp64.block`.  The port's blocks run in fp32 on the
evaluator's own input rounded to fp32, so each block's error is its own; the largest measured was 1.8e-7 (x86-64,
torch 2.11), and BAR_FP32 is about 4x that."""
import pytest
import torch

import vit_fp64 as V
from gigapose_b200 import synth
from gigapose_b200.vit_engine import _params_in_abi_order
from oracle import port

BAR_FP32 = 7e-7                 # one block in fp32 against fp64, of the magnitude sum          [1.8e-7]
BAR_TABLE = 1.5e-4              # the host's fp32 bicubic table, of sum |w_y| |w_x| |pe|          [3.8e-5]
TANH_ALPHA = 1e-4               # see test_every_mutation_moves_the_output_far_beyond_fp32  [2.7e-5]


@pytest.fixture(scope="module")
def depth2():
    m = V.realistic_weights(2, seed=3)
    ref = port.DinoV2Port(depth=2, seed=None)
    ref.load_state_dict(m.state_dict())
    rgb, _ = synth.make_crops(1, seed=9)
    rgb[:, :, :112, :112] = 0.0                     # a masked-out quadrant: tokens b + pos, of variance ~5e-5
    with torch.no_grad():
        x, _ = V.embed(m, rgb)
        ps = [V.block_params(m, i) for i in range(2)]
        xs, dens, port_out = [x], [], []
        for i in range(2):
            y, d = V.block(xs[-1], ps[i])
            port_out.append(ref.blocks[i](xs[-1].float()))
            xs.append(y)
            dens.append(d)
    return m, ref, rgb, ps, xs, dens, port_out


def test_evaluator_matches_fp32_port_block_by_block(depth2):
    m, ref, rgb, ps, xs, dens, port_out = depth2
    errs = [V.nerr(port_out[i], xs[i + 1], dens[i]) for i in range(2)]
    assert max(errs) < BAR_FP32, errs
    # and end to end: forward_features agrees within the fp32 rounding of the host's positional table, whose bicubic
    # weights and source coordinates are computed in fp32
    with torch.no_grad():
        want = ref.forward_features(rgb)["x_prenorm"]
        host = m.interpolated_pos_embed(V.GRID, V.GRID)[0]
    pos, pos_den = V.pos_table(m)
    assert V.nerr(host, pos, pos_den) < BAR_TABLE
    assert V.nerr(want, V.forward(m, rgb), dens[1]) < BAR_TABLE


def test_every_mutation_moves_the_output_far_beyond_fp32(depth2):
    """Each mutation, applied to the same fp64 input, misses the evaluator's block output by >= 100x BAR_FP32 on some
    block, and the LayerScale mutations on every block where they apply.

    tanh-GELU is the exception: tanh and erf GELU differ by at most 4.7e-4 (at x = -2.7), and fc2 sums that difference
    over 4096 hidden units of random sign, so the output moves by ~2.5e-5 of its magnitude sum (~35x BAR_FP32) whatever
    the weights.  It is detected by projection instead: the fp32 port's error e = port - fp64 has, along the mutation's
    displacement D = mutated - fp64, the coefficient <e, D> / <D, D>, which is 1 for a port that computed tanh-GELU and
    at most 2.7e-5 for this one.  The kernel test of the GELU epilogue pins the form directly."""
    _, _, _, ps, xs, dens, port_out = depth2
    moved = {}
    for name, (needs_next, f) in V.MUTATIONS.items():
        moved[name] = [V.nerr(f(xs[i], ps[i], ps[i + 1] if i + 1 < 2 else None), xs[i + 1], dens[i])
                       for i in range(2 if not needs_next else 1)]
    gammas = ("ls1<->ls2", "gammas of block k+1", "gamma=1")
    weak = {k: v for k, v in moved.items() if k != "tanh-GELU" and (min(v) if k in gammas else max(v)) < 100 * BAR_FP32}
    assert not weak, weak
    assert min(moved["tanh-GELU"]) > 10 * BAR_FP32, moved["tanh-GELU"]
    for i in range(2):
        D = V.MUTATIONS["tanh-GELU"][1](xs[i], ps[i], None) - xs[i + 1]
        e = port_out[i].double() - xs[i + 1]
        alpha = float((e * D).sum() / (D * D).sum())
        assert abs(alpha) < TANH_ALPHA, (i, alpha)


def test_realistic_weights_have_distinct_layerscales_and_planted_channels():
    m = V.realistic_weights(3, seed=3)
    g = [(b.ls1.gamma.detach(), b.ls2.gamma.detach()) for b in m.blocks]
    for i, (g1, g2) in enumerate(g):
        assert not torch.equal(g1, g2) and not torch.equal(g1, g[(i + 1) % 3][0]) and not torch.equal(g2, g[(i + 1) % 3][1])
        for t in (g1, g2):
            assert float(t.abs().min()) >= 1e-3 * (1 - 1e-6) and float(t.abs().max()) <= 1.0
            assert 0.3 < float((t < 0).float().mean()) < 0.7
    pos, _ = V.pos_table(m)
    big = (pos[:, list(V.MASSIVE_CHANNELS)].abs() > 100).all(-1)
    assert bool(big[0]) and int(big[1:].sum()) >= len(V.MASSIVE_POSITIONS), int(big[1:].sum())


def test_abi_order_puts_each_blocks_layerscales_where_gp_vit_create_reads_them():
    """include/gigapose_b200.h: 4 + 14 depth pointers, per block in upstream state-dict order; gp_vit_create reads
    ls1.gamma at 4 + 14 i + 6 and ls2.gamma at 4 + 14 i + 13."""
    m = V.realistic_weights(3, seed=4)
    w = _params_in_abi_order(m, "cpu")
    assert len(w) == 4 + 14 * 3
    for i, blk in enumerate(m.blocks):
        named = dict(blk.named_parameters())
        for j, name in enumerate(V.BLOCK_NAMES):
            assert torch.equal(w[4 + 14 * i + j], named[name].detach()), (i, name)
        assert w[4 + 14 * i + 6].data_ptr() == blk.ls1.gamma.data_ptr()
        assert w[4 + 14 * i + 13].data_ptr() == blk.ls2.gamma.data_ptr()
