"""The fp64 IST evaluator (tests/ist_fp64.py) on the CPU: it agrees with `port.ISTBackbonePort` and
`port.RegressorPort` run in float64, `realistic_trunk` has the properties it plants, every mutated BatchNorm fold moves
the trunk far beyond the GPU bars on those weights (while the two quiet ones stay inside the bar of
test_gpu_ist_trunk.py on the statistics the older tests use), the RANSAC margin covers every decision a bounded change
of the regressor outputs can flip, and the fp64 decisions equal port.ransac's wherever no decision is inside its
margin."""
import copy
import math

import numpy as np
import pytest
import torch

import ist_fp64 as I
from gigapose_b200 import synth
from oracle import port
from test_gpu_ist_fp64 import BAR_CHAIN, BAR_CONV

OLD_TRUNK_BAR = 3e-4            # test_gpu_ist_trunk.py: the final map within 3e-4 of its largest value
EXACT = 1e-12                   # two fp64 evaluations of the same formula, of the magnitude


@pytest.fixture(scope="module")
def trunk():
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    net = I.resnet(I.realistic_trunk(0))
    rgb, _ = synth.make_crops(1, seed=5)
    x = torch.cat([rgb, torch.zeros_like(rgb)])            # a textured crop and an all-zero crop
    with torch.no_grad():
        acts, dens = I.forward(net, x)
    return net, x, acts, dens


def test_trunk_evaluator_matches_the_port_in_float64(trunk):
    net, x, acts, dens = trunk
    ref = port.ISTBackbonePort(seed=None)
    ref.load_state_dict(net.state_dict())
    with torch.no_grad():
        want = ref.double()(x.double())
    assert I.nerr(want, acts[-1], dens[-1]) < EXACT


def test_regressor_evaluator_matches_the_port_in_float64(trunk):
    net, x, acts, dens = trunk
    reg = I.realistic_regressor(5, acts[-1])
    reg64 = copy.deepcopy(reg).double()
    f = acts[-1].flatten(2)
    g = torch.Generator().manual_seed(1)
    rows = torch.cat([f[0, :, torch.randint(0, 256, (300,), generator=g)].T,
                      f[1, :, torch.randint(0, 256, (300,), generator=g)].T], 1)
    (s, sden), (c, cden) = I.regressor(reg, rows)
    with torch.no_grad():
        assert I.nerr(reg64.scale_predictor(rows), s, sden) < EXACT
        assert I.nerr(reg64.inplane_predictor(rows), c, cden) < EXACT
    # and its outputs are where realistic_regressor puts them, on the zero crop's rows too
    assert float(((s > 0.5) & (s < 2)).double().mean()) > 0.9
    assert float(c.norm(dim=1).min()) > 0.8 and 0.15 < float(c[:, 1].mean()) < 0.45
    # the Lipschitz bound holds for a random perturbation
    d = 1e-3 * torch.rand(rows.shape, generator=g, dtype=torch.float64)
    e = d * torch.sign(torch.randn(rows.shape, generator=g, dtype=torch.float64))
    (s2, _), (c2, _) = I.regressor(reg, rows + e)
    ls, lc = I.lipschitz(reg, d)
    assert bool(((s2 - s).abs() <= ls).all()) and bool(((c2 - c).abs() <= lc).all())


def test_realistic_trunk_has_its_planted_properties(trunk):
    net, x, acts, dens = trunk
    bns = [s.bn for s in I.schedule(net) if s.bn is not None]
    assert len(bns) == 20
    dead = I._dead_channels(net)
    assert all(len(d) == I.DEAD_PER_LAYER for d in dead), [len(d) for d in dead]
    var = torch.cat([bn.running_var for bn in bns])
    assert float(var.min()) >= I.DEAD_VAR[0] * (1 - 1e-6) and float(var.max()) < 10
    assert int((var <= 2e-4).sum()) >= 10                  # the variance reaches 1e-4
    gam = torch.cat([bn.weight.detach() for bn in bns])
    assert 0.1 < float((gam < 0).double().mean()) < 0.2
    assert int((gam.abs() < 1e-3).sum()) >= 20 and float(gam.abs().max()) <= 1.5
    z = torch.cat([(bn.running_mean / bn.running_var.sqrt()).abs() for bn in bns])
    assert int((z >= 2).sum()) >= 100                      # running means several sigma from 0
    for a in acts[1:]:                                     # O(1) activations through all 21 layers, on both crops
        assert bool(torch.isfinite(a).all())
        assert 1 < float(a.abs().max()) < 100, float(a.abs().max())
    assert float(acts[-1][1].abs().max()) > 1               # the zero crop does not collapse to 0


def test_every_mutated_fold_moves_the_trunk_far_beyond_the_gpu_bars(trunk):
    """Each mutated fold, in fp64 on the same crops, moves every BatchNorm layer's output (from the same input) by
    >= 50x BAR_CONV and the final map by >= 100x BAR_CHAIN, normalised by the evaluator's magnitudes."""
    net, x, acts, dens = trunk
    sched = I.schedule(net)
    with torch.no_grad():
        for name, fold in I.MUTATED_FOLDS.items():
            per = [I.nerr(I.layer(s, acts, fold=fold)[0], acts[i], dens[i]) for i, s in enumerate(sched, 1)]
            final = I.forward(net, x, fold=fold)[0][-1]
            moved = I.nerr(final, acts[-1], dens[-1])
            assert min(per[:20]) >= 50 * BAR_CONV, (name, min(per[:20]))
            assert per[20] == 0.0                          # the output convolution has no BatchNorm
            assert moved >= 100 * BAR_CHAIN, (name, moved)
        # and the correct fold, evaluated the same way, is exact
        fold = I._folder()
        per = [I.nerr(I.layer(s, acts, fold=fold)[0], acts[i], dens[i]) for i, s in enumerate(sched, 1)]
        assert max(per) < 1e-6, max(per)                   # fp32 folded weights


@pytest.mark.parametrize("stats", ["test_gpu_ist_trunk", "port"])
def test_quiet_folds_stay_inside_the_older_bars(stats):
    """On the BatchNorm statistics the older tests use -- variances uniform in [0.5, 1.5] (test_gpu_ist_trunk.py,
    test_gpu_encoder_kernels.py) or in [1.0, 1.2] (port.ISTBackbonePort, test_gpu_chain_parity.py) -- dropping eps or
    using 1e-6 moves the final map by less than 3e-4 of its largest value, the bar of test_gpu_ist_trunk.py.
    test_gpu_encoder_kernels.py builds its reference from the host's folded filters, so no fold mistake can show
    there, and test_gpu_chain_parity.py compares the trunk only through the regressor at 1e-3 of its range.  Only
    trained-like statistics expose them (test_every_mutated_fold_moves_the_trunk_far_beyond_the_gpu_bars)."""
    if stats == "port":
        net = I.resnet(port.ISTBackbonePort().state_dict())
    else:
        torch.manual_seed(0)
        net = I.resnet()
        g = torch.Generator().manual_seed(0)
        with torch.no_grad():
            for m in net.modules():
                if isinstance(m, torch.nn.BatchNorm2d):
                    n = m.num_features
                    m.running_mean.copy_(0.2 * torch.randn(n, generator=g))
                    m.running_var.copy_(0.5 + torch.rand(n, generator=g))
                    m.weight.copy_(0.5 + torch.rand(n, generator=g))
                    m.bias.copy_(0.2 * torch.randn(n, generator=g))
    x, _ = synth.make_crops(1, seed=5)
    with torch.no_grad():
        want = I.forward(net, x)[0][-1]
        for name in I.QUIET_FOLDS:
            got = I.forward(net, x, fold=I.MUTATED_FOLDS[name])[0][-1]
            rel = float((got - want).abs().max() / want.abs().max())
            assert rel < OLD_TRUNK_BAR / 2, (stats, name, rel)


def _hypothesis(rng, n, noise):
    """n correspondences of one hypothesis: target = source + a small offset, regressor outputs near (1, cos 0.3,
    sin 0.3) with the given noise; [256]-slot layout with -1 / -1000 for invalid slots."""
    src = np.full((256, 2), -1, np.int64)
    tar = np.full((256, 2), -1, np.int64)
    sc = np.full(256, -1000.0)
    cs = np.full((256, 2), -1000.0)
    slots = rng.choice(256, n, replace=False)
    src[slots] = rng.integers(0, 16, (n, 2))
    tar[slots] = np.clip(src[slots] + rng.integers(-2, 3, (n, 2)), 0, 15)
    sc[slots] = 1 + noise * rng.standard_normal(n)
    cs[slots, 0] = math.cos(0.3) + noise * rng.standard_normal(n)
    cs[slots, 1] = math.sin(0.3) + noise * rng.standard_normal(n)
    return src, tar, sc.astype(np.float32).astype(np.float64), cs.astype(np.float32).astype(np.float64)


def test_margin_covers_every_flip_a_bounded_output_change_can_cause():
    """Regressor outputs moved at random within |d_sc|, |d_cs| per correspondence never flip a decision outside the
    margin `decisions` gives for those bounds; and some decisions inside it do flip (the check is not vacuous)."""
    rng = np.random.default_rng(4)
    flips_inside = 0
    for h in range(6):
        src, tar, sc, cs = _hypothesis(rng, 120, 0.1)
        d_sc = 10.0 ** rng.uniform(-5, -2, 256)
        d_cs = 10.0 ** rng.uniform(-5, -2, (256, 2))
        r = I.ransac(src, tar, sc, cs, d_sc=d_sc, d_cs=d_cs)
        k = r.keep
        for _ in range(100):
            u = rng.uniform(-1, 1, 256) * d_sc
            v = rng.uniform(-1, 1, (256, 2)) * d_cs
            D, _ = I.decisions(src[k], tar[k], sc[k] + u[k], cs[k] + v[k])
            flip = D != r.D
            assert not (flip & ~r.near).any(), f"hypothesis {h}: a flip outside the margin"
            flips_inside += int(flip.sum())
    assert flips_inside > 0


def test_fp64_ransac_equals_port_where_unambiguous():
    """port.ransac (fp32 torch) and `ransac` (fp64) on the same fp32-representable inputs: wherever no decision of a
    hypothesis lies within 2^-18 of its magnitudes from the threshold, the inlier sets, failed flags and counts are
    identical and M agrees to fp32 rounding."""
    rng = np.random.default_rng(5)
    hyps = [_hypothesis(rng, int(n), 0.05) for n in (0, 1, 2, 9, 17, 40, 64, 100, 256) * 4]
    st = lambda j: torch.from_numpy(np.stack([h[j] for h in hyps]))[None]
    M, failed, in_src, in_tar, in_sc = port.ransac(st(0), st(1), st(2).float(), st(3).float())
    unambiguous = 0
    for i, (src, tar, sc, cs) in enumerate(hyps):
        r = I.ransac(src, tar, sc, cs)
        if r.near is not None and r.near.any():
            continue
        unambiguous += 1
        assert np.array_equal(in_src[0, i].numpy(), r.in_src) and np.array_equal(in_tar[0, i].numpy(), r.in_tar), i
        assert bool(failed[0, i]) == r.failed and int(in_sc[0, i].sum()) == r.count, i
        assert np.allclose(M[0, i].double().numpy(), r.M, rtol=1e-6, atol=1e-3), i
    assert unambiguous >= 20, unambiguous
