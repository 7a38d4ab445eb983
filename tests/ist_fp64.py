"""An fp64 IST branch written from the definitions, independent of gigapose_b200 (torch is used for fp64 tensor
arithmetic only): the ResNet trunk from its *unfolded* module parameters, the regressor's two heads, RANSAC's inlier
decisions with the margin inside which another precision may decide otherwise, and pose lifting; with the weights and
the mutated BatchNorm folds the IST tests use.

- `layer`: one convolution of the trunk with its BatchNorm applied explicitly, (y - mu) / sqrt(var + eps) * gamma + beta
  with the module's eps, then the shortcut and ReLU where the block has them; and, per element, the magnitude the output
  is built from, |gamma| / sqrt(var + eps) sum |a||w| + |beta| + |mu gamma / sqrt(var + eps)| + |shortcut|, the
  denominator every normalised trunk error uses.  It reads its inputs from a list of activations, so it runs on its own
  chain (`forward`) or on the kernels' dumps;
- `regressor`: both heads in fp64 with the propagated magnitude |W3| (|W2| (|W1||x| + |b1|) + |b2|) + |b3|, and
  `lipschitz`, the bound |W3| (|W2| (|W1| |delta|)) on how far an input change delta can move each output (ReLU and tanh
  are 1-Lipschitz);
- `decisions` / `ransac`: the exhaustive one-point RANSAC of port.ransac in fp64, with per-decision margins;
- `pose`: port.pose_recovery in fp64;
- `realistic_trunk` / `realistic_regressor`: trained-like statistics (see there);
- `MUTATED_FOLDS`: wrong versions of `gigapose_b200.ist_trunk._fold`, which the tests require to be visibly wrong.
"""
from __future__ import annotations

import functools
import math
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

CFG = dict(input_dim=3, input_size=256, initial_dim=128, block_dims=[128, 192, 256, 512], descriptor_size=256, n_heads=0)
NUM_CONVS = 21
P = 256
DEAD_PER_LAYER = 8               # near-dead channels planted in every BatchNorm layer
DEAD_VAR = (1e-4, 1e-3)          # their conv output variance, log-uniform


def resnet(state=None, device="cpu"):
    """The shipped trunk geometry (configs/model/ist_net/resnet.yaml), in eval mode, optionally loaded."""
    from src.models.network.resnet import ResNet
    net = ResNet(CFG)
    if state is not None:
        net.load_state_dict(state)
    return net.to(device).eval()


def schedule(net):
    """Per convolution i = 1 .. 21 in the execution order of gp_ist_trunk_create: the conv, its BatchNorm, the activation
    it reads (0 = the resized crop, j = the output of convolution j), whether ReLU follows and the activation of the
    shortcut it adds."""
    s = [SimpleNamespace(conv=net.conv1, bn=net.bn1, src=0, relu=True, res=None)]
    x = 1
    for stage in (net.layer1, net.layer2, net.layer3, net.layer4):
        for blk in stage:
            s.append(SimpleNamespace(conv=blk.conv1, bn=blk.bn1, src=x, relu=True, res=None))
            y, res = len(s), x
            if blk.downsample is not None:
                s.append(SimpleNamespace(conv=blk.downsample[0], bn=blk.downsample[1], src=x, relu=False, res=None))
                res = len(s)
            s.append(SimpleNamespace(conv=blk.conv2, bn=blk.bn2, src=y, relu=True, res=res))
            x = len(s)
    s.append(SimpleNamespace(conv=net.layer4_outconv, bn=None, src=x, relu=False, res=None))
    assert len(s) == NUM_CONVS
    return s


def resize(crops):
    """The reference's bilinear align_corners resize 224 -> 256 in fp64 (resnet.py:365-368)."""
    return F.interpolate(crops.double(), (256, 256), mode="bilinear", align_corners=True)


def _d(t, dev):
    return t.detach().to(dev, torch.float64)


def bn_stats(bn, dev):
    return _d(bn.running_mean, dev), _d(bn.running_var, dev), _d(bn.weight, dev), _d(bn.bias, dev)


def layer(s, acts, eps=None, fold=None):
    """Convolution s on acts[s.src] (NCHW fp64), BatchNorm applied explicitly with eps (default: the module's), then
    + acts[s.res] and ReLU as the block has them.  Returns (output, magnitude).  With `fold` (a function like
    ist_trunk._fold) the convolution uses that function's folded filter and bias instead, in fp64."""
    x = acts[s.src].double()
    dev = x.device
    st, pad = s.conv.stride[0], s.conv.padding[0]
    if fold is not None:
        w, b = fold(s.conv, s.bn, dev)
        W = w.double().permute(0, 3, 1, 2)
        y = F.conv2d(x, W, stride=st, padding=pad)
        d = F.conv2d(x.abs(), W.abs(), stride=st, padding=pad)
        if b is not None:
            y, d = y + b.double()[:, None, None], d + b.double().abs()[:, None, None]
    else:
        W = _d(s.conv.weight, dev)
        y = F.conv2d(x, W, stride=st, padding=pad)
        d = F.conv2d(x.abs(), W.abs(), stride=st, padding=pad)
        if s.bn is not None:
            mu, var, gam, beta = bn_stats(s.bn, dev)
            sd = torch.sqrt(var + (s.bn.eps if eps is None else eps))
            c = lambda t: t[:, None, None]
            y = (y - c(mu)) / c(sd) * c(gam) + c(beta)
            d = d * c(gam.abs() / sd) + c(beta.abs()) + c((mu * gam / sd).abs())
    if s.res is not None:
        r = acts[s.res].double()
        y, d = y + r, d + r.abs()
    if s.relu:
        y = y.clamp(min=0)
    return y, d


def forward(net, crops, eps=None, fold=None):
    """The trunk from the crops: activations [resized crop, out_1 .. out_21] and magnitudes [None, den_1 .. den_21],
    NCHW fp64 on the crops' device."""
    acts, dens = [resize(crops)], [None]
    for s in schedule(net):
        y, d = layer(s, acts, eps, fold)
        acts.append(y)
        dens.append(d)
    return acts, dens


def nerr(got, ref, den):
    """Largest |got - ref| / den over all elements."""
    return float(((got.double() - ref).abs() / den.clamp(min=1e-300)).max())


# ------------------------------------------------------------------------------------------------ mutated folds
def _folder(eps=None, sqrt_in_bias=True):
    """A BatchNorm fold like ist_trunk._fold (fp32 [cout, kh, kw, cin] filter and bias) with one thing changed:
    eps replaced (0 drops it), or the bias computed as beta - mu gamma, without the 1 / sqrt(var + eps)."""
    def fold(conv, bn, device):
        w = conv.weight.detach().to(device=device, dtype=torch.float32)
        if bn is None:
            return w.permute(0, 2, 3, 1).contiguous(), None
        e = bn.eps if eps is None else eps
        g = (bn.weight / torch.sqrt(bn.running_var + e)).detach().to(device=device, dtype=torch.float32)
        gb = g if sqrt_in_bias else bn.weight.detach().to(device=device, dtype=torch.float32)
        b = (bn.bias.detach().to(device) - bn.running_mean.detach().to(device) * gb).to(torch.float32).contiguous()
        return (w * g.view(-1, 1, 1, 1)).permute(0, 2, 3, 1).contiguous(), b
    return fold


MUTATED_FOLDS = {
    "no eps": _folder(eps=0.0),
    "eps 1e-6": _folder(eps=1e-6),
    "eps 1e-3": _folder(eps=1e-3),
    "bias without sqrt": _folder(sqrt_in_bias=False),
}
QUIET_FOLDS = ("no eps", "eps 1e-6")


# -------------------------------------------------------------------------------------------------- the weights
def calibration_crops():
    from gigapose_b200 import synth
    rgb, _ = synth.make_crops(2, seed=77)
    return rgb


@functools.lru_cache(maxsize=4)
def _realistic_trunk(seed: int):
    torch.manual_seed(seed)
    net = resnet()
    g = torch.Generator().manual_seed(seed + 1)
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    log_uniform = lambda n, lo, hi: torch.exp(math.log(lo) + (math.log(hi) - math.log(lo)) * rnd(n))
    acts = [resize(calibration_crops())]
    with torch.no_grad():
        for s in schedule(net):
            if s.bn is not None:
                cout = s.conv.out_channels
                W = s.conv.weight
                y = F.conv2d(acts[s.src], W.double(), stride=s.conv.stride[0], padding=s.conv.padding[0])
                mean, var = y.mean((0, 2, 3)), y.var((0, 2, 3))
                dead = torch.randperm(cout, generator=g)[:DEAD_PER_LAYER]
                target = log_uniform(DEAD_PER_LAYER, *DEAD_VAR)
                r = torch.sqrt(target / var[dead])
                W[dead] *= r.to(W)[:, None, None, None].to(W.device)
                mean[dead] *= r.to(mean)
                var[dead] = target.to(var)
                sd = var.sqrt()
                # trained statistics do not match one batch: the mean moved by up to 0.5 sigma, and on one channel in
                # six by 2 .. 4 sigma either way; the variance scaled by a factor log-uniform over [0.5, 2] (not on the
                # planted channels, which keep var <= 1e-3)
                shift = (rnd(cout) - 0.5).to(sd)
                far = (rnd(cout) < 1 / 6).to(sd.device)
                shift = torch.where(far, torch.sign(shift) * (2 + 4 * shift.abs()), shift)
                fac = log_uniform(cout, 0.5, 2.0).to(var)
                fac[dead] = 1.0
                gam = log_uniform(cout, 0.05, 1.5)
                gam[rnd(cout) < 0.15] *= -1
                gam[torch.randperm(cout, generator=g)[:cout // 32]] = 1e-3 * (rnd(cout // 32) - 0.5)
                s.bn.running_mean.copy_(mean + shift * sd)
                s.bn.running_var.copy_(var * fac)
                s.bn.weight.copy_(gam.to(s.bn.weight))
                s.bn.bias.copy_((0.2 * torch.randn(cout, generator=g, dtype=torch.float64)).to(s.bn.bias))
            acts.append(layer(s, acts)[0])
    return {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}


def realistic_trunk(seed: int) -> dict:
    """A `ResNet` state dict with trained-like BatchNorm: the seeded init, then, layer by layer in execution order on
    two calibration crops in fp64 on the CPU (so that every machine derives the same weights up to fp64 rounding),
    - DEAD_PER_LAYER near-dead channels per BatchNorm: their filter rows scaled so that the convolution's output
      variance is log-uniform over [1e-4, 1e-3] (there eps = 1e-5 against 0 moves the channel's gain by 0.5 .. 5 %);
    - running mean and variance calibrated from the convolution's output, the mean then moved by up to 0.5 sigma (by
      2 .. 4 sigma on one channel in six) and the variance scaled by a log-uniform factor in [0.5, 2], so that
      activations stay O(1) through 21 layers;
    - |gamma| log-uniform over [0.05, 1.5], 15 % negative, and one channel in 32 with |gamma| < 5e-4; beta ~ N(0, 0.2).
    These statistics are assumed, not read from the released checkpoint, which is not available here."""
    return {k: v.clone() for k, v in _realistic_trunk(seed).items()}


def _dead_channels(net):
    """Per BatchNorm in execution order, the channels with running_var <= 1e-3."""
    return [(s.bn.running_var <= 1e-3).nonzero().flatten().tolist() for s in schedule(net) if s.bn is not None]


SCALE_STD = 0.15                 # relScale ~ 1 +- SCALE_STD
INPLANE_ANGLE = 0.3              # (cos, sin) ~ (cos 0.3, sin 0.3) = (0.955, 0.296)
INPLANE_STD = 0.1                # spread of the in-plane head's pre-tanh outputs


def realistic_regressor(seed: int, feats: torch.Tensor):
    """A `port.RegressorPort` whose output layers are rescaled on rows of `feats` ([n, 256, 16, 16] trunk features):
    relScale = 1 + N(0, SCALE_STD) on those rows, and the in-plane head's pre-tanh outputs centred on
    atanh(cos 0.3), atanh(sin 0.3) with spread INPLANE_STD, so that (cos, sin) is well away from 0.  (Random weights put
    relScale anywhere in +-100, where RANSAC's 14-px test is a knife edge.)"""
    from oracle import port
    reg = port.RegressorPort(seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    f = feats.detach().cpu().double().flatten(2)
    n = f.shape[0]
    a, b = torch.randint(0, n, (512,), generator=g), torch.randint(0, n, (512,), generator=g)
    pa, pb = torch.randint(0, P, (512,), generator=g), torch.randint(0, P, (512,), generator=g)
    rows = torch.cat([f[a, :, pa], f[b, :, pb]], 1)
    with torch.no_grad():
        for head, target, std in ((reg.scale_predictor, [1.0], SCALE_STD),
                                  (reg.inplane_predictor, [math.atanh(math.cos(INPLANE_ANGLE)),
                                                           math.atanh(math.sin(INPLANE_ANGLE))], INPLANE_STD)):
            h = rows
            for i in (0, 2):
                h = (h @ head[i].weight.double().T + head[i].bias.double()).clamp(min=0)
            out = h @ head[4].weight.double().T
            scale = std / out.std(0)
            head[4].weight.mul_(scale[:, None].float())
            head[4].bias.copy_(torch.tensor(target) - (out * scale).mean(0))
    return reg


# ------------------------------------------------------------------------------------------------------ regressor
def regressor(reg, rows):
    """rows [n, 512] fp64 -> [(scale [n,1], magnitude), (cos/sin [n,2], magnitude)] in fp64."""
    out = []
    for head in (reg.scale_predictor, reg.inplane_predictor):
        x, den = rows, rows.abs()
        for i in (0, 2, 4):
            W, b = _d(head[i].weight, rows.device), _d(head[i].bias, rows.device)
            x, den = x @ W.T + b, den @ W.abs().T + b.abs()
            if i < 4:
                x = x.clamp(min=0)
        if isinstance(head[-1], torch.nn.Tanh):
            x = torch.tanh(x)
        out.append((x, den))
    return out


def lipschitz(reg, delta):
    """|W3| (|W2| (|W1| delta)) per head: a rigorous bound on |f(x + e) - f(x)| for |e| <= delta elementwise."""
    out = []
    for head in (reg.scale_predictor, reg.inplane_predictor):
        d = delta
        for i in (0, 2, 4):
            d = d @ _d(head[i].weight, delta.device).abs().T
        out.append(d)
    return out


# --------------------------------------------------------------------------------------------------------- RANSAC
def decisions(src, tar, sc, cs, thr=14.0, patch_size=14, d_sc=None, d_cs=None):
    """Inlier decisions of one hypothesis' n valid correspondences (src / tar [n, 2] patch coordinates, sc [n], cs [n, 2]
    fp64): D[c, j] = |t_j - (M_c s_j + t_c - M_c s_c)| <= thr, M_c = sc_c [[cos, -sin], [sin, cos]], the diagonal False
    (port.ransac).  Also the margin of each decision, within which another evaluation may decide otherwise:
    - 2^-18 of the magnitudes summed into each coordinate: fp32 arithmetic (as in test_gpu_tail.py);
    - |dM_c| |s_j - s_c|, where dM_c is the change of candidate c's similarity when its regressor outputs move by at
      most d_sc [n] and d_cs [n, 2]: the residual is t_j - t_c - M_c (s_j - s_c), and for dM = [[dA, -dB], [dB, dA]]
      |dM v| = sqrt(dA^2 + dB^2) |v|, with dA <= |cos| d_sc + |sc| d_cos + d_sc d_cos (dB likewise with sin)."""
    s, t = src.astype(np.float64) * patch_size, tar.astype(np.float64) * patch_size
    c, sn = cs[:, 0], cs[:, 1]
    m00, m01, m10, m11 = c * sc, -sn * sc, sn * sc, c * sc
    m02 = t[:, 0] - (m00 * s[:, 0] + m01 * s[:, 1])
    m12 = t[:, 1] - (m10 * s[:, 0] + m11 * s[:, 1])
    ux, uy = m00[:, None] * s[None, :, 0], m01[:, None] * s[None, :, 1]
    vx, vy = m10[:, None] * s[None, :, 0], m11[:, None] * s[None, :, 1]
    dx = t[None, :, 0] - (ux + uy + m02[:, None])
    dy = t[None, :, 1] - (vx + vy + m12[:, None])
    err = np.sqrt(dx * dx + dy * dy)
    mag = np.maximum(np.abs(ux) + np.abs(uy) + np.abs(m02)[:, None] + np.abs(t[None, :, 0]),
                     np.abs(vx) + np.abs(vy) + np.abs(m12)[:, None] + np.abs(t[None, :, 1]))
    margin = 2.0 ** -18 * mag
    if d_sc is not None:
        dA = np.abs(c) * d_sc + np.abs(sc) * d_cs[:, 0] + d_sc * d_cs[:, 0]
        dB = np.abs(sn) * d_sc + np.abs(sc) * d_cs[:, 1] + d_sc * d_cs[:, 1]
        dist = np.sqrt(((s[None, :, :] - s[:, None, :]) ** 2).sum(-1))
        margin = margin + np.sqrt(dA * dA + dB * dB)[:, None] * dist
    D = err <= thr
    np.fill_diagonal(D, False)
    near = np.abs(err - thr) <= margin
    np.fill_diagonal(near, False)
    return D, near


def ransac(src_pts, tar_pts, sc, cs, thr=14.0, patch_size=14, d_sc=None, d_cs=None):
    """One hypothesis (src_pts / tar_pts [256, 2] with -1 for invalid slots, sc [256], cs [256, 2]) in fp64: the first
    candidate with the most inliers wins.  Returns keep (valid slots), D, near, best, count, failed, M [3, 3] and the
    compacted inlier src / tar points [256, 2] (-1 tails), as port.ransac lays them out."""
    keep = np.nonzero(src_pts[:, 0] != -1)[0]
    n = len(keep)
    out = SimpleNamespace(keep=keep, D=None, near=None, best=None, count=0, failed=False, M=np.eye(3),
                          in_src=np.full((P, 2), -1, np.int64), in_tar=np.full((P, 2), -1, np.int64))
    if n == 0:
        return out
    sel = lambda a: None if a is None else a[keep]
    D, near = decisions(src_pts[keep], tar_pts[keep], sc[keep], cs[keep], thr, patch_size, sel(d_sc), sel(d_cs))
    score = D.sum(1)
    best = int(np.argmax(score))
    j = np.nonzero(D[best])[0]
    s = src_pts[keep].astype(np.float64) * patch_size
    t = tar_pts[keep].astype(np.float64) * patch_size
    c, sn, k = cs[keep][best, 0], cs[keep][best, 1], sc[keep][best]
    R = np.array([[c * k, -sn * k], [sn * k, c * k]])
    out.M[:2, :2] = R
    out.M[:2, 2] = t[best] - R @ s[best]
    out.in_src[:len(j)], out.in_tar[:len(j)] = src_pts[keep][j], tar_pts[keep][j]
    out.D, out.near, out.best, out.count, out.failed = D, near, best, int(score[best]), bool(score[best] == 0)
    return out


# ------------------------------------------------------------------------------------------------- pose lifting
def pose(q_obj, qK, qM, id_src, M, tK, tM, tP):
    """port.pose_recovery in fp64 (object index given 0-based): [B, k, 4, 4]."""
    d = lambda t: t.double()
    qK, qM, M, tK, tM, tP = map(d, (qK, qM, M, tK, tM, tP))
    B, k = id_src.shape
    o = q_obj.long()[:, None].expand(B, k)
    tKb, tMb, P_ = tK[o], tM[o, id_src], tP[o, id_src].clone()
    sc = M[..., :2, 0].norm(dim=-1)
    Rin = torch.eye(3, dtype=torch.float64).repeat(B, k, 1, 1)
    Rin[..., :2, :2] = M[..., :2, :2] / sc[..., None, None]
    R = Rin @ P_[..., :3, :3]
    tz = P_[..., 2, 3]
    c2d = tKb @ P_[..., :3, 3:4]
    c2d = c2d / c2d[..., 2:3, :]
    qs = qM[:, 0, 0]
    Minv = torch.eye(3, dtype=torch.float64).repeat(B, 1, 1)
    Minv[:, 0, 0] = Minv[:, 1, 1] = 1 / qs
    Minv[:, :2, 2] = -qM[:, :2, 2] / qs[:, None]
    aff = Minv[:, None] @ M @ tMb
    qc = aff @ c2d
    s2d = aff[..., :2, 0].norm(dim=-1)
    qz = (tz / s2d) * (qK[:, None, 0, 0] / tKb[..., 0, 0])
    tr = (torch.inverse(qK)[:, None] @ qc)[..., 0]
    tr = tr / tr[..., 2:3] * qz[..., None]
    P_[..., :3, :3] = R
    P_[..., :3, 3] = tr
    return P_
