"""An fp64 DINOv2 ViT-L/14 forward written from the definitions, independent of the kernels' operation order and of
oracle/port.py's modules (torch is used for fp64 tensor arithmetic only), with the weights and mutations the ViT tests
use.

- `embed`: patch embedding (stride-14 convolution + bias), the CLS row and the bicubic positional table;
- `block`: one pre-norm transformer block,
      y = LN1(x) (eps 1e-6, two-pass variance);  q, k, v = split(y W_qkv^T + b_qkv) into 16 heads of 64;
      a = softmax(q k^T / 8) v;  x' = x + g1 * (a W_proj^T + b_proj);
      h = GELU_erf(LN2(x') W_fc1^T + b_fc1);  out = x' + g2 * (h W_fc2^T + b_fc2),
  and, per element, the fp64 sum of the magnitudes the output is built from,
      |x| + |g1| (|a| |W_proj|^T + |b_proj|) + |g2| (|h| |W_fc2|^T + |b_fc2|),
  the denominator the tests normalise errors by (as tests/test_gpu_kernels.py does for single kernels);
- `descriptors`: AENet's tail (ae_net.py:65-69): drop CLS, b (h w) c -> b c h w, F.normalize over c with eps 1e-12;
- `realistic_weights`: per-channel LayerScales, spread LayerNorm weights and planted high-norm channels (see there);
- `MUTATIONS`: named wrong versions of the block, which the tests require to be visibly wrong on these weights.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F

DIM, HEADS, HEAD_DIM, PATCH, GRID, TOK = 1024, 16, 64, 14, 16, 257
LN_EPS = 1e-6
MASSIVE_CHANNELS = (203, 771)       # the channels realistic_weights plants its high-norm values in
# (row, col) of the 37 x 37 table: each lies within 0.18 of a point the resize to 16 x 16 samples, (i + 0.5) 37 / 16.1 - 0.5
MASSIVE_POSITIONS = ((3, 19), (10, 33), (12, 12), (19, 26), (26, 3), (33, 10))
MASSIVE_VALUES = ((300.0, -250.0), (-220.0, 280.0), (350.0, 200.0), (-260.0, -300.0), (240.0, 330.0), (-310.0, 210.0))
MASSIVE_CLS = (320.0, -270.0)

BLOCK_NAMES = ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias",
          "ls1.gamma", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias",
          "ls2.gamma")


def block_params(model, i, device=None) -> dict:
    """Block i's parameters in fp64 under their state-dict names (the names of upstream DINOv2)."""
    p = dict(model.blocks[i].named_parameters())
    return {n: p[n].detach().to(device=device or p[n].device, dtype=torch.float64) for n in BLOCK_NAMES}


def layernorm(x, w, b, eps=LN_EPS):
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    return d / torch.sqrt((d * d).mean(-1, keepdim=True) + eps) * w + b


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def block(x, p, eps=LN_EPS, gelu=gelu_erf, scale=HEAD_DIM ** -0.5, swap_qk=False):
    """x [b, 257, 1024] fp64 -> (block output, per-element magnitude sum), both fp64."""
    B, N, C = x.shape
    y = layernorm(x, p["norm1.weight"], p["norm1.bias"], eps)
    qkv = (y @ p["attn.qkv.weight"].T + p["attn.qkv.bias"]).reshape(B, N, 3, HEADS, HEAD_DIM).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if swap_qk:
        q, k = k, q
    a = torch.softmax((q @ k.transpose(-1, -2)) * scale, dim=-1) @ v
    a = a.transpose(1, 2).reshape(B, N, C)
    g1, g2 = p["ls1.gamma"], p["ls2.gamma"]
    x1 = x + g1 * (a @ p["attn.proj.weight"].T + p["attn.proj.bias"])
    h = gelu(layernorm(x1, p["norm2.weight"], p["norm2.bias"], eps) @ p["mlp.fc1.weight"].T + p["mlp.fc1.bias"])
    out = x1 + g2 * (h @ p["mlp.fc2.weight"].T + p["mlp.fc2.bias"])
    den = (x.abs() + g1.abs() * (a.abs() @ p["attn.proj.weight"].abs().T + p["attn.proj.bias"].abs())
           + g2.abs() * (h.abs() @ p["mlp.fc2.weight"].abs().T + p["mlp.fc2.bias"].abs()))
    return out, den


def _swap(p, a, b):
    q = dict(p)
    q[a], q[b] = p[b], p[a]
    return q


def _norms_swapped(p):
    return _swap(_swap(p, "norm1.weight", "norm2.weight"), "norm1.bias", "norm2.bias")


def _next_gammas(p, p_next):
    return dict(p, **{"ls1.gamma": p_next["ls1.gamma"], "ls2.gamma": p_next["ls2.gamma"]})


def _unit_gammas(p):
    one = torch.ones_like(p["ls1.gamma"])
    return dict(p, **{"ls1.gamma": one, "ls2.gamma": one})


# name -> (needs the next block's parameters, f(x, p, p_next) -> block output)
MUTATIONS = {
    "ls1<->ls2": (False, lambda x, p, pn: block(x, _swap(p, "ls1.gamma", "ls2.gamma"))[0]),
    "gammas of block k+1": (True, lambda x, p, pn: block(x, _next_gammas(p, pn))[0]),
    "gamma=1": (False, lambda x, p, pn: block(x, _unit_gammas(p))[0]),
    "eps 1e-5": (False, lambda x, p, pn: block(x, p, eps=1e-5)[0]),
    "tanh-GELU": (False, lambda x, p, pn: block(x, p, gelu=gelu_tanh)[0]),
    "norm1<->norm2": (False, lambda x, p, pn: block(x, _norms_swapped(p))[0]),
    "q<->k": (False, lambda x, p, pn: block(x, p, swap_qk=True)[0]),
    "scale 1/sqrt(1024)": (False, lambda x, p, pn: block(x, p, scale=DIM ** -0.5)[0]),
}


def _cubic(n_in, n_out, scale_factor, device):
    """[n_out, n_in] weights of 1-D bicubic resampling (Keys, a = -0.75) at source x = (i + 0.5) / scale_factor - 0.5,
    the four taps clamped to the border: upstream's F.interpolate(scale_factor=..., mode="bicubic")."""
    a = -0.75
    src = (torch.arange(n_out, dtype=torch.float64, device=device) + 0.5) * (1.0 / scale_factor) - 0.5
    i0 = torch.floor(src)
    t = src - i0
    near = lambda d: ((a + 2) * d - (a + 3)) * d * d + 1                    # |d| <= 1
    far = lambda d: ((a * d - 5 * a) * d + 8 * a) * d - 4 * a               # 1 < |d| < 2
    W = torch.zeros(n_out, n_in, dtype=torch.float64, device=device)
    rows = torch.arange(n_out, device=device)
    for off, w in ((-1, far(t + 1)), (0, near(t)), (1, near(1 - t)), (2, far(2 - t))):
        W.index_put_((rows, (i0.long() + off).clamp(0, n_in - 1)), w, accumulate=True)
    return W


def pos_table(model, device=None):
    """The [257, 1024] positional rows for a 16 x 16 grid in fp64, and their magnitude sums: the CLS row as stored, and
    the 37 x 37 patch table resized as upstream's interpolate_pos_encoding does (bicubic, scale factor (16 + 0.1) / 37
    on both axes) -- sum_ij wy_i wx_j pe_ij and sum_ij |wy_i| |wx_j| |pe_ij|."""
    pe = model.pos_embed.detach().to(device=device or model.pos_embed.device, dtype=torch.float64)[0]
    m = math.isqrt(pe.shape[0] - 1)
    W = _cubic(m, GRID, (GRID + 0.1) / m, pe.device)
    grid = pe[1:].reshape(m, m, DIM)
    res = lambda W, g: torch.einsum("yi,xj,ijc->yxc", W, W, g).reshape(GRID * GRID, DIM)
    return torch.cat([pe[:1], res(W, grid)]), torch.cat([pe[:1].abs(), res(W.abs(), grid.abs())])


def embed(model, img):
    """img [b, 3, 224, 224] -> (block 0's input rows [b, 257, 1024], magnitude sum), fp64 on img's device."""
    dev = img.device
    W = model.patch_embed.proj.weight.detach().to(dev, torch.float64)
    bias = model.patch_embed.proj.bias.detach().to(dev, torch.float64)
    cls = model.cls_token.detach().to(dev, torch.float64).reshape(1, 1, DIM)
    pos, pos_den = pos_table(model, dev)
    X = img.to(torch.float64)
    tok = lambda t: t.flatten(2).transpose(1, 2)
    x = torch.cat([cls.expand(len(X), 1, DIM), tok(F.conv2d(X, W, bias, stride=PATCH))], 1) + pos
    den = torch.cat([cls.abs().expand(len(X), 1, DIM), tok(F.conv2d(X.abs(), W.abs(), bias.abs(), stride=PATCH))], 1) \
        + pos_den
    return x, den


def forward(model, img, depth=None):
    """fp64 x_prenorm after the first `depth` blocks (all by default)."""
    x, _ = embed(model, img)
    for i in range(len(model.blocks) if depth is None else depth):
        x, _ = block(x, block_params(model, i, img.device))
    return x


def descriptors(x_prenorm):
    """AENet's unit-norm patch features [b, 1024, 16, 16] from x_prenorm [b, 257, 1024]."""
    t = x_prenorm[:, 1:]
    return F.normalize(t.reshape(len(t), GRID, GRID, DIM).permute(0, 3, 1, 2), dim=1, eps=1e-12)


@torch.no_grad()
def realistic_weights(depth: int, seed: int) -> nn.Module:
    """A `DinoVisionTransformer` of `depth` blocks: the seeded init, then
    - per-channel LayerScales g1, g2 with |g| log-uniform over [1e-3, 1] and a random sign, drawn independently for
      every block and for ls1 and ls2;
    - LayerNorm weights with |w| log-uniform over [0.05, 3], one in ten negative;
    - the patch-embedding bias and the positional table drawn at 0.005 rather than 0.02, so that the tokens of a zero
      image region (a masked-out query) have a variance of about 5e-5, where LayerNorm's eps shows;
    - two high-norm channels (MASSIVE_CHANNELS) planted through pos_embed: a few hundred on the CLS row and on six patch
      positions of the 37 x 37 table, which the host's bicubic resize to 16 x 16 spreads over neighbouring patches.
    These statistics are assumed, not read from the released checkpoint, which is not available here: DINOv2 ViT-L is
    reported to carry per-channel LayerScales and high-norm tokens concentrated in a few channels (Darcet et al.,
    "Vision Transformers Need Registers", 2023), and the magnitudes above are guesses of that order."""
    from gigapose_b200.vit import DinoVisionTransformer
    m = DinoVisionTransformer(depth=depth, init_seed=seed)
    g = torch.Generator().manual_seed(seed + 1)

    def log_uniform(n, lo, hi, neg):
        mag = 10.0 ** (math.log10(lo) + (math.log10(hi) - math.log10(lo)) * torch.rand(n, generator=g))
        return torch.where(torch.rand(n, generator=g) < neg, -mag, mag)

    for blk in m.blocks:
        blk.ls1.gamma.copy_(log_uniform(DIM, 1e-3, 1.0, 0.5))
        blk.ls2.gamma.copy_(log_uniform(DIM, 1e-3, 1.0, 0.5))
        blk.norm1.weight.copy_(log_uniform(DIM, 0.05, 3.0, 0.1))
        blk.norm2.weight.copy_(log_uniform(DIM, 0.05, 3.0, 0.1))
    m.norm.weight.copy_(log_uniform(DIM, 0.05, 3.0, 0.1))
    m.patch_embed.proj.bias.copy_(0.005 * torch.randn(DIM, generator=g))
    m.pos_embed.copy_(0.005 * torch.randn(m.pos_embed.shape, generator=g))
    pe = m.pos_embed[0]
    side = math.isqrt(pe.shape[0] - 1)
    for c, v in zip(MASSIVE_CHANNELS, MASSIVE_CLS):
        pe[0, c] = v
    for (r, col), vals in zip(MASSIVE_POSITIONS, MASSIVE_VALUES):
        for c, v in zip(MASSIVE_CHANNELS, vals):
            pe[1 + r * side + col, c] = v
    return m


def truncated(model, k: int) -> nn.Module:
    """A `DinoVisionTransformer` sharing (not copying) the embedding and the first k blocks of `model`."""
    from gigapose_b200.vit import DinoVisionTransformer
    t = DinoVisionTransformer(depth=0)
    t.cls_token, t.pos_embed, t.mask_token, t.patch_embed = model.cls_token, model.pos_embed, model.mask_token, model.patch_embed
    t.blocks = nn.ModuleList(list(model.blocks[:k]))
    t.norm = model.norm
    return t


def nerr(got, ref, den):
    """Largest |got - ref| / den over all elements."""
    return float(((got.double() - ref).abs() / den.clamp(min=1e-300)).max())
