"""-m gpu: the kernels that produce the descriptors, each alone against a plain high-precision statement of the same
operation -- the IST trunk's 21 implicit-GEMM convolutions and its resize, the ViT's patch embedding, CLS rows and
LayerNorm, and the bank / query writes (descriptor split, mask sampling, IST transpose, object order).

As in test_gpu_kernels.py, fp64 references are computed from the reconstructed split operands (hi + lo) the kernel
itself read, so a measured error belongs to the kernel and not to the layers before it.  Convolution errors are
normalised per element by sum |a| |w| (+ |bias| + |shortcut|).  Each bar is about 4x the largest value measured on an
H100 SXM (80 GB, 700 W power limit), stated next to it; the sensitivity checks show that each bar rejects the defect
it is there for (one split pass, replicate instead of zero padding, a swapped im2col order, LayerNorm eps 1e-5).
Where the test owns an output buffer it is prefilled with a sentinel that what the kernel must not write keeps."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from gigapose_b200 import _lib
from gigapose_b200._lib import check
from gigapose_b200.engine import Engine
from gigapose_b200.ist_trunk import NativeISTTrunk
from gigapose_b200.vit import DinoVisionTransformer
from gigapose_b200.vit_engine import NativeViT
from oracle import port

from helpers import write_report

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
SENT16 = -1                     # int16 0xFFFF: a NaN in bf16
P = 256

# --- bars, with the largest value measured on an H100 SXM (700 W limit) in brackets
BAR_CONV = 2.5e-5               # trunk convolutions 1-20, bf16 hi/lo output planes,        [6.3e-6 stem, 5.0e-6 others]
                                # of sum |a||w| + |b| + |shortcut|
BAR_OUTCONV = 7e-6              # output convolution (1x1, fp32 rows)                        [1.7e-6]
BAR_RESIZE = 3e-5               # bilinear 224 -> 256, of the largest of the four neighbours [7.0e-6]
BAR_PATCH = 6e-6                # patch embedding, of sum |x||w| + |b| + |pos|                [1.5e-6]
BAR_LN = 2.5e-5                 # LayerNorm, of |w| (1 + |x_hat|) + |b|: ordinary rows        [5.6e-6]
BAR_LN_SMALL_VAR = 1.2e-4       # rows with variance ~1e-6, where eps matters                 [2.8e-5]
BAR_LN_OFFSET = 0.2             # rows with mean 1e3 and sigma 1e-3: the fp32 mean is off by  [5.5e-2]
                                # ~1e-5 of 1e3 (a few ulps), i.e. ~1e-2 sigma
BAR_DESC = 3e-5                 # descriptor planes hi + lo, relative per element             [7.7e-6]
                                # (the split's own bound is 2^-17 = 7.6e-6)


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=_gen(seed), device=DEV) * scale


def split(x):
    """hi = bf16_rn(x), lo = bf16_rn(x - hi): the split of launch_split_planes, im2col and the GEMM epilogue."""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def joined(planes):
    return planes[0].double() + planes[1].double()


def nerr(got, ref, den):
    return float(((got.double() - ref).abs() / den.clamp(min=1e-300)).max())


def bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _carve(sizes):
    """Byte offsets of buffers taken one after another at 1024-byte alignment (the Carver of api.cu), and the total."""
    offs, off = [], 0
    for s in sizes:
        offs.append(off)
        off += -(-s // 1024) * 1024
    return offs, off


# ================================================================================================ IST trunk
CFG = dict(input_dim=3, input_size=256, initial_dim=128, block_dims=[128, 192, 256, 512], descriptor_size=256, n_heads=0)
NUM_CONVS = 21


def _network(seed=0):
    from src.models.network.resnet import ResNet
    torch.manual_seed(seed)
    net = ResNet(CFG).to(DEV).eval()
    with torch.no_grad():
        for m in net.modules():                      # non-trivial inference statistics so that the folding is exercised
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.2); m.running_var.uniform_(0.5, 1.5)
                m.weight.uniform_(0.5, 1.5); m.bias.normal_(0, 0.2)
    return net


def _schedule(net):
    """Per convolution i = 1 .. 21 (execution order): the module, the dump it reads (dump j = output of convolution j,
    dump 0 = the resized crop), whether ReLU follows and the dump of the shortcut it adds -- derived from the blocks."""
    sched = [SimpleNamespace(conv=net.conv1, src=0, relu=True, res=None)]
    x = 1
    for layer in (net.layer1, net.layer2, net.layer3, net.layer4):
        for blk in layer:
            sched.append(SimpleNamespace(conv=blk.conv1, src=x, relu=True, res=None))
            y, res = len(sched), x
            if blk.downsample is not None:
                sched.append(SimpleNamespace(conv=blk.downsample[0], src=x, relu=False, res=None))
                res = len(sched)
            sched.append(SimpleNamespace(conv=blk.conv2, src=y, relu=True, res=res))
            x = len(sched)
    sched.append(SimpleNamespace(conv=net.layer4_outconv, src=x, relu=False, res=None))
    assert len(sched) == NUM_CONVS
    return sched


def _trunk_crops(seed):
    """Five different crops: N(0,1) in a +50 frame (outer 4 pixels), plain N(0,1), all zero (a masked-out query),
    zero but for single bright pixels at (0, 0) and (223, 223), N(0,1) in a -50 frame."""
    x = _rand(5, 3, 224, 224, seed=seed)
    frame = torch.zeros(224, 224, dtype=torch.bool, device=DEV)
    frame[:4] = frame[-4:] = True
    frame[:, :4] = frame[:, -4:] = True
    x[0][:, frame] = 50.0
    x[4][:, frame] = -50.0
    x[2] = 0.0
    x[3] = 0.0
    x[3, :, 0, 0] = torch.tensor([50.0, -50.0, 30.0], device=DEV)
    x[3, :, 223, 223] = torch.tensor([-40.0, 50.0, 50.0], device=DEV)
    return x


FRAMED = [0, 4]


def _stem_interior(d):
    """[n, 262, 264, 4] stem planes -> the [n, 256, 256, 3] resized crop."""
    return d[:, 3:259, 4:260, :3]


def _border_is_zero(d):
    rest = d.clone()
    rest[:, 3:259, 4:260, :3] = 0
    return bool((bits(rest) == 0).all())


def _conv_ref(x, sched_i, weights_i, padding_mode="zeros"):
    """fp64 convolution of the NHWC input x with the split-reconstructed folded filter, + bias; and the magnitude sum
    sum |x||w| + |b| (fp32 is enough for a normaliser).  Both NHWC."""
    conv = sched_i.conv
    stride, pad = conv.stride[0], conv.padding[0]
    w, b = weights_i
    W = joined(split(w)).permute(0, 3, 1, 2)                   # [cout, kh, kw, cin] -> OIHW
    X = x.permute(0, 3, 1, 2).double()
    if padding_mode == "replicate":
        X, pad = F.pad(X, (pad,) * 4, mode="replicate"), 0
    ref = F.conv2d(X, W, stride=stride, padding=pad)
    den = F.conv2d(X.abs().float(), W.abs().float(), stride=stride, padding=pad).double()
    if b is not None:
        ref, den = ref + b.double()[:, None, None], den + b.abs().double()[:, None, None]
    return ref.permute(0, 2, 3, 1), den.permute(0, 2, 3, 1)


def _layer_err(dumps, final, sched, weights, i, crops=None, padding_mode="zeros"):
    """Normalised error of convolution i's output (dump i, or the forward output for i = 21) against fp64 from the
    kernel's own input dump."""
    s = sched[i - 1]
    pick = (lambda t: t) if crops is None else (lambda t: t[crops])
    x = pick(dumps[s.src])
    if i == 1:
        x = _stem_interior(x)
    ref, den = _conv_ref(x, s, weights[i - 1], padding_mode)
    if s.res is not None:
        r = pick(dumps[s.res]).double()
        ref, den = ref + r, den + r.abs()
    if s.relu:
        ref = ref.clamp(min=0)
    got = pick(final.permute(0, 2, 3, 1) if i == NUM_CONVS else dumps[i])
    return nerr(got, ref, den)


def _run_all(eng, x):
    dumps = [eng.activation_after(x, i) for i in range(NUM_CONVS)]
    return dumps, eng.forward(x)


@pytest.fixture(scope="module")
def trunk():
    net = _network(0)
    x = _trunk_crops(seed=1)
    eng = NativeISTTrunk(net, DEV, max_crops=len(x))
    dumps, final = _run_all(eng, x)
    torch.cuda.synchronize(DEV)
    return SimpleNamespace(net=net, x=x, eng=eng, dumps=dumps, final=final, sched=_schedule(net))


def test_trunk_schedule_covers_every_convolution_form(trunk):
    """The layers checked below cover every filter shape, epilogue, the swapped operand form (128 output channels),
    192-column tiles and every input width."""
    sched, w = trunk.sched, trunk.eng.weights
    for s, (wi, _) in zip(sched, w):
        c = s.conv
        assert tuple(wi.shape) == (c.out_channels, *c.kernel_size, c.in_channels)
    assert {(s.conv.kernel_size[0], s.conv.stride[0]) for s in sched} == {(7, 2), (3, 1), (3, 2), (1, 2), (1, 1)}
    assert {(s.relu, s.res is not None) for s in sched} == {(True, False), (True, True), (False, False)}
    assert {s.conv.out_channels for s in sched} >= {128, 192}
    assert {s.conv.in_channels for s in sched} >= {128, 192, 256, 512}


def test_stem_input_is_the_align_corners_resize_with_a_zero_border(trunk):
    """num_convs = 0 dumps the stem's input planes: the interior is the bilinear align_corners resize 224 -> 256 (index
    and weights in fp32, as the kernel and ATen compute them, blended in fp64), the border and channel 3 are 0."""
    d = trunk.dumps[0]
    assert d.shape == (5, 262, 264, 4)
    assert _border_is_zero(d)
    scale = torch.tensor(223.0, device=DEV) / torch.tensor(255.0, device=DEV)
    f = scale * torch.arange(256, device=DEV, dtype=torch.float32)
    i0 = f.long()
    ip = torch.where(i0 < 223, i0 + 1, i0)
    lw = (f - i0.float()).double()
    hw = (1.0 - (f - i0.float())).double()
    x = trunk.x.double()
    a, b = x[:, :, i0][:, :, :, i0], x[:, :, i0][:, :, :, ip]
    c, e = x[:, :, ip][:, :, :, i0], x[:, :, ip][:, :, :, ip]
    hy, ly, hx, lx = hw[:, None], lw[:, None], hw[None, :], lw[None, :]
    ref = hy * (hx * a + lx * b) + ly * (hx * c + lx * e)
    den = torch.stack([a.abs(), b.abs(), c.abs(), e.abs()]).amax(0)
    err = nerr(_stem_interior(d).permute(0, 3, 1, 2), ref, den)
    write_report("encoder_trunk_resize.json", {"err": err})
    assert err < BAR_RESIZE, f"resize error {err:.3e}"


def test_every_trunk_convolution_against_fp64(trunk):
    """Each of the 21 convolutions from the GPU's own input: folded filters split like launch_split_planes, F.conv2d in
    fp64 with the layer's stride and zero padding, + bias, then the layer's epilogue (ReLU; + shortcut dump and ReLU;
    nothing for the downsample and the output convolution, which is checked through forward()).  On the framed crops
    the same outputs against replicate padding must miss by >= 100x the bar: the padding taps carry weight at every
    level."""
    errs, rep = {}, {}
    for i in range(1, NUM_CONVS + 1):
        errs[i] = _layer_err(trunk.dumps, trunk.final, trunk.sched, trunk.eng.weights, i)
        if trunk.sched[i - 1].conv.padding[0] > 0:
            rep[i] = _layer_err(trunk.dumps, trunk.final, trunk.sched, trunk.eng.weights, i, FRAMED, "replicate")
    write_report("encoder_trunk_convs.json", {"err": errs, "replicate_padding": rep})
    bad = {i: e for i, e in errs.items() if e >= (BAR_OUTCONV if i == NUM_CONVS else BAR_CONV)}
    assert not bad, f"convolutions over the bar: {bad}"
    weak = {i: e for i, e in rep.items() if e < 100 * BAR_CONV}                         # [8.6e-2 smallest]
    assert not weak, f"replicate padding within 100x the bar: {weak}"


def test_one_pass_trunk_misses_every_convolution_bar_by_10x(trunk):
    """precision="bf16" (hi * hi only) measured the same way, on its own inputs: >= 10x the bar on every layer."""
    x = trunk.x[:2]
    eng = NativeISTTrunk(trunk.net, DEV, max_crops=2, precision="bf16")
    dumps, final = _run_all(eng, x)
    errs = {i: _layer_err(dumps, final, trunk.sched, eng.weights, i) for i in range(1, NUM_CONVS + 1)}
    write_report("encoder_trunk_one_pass.json", {"err": errs})
    # [4.1e-4 smallest, layer4; 1.0e-3 for the output convolution]
    weak = {i: e for i, e in errs.items() if e < 10 * (BAR_OUTCONV if i == NUM_CONVS else BAR_CONV)}
    assert not weak, f"one-pass layers within 10x the bar: {weak}"


def _tiles(sched, dumps, n):
    """Output tiles of each convolution at n crops: 128 pixels x all / 192 / 256 channels, or for 128 output channels
    (the swapped form) 256 pixels x 128 channels."""
    out = []
    for i, s in enumerate(sched, 1):
        h = dumps[i].shape[1] if i < NUM_CONVS else 16
        cout = s.conv.out_channels
        if cout == 128:
            out.append(n * h * h // 256)
        else:
            out.append(-(-n * h * h // 128) * (cout // (192 if cout == 192 else 256)))
    return out


def test_persistent_trunk_batches_are_bit_identical_and_leave_no_stale_data(trunk):
    """A batch large enough that every convolution, layer4 and the output convolution included, has more tiles than
    the device has SMs (persistent CTAs run several tiles), with the five fp64-checked crops last: their dumps and
    features are bit-identical to the small batch (tiles never straddle images; the accumulation order per tile is
    fixed).  Then a small call on the same engine gives the same bits as the fresh small engine."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    n = sms // 2 + 1
    tiles = _tiles(trunk.sched, trunk.dumps, n)
    assert min(tiles) > sms, tiles
    k = len(trunk.x)
    xb = torch.cat([_rand(n - k, 3, 224, 224, seed=2), trunk.x])
    eng = NativeISTTrunk(trunk.net, DEV, max_crops=n)
    write_report("encoder_trunk_persistent.json", {"crops": n, "sms": sms, "tiles": tiles})
    for i in range(NUM_CONVS):
        d = eng.activation_after(xb, i)
        if i == 0:
            assert _border_is_zero(d), "stem border after a max_crops batch"
        assert torch.equal(bits(d[n - k:]), bits(trunk.dumps[i])), f"dump {i} of the large batch differs"
    assert torch.equal(bits(eng.forward(xb)[n - k:].contiguous()), bits(trunk.final.contiguous()))
    for i in range(NUM_CONVS):
        d = eng.activation_after(trunk.x, i)
        if i == 0:
            assert _border_is_zero(d), "stem border after a small batch"
        assert torch.equal(bits(d), bits(trunk.dumps[i])), f"dump {i} of the small call after a large one differs"
    assert torch.equal(bits(eng.forward(trunk.x).contiguous()), bits(trunk.final.contiguous()))


# ====================================================================================== ViT patch embedding
@pytest.fixture(scope="module")
def vit():
    """Depth-1 ViT with both LayerScales zeroed: the residual GEMMs add 0, so x_prenorm is the embedding itself."""
    ref = port.DinoV2Port(depth=1, seed=5)
    with torch.no_grad():
        ref.blocks[0].ls1.gamma.zero_()
        ref.blocks[0].ls2.gamma.zero_()
    m = DinoVisionTransformer(depth=1)
    m.load_state_dict(ref.state_dict())
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    many = sms // 8 + 1                              # 2 x 4 tiles of 128 x 256 per crop
    return SimpleNamespace(eng=NativeViT(m.to(DEV), DEV, max_crops=many), many=many, sms=sms)


@pytest.mark.parametrize("b", [1, 3, "many"])
def test_patch_embedding_and_cls_rows_against_fp64(vit, b):
    """Token 0 of every crop is cls_token + pos[0] in fp32 (== : only -0.0 may change); tokens 1..256 are the fp64
    conv2d(img, W, stride 14) + b + pos[1:] of the split image and weights (im2col, patch-embed GEMM epilogue).  'many'
    has more patch-embedding tiles than SMs.  Swapping (ky, kx) in the reference misses by orders of magnitude."""
    b = vit.many if b == "many" else b
    if b == vit.many:
        assert 8 * b > vit.sms
    img = _rand(b, 3, 224, 224, seed=40 + b)
    out = vit.eng.forward(img)
    torch.cuda.synchronize(DEV)
    W, bias, cls, pos = vit.eng.weights[:4]
    assert bool((out[:, 0] == (cls + pos[0])[None]).all()), "CLS rows"
    X = joined(split(img))
    W64 = joined(split(W)).reshape(1024, 3, 14, 14)
    tok = lambda t: t.flatten(2).transpose(1, 2)
    extra = bias.double() + pos[1:].double()
    ref = tok(F.conv2d(X, W64, stride=14)) + extra
    den = tok(F.conv2d(X.abs(), W64.abs(), stride=14)) + bias.double().abs() + pos[1:].double().abs()
    swapped = tok(F.conv2d(X, W64.transpose(2, 3), stride=14)) + extra
    err, err_sw = nerr(out[:, 1:], ref, den), nerr(out[:, 1:], swapped, den)
    write_report(f"encoder_patch_embed_b{b}.json", {"err": err, "swapped_ky_kx": err_sw})
    assert err < BAR_PATCH, f"patch embedding error {err:.3e}"
    assert err_sw > 1000 * BAR_PATCH, f"swapped im2col order only {err_sw:.3e}"       # [0.43]


# =============================================================================================== LayerNorm
LN_EPS = 1e-6


def _ln_rows(M, seed):
    """Row classes: ordinary; mean 1e3 and sigma 1e-3; constant rows of values whose row sum is exact; variance ~1e-6."""
    g = _gen(seed)
    x = torch.randn(M, 1024, generator=g, device=DEV)
    s = 10 ** (2 * torch.rand(M, 1, generator=g, device=DEV) - 1)
    x = x * s + torch.randn(M, 1, generator=g, device=DEV) * s
    cls = {"ordinary": list(range(0, 300)) + list(range(620, M)), "offset": list(range(300, 428)),
           "constant": list(range(428, 492)), "small_var": list(range(492, 620))}
    o = cls["offset"]
    x[o] = 1000.0 + 1e-3 * torch.randn(len(o), 1024, generator=g, device=DEV)
    c = cls["constant"]
    x[c] = torch.tensor([0.75, -3.5, 0.0, 1024.0], device=DEV).repeat(len(c) // 4)[:, None]
    v = cls["small_var"]
    x[v] = 0.25 * torch.randn(len(v), 1, generator=g, device=DEV) + 1e-3 * torch.randn(len(v), 1024, generator=g, device=DEV)
    return x, {k: torch.tensor(i, device=DEV) for k, i in cls.items()}


def _ln64(x, w, b, eps):
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    xh = (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    return xh * w.double() + b.double(), w.double().abs() * (1.0 + xh.abs()) + b.double().abs()


def test_layernorm_against_fp64_with_its_edge_rows():
    """gp_debug_layernorm (the kernel and eps gp_vit_forward uses) on M = 771 rows (not a multiple of the 8 rows per
    block), sentinel rows after M untouched.  Constant rows give exactly the split of the bias.  The variance-1e-6
    rows reject eps = 1e-5; the mean-1e3 rows reject a one-pass variance E[x^2] - mean^2."""
    M, extra = 771, 13
    x, cls = _ln_rows(M, seed=7)
    w = 1.0 + 0.1 * _rand(1024, seed=8)
    b = 0.5 * _rand(1024, seed=9)
    out = tuple(torch.full((M + extra, 1024), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16) for _ in range(2))
    check(_lib.load().gp_debug_layernorm(M, x.data_ptr(), w.data_ptr(), b.data_ptr(), out[0].data_ptr(),
                                         out[1].data_ptr(), _stream()))
    torch.cuda.synchronize(DEV)
    assert bool((bits(out[0][M:]) == SENT16).all() and (bits(out[1][M:]) == SENT16).all()), "rows >= M were written"
    got = joined((out[0][:M], out[1][:M]))
    ref, den = _ln64(x, w, b, LN_EPS)
    errs = {k: nerr(got[i], ref[i], den[i]) for k, i in cls.items() if k != "constant"}
    v = cls["small_var"]
    errs["small_var_eps_1e-5"] = nerr(got[v], *_ln64(x[v], w, b, 1e-5))
    o = cls["offset"]
    xo = x[o]
    mu = xo.mean(-1, keepdim=True)
    one_pass = (xo - mu) / torch.sqrt(((xo * xo).mean(-1, keepdim=True) - mu * mu).clamp(min=0) + LN_EPS) * w + b
    errs["offset_one_pass_fp32"] = nerr(one_pass, ref[o], den[o])
    write_report("encoder_layernorm.json", errs)
    hi, lo = split(b.expand(len(cls["constant"]), -1).contiguous())
    c = cls["constant"]
    assert torch.equal(bits(out[0][c]), bits(hi)) and torch.equal(bits(out[1][c]), bits(lo)), "constant rows != bias"
    assert errs["ordinary"] < BAR_LN, errs
    assert errs["small_var"] < BAR_LN_SMALL_VAR, errs
    assert errs["offset"] < BAR_LN_OFFSET, errs
    assert errs["small_var_eps_1e-5"] > 100 * BAR_LN_SMALL_VAR, errs                 # [0.74]
    assert errs["offset_one_pass_fp32"] > 2 * BAR_LN_OFFSET, errs                     # [0.75]


# ==================================================================================== bank and query writes
def _bank(eng):
    """The bank regions at the offsets carve_bank (api.cu) gives them; the carved total must equal bank_bytes."""
    OT, OTg = eng.O * eng.T, eng.O * eng.T_global
    names = ["hi", "lo", "mask16", "ist", "K", "M", "pose"]
    sizes = [OT * P * 1024 * 2, OT * P * 1024 * 2, OT * P * 4, (OTg if eng.ist_bank_global else OT) * P * 256 * 4,
             eng.O * 9 * 4, OTg * 9 * 4, OTg * 16 * 4]
    offs, total = _carve(sizes)
    assert total == eng.bank_bytes, "the bank layout changed"
    view = eng._bank_view()
    return {k: view[o:o + s] for k, o, s in zip(names, offs, sizes)}


def _workspace(eng):
    """The first workspace regions at the offsets carve_workspace (api.cu) gives them."""
    Bm = eng.max_batch
    names = ["q_hi", "q_lo", "q_mask16", "q_ist", "perm", "q_obj"]
    sizes = [Bm * P * 1024 * 2, Bm * P * 1024 * 2, Bm * P * 4, Bm * P * 256 * 4, Bm * 4, Bm * 4]
    offs, total = _carve(sizes)
    assert total <= eng.workspace_bytes
    off = (-eng._ws_mem.data_ptr()) % 1024
    view = eng._ws_mem[off:off + eng.workspace_bytes]
    return {k: view[o:o + s] for k, o, s in zip(names, offs, sizes)}


def _untiled(plane, n):
    """[n][c / 32][patch][c % 32] bf16 -> [n, 256, 1024]."""
    return plane.view(torch.bfloat16).view(n, 32, P, 32).permute(0, 2, 1, 3).reshape(n, P, 1024)


def _prefilled_engine(*args, **kw):
    eng = Engine(*args, **kw)
    eng._bank_view().fill_(0xFF)
    return eng


LAYOUTS = {"channel_major": _lib.LAYOUT_CHANNEL_MAJOR, "patch_major": _lib.LAYOUT_PATCH_MAJOR,
           "vit_tokens": _lib.LAYOUT_VIT_TOKENS}


@pytest.mark.parametrize("norm_passes", [0, 1, 2])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_descriptor_planes_each_layout_and_norm_passes(layout, norm_passes):
    """gp_bank_write of 3 templates into slots [1, 4) of object 1 (of 2 x 5), and gp_set_queries of the same
    descriptors: de-tiled hi + lo equals fp64 F.normalize (applied norm_passes times) per element within the bar,
    hi = bf16_rn(hi + lo) and |lo| <= ulp(hi) / 2, zero rows stay 0, the CLS row of raw ViT tokens (1e30) is never read,
    and every other slot keeps its 0xFF bytes.  The query planes equal the bank planes bit for bit."""
    n, O, T, obj, t0 = 3, 2, 5, 1, 1
    feat = _rand(n, P, 1024, seed=60) * 10 ** (6 * torch.rand(n, P, 1, generator=_gen(61), device=DEV) - 3)
    feat[0, 7] = 0.0
    feat[2, 200] = 0.0
    if layout == "channel_major":
        arg = feat.permute(0, 2, 1).reshape(n, 1024, 16, 16).contiguous()
    elif layout == "vit_tokens":
        arg = torch.cat([torch.full((n, 1, 1024), 1e30, device=DEV), feat], 1)
    else:
        arg = feat
    eng = _prefilled_engine(O, T, n, device=DEV)
    mask = torch.ones(n, 16, 16, device=DEV)
    eng.bank_write(obj, t0, arg, mask, norm_passes=norm_passes)
    eng.set_queries(arg, mask, torch.full((n,), obj, dtype=torch.int32, device=DEV), norm_passes=norm_passes)
    torch.cuda.synchronize(DEV)
    bank, ws = _bank(eng), _workspace(eng)
    slot = obj * T + t0
    per = P * 1024 * 2
    hi = _untiled(bank["hi"][slot * per:(slot + n) * per], n)
    lo = _untiled(bank["lo"][slot * per:(slot + n) * per], n)
    for name in ("hi", "lo"):
        assert bool((bank[name][:slot * per] == 0xFF).all()) and bool((bank[name][(slot + n) * per:] == 0xFF).all()), \
            f"{name} plane outside the written slots"
        assert torch.equal(ws["q_" + name][:n * per], bank[name][slot * per:(slot + n) * per]), f"query {name} plane"
    ref = feat.double()
    for _ in range(norm_passes):
        ref = F.normalize(ref, dim=-1)
    got = joined((hi, lo))
    nz = ref != 0
    assert bool((got[~nz] == 0).all()) and not bool(got.isnan().any()), "zero rows"
    assert bool((bits(hi[~nz]) == 0).all() and (bits(lo[~nz]) == 0).all())
    err = float(((got - ref).abs()[nz] / ref.abs()[nz]).max())
    _, e = torch.frexp(hi.float())
    half_ulp = torch.ldexp(torch.ones_like(lo, dtype=torch.float64), e.long() - 9)      # |hi| in [2^(e-1), 2^e)
    assert bool((lo.double().abs() <= half_ulp).all()), "|lo| > ulp(hi) / 2"
    # where rounding v - hi to bf16 lands lo on exactly half an ulp, hi + lo is a tie that rounds to the even neighbour
    below = lo.double().abs() < half_ulp
    assert torch.equal(bits((hi.float() + lo.float()).to(torch.bfloat16)[below]), bits(hi[below])), "hi != bf16_rn(hi + lo)"
    write_report(f"encoder_descriptors_{layout}_norm{norm_passes}.json", {"err": err, "ties": int((~below).sum())})
    assert err < BAR_DESC, f"descriptor error {err:.3e}"


MASK_SIZES = [(224, 224), (480, 640), (17, 23), (16, 16), (100, 37)]


@pytest.mark.parametrize("H,W", MASK_SIZES, ids=[f"{h}x{w}" for h, w in MASK_SIZES])
def test_mask16_is_nearest_interpolate_in_bank_and_queries(H, W):
    """sample_mask16 equals F.interpolate(size=16, mode="nearest") on the GPU exactly, in the bank (slots [1, 4) of
    object 0; the other slots keep 0xFF) and in the query workspace (q_mask16).  Mask values are random floats, so any
    wrong source pixel shows."""
    n, T = 3, 5
    mask = torch.rand(n, H, W, generator=_gen(H * 1000 + W), device=DEV)
    eng = _prefilled_engine(1, T, n, device=DEV)
    eng.bank_write(0, 1, torch.zeros(n, P, 1024, device=DEV), mask, norm_passes=0)
    eng.set_queries(torch.zeros(n, P, 1024, device=DEV), mask, torch.zeros(n, dtype=torch.int32, device=DEV), norm_passes=0)
    torch.cuda.synchronize(DEV)
    want = F.interpolate(mask[:, None], size=16, mode="nearest").reshape(n, P)
    m16 = _bank(eng)["mask16"].view(torch.float32).view(T, P)
    assert torch.equal(bits(m16[1:1 + n]), bits(want)), "bank mask16"
    assert bool((bits(m16[0]) == -1).all() and (bits(m16[1 + n:]) == -1).all()), "bank mask16 outside the slots"
    q = _workspace(eng)["q_mask16"].view(torch.float32).view(n, P)
    assert torch.equal(bits(q), bits(want)), "q_mask16"


def test_ist_transpose_into_local_and_global_ist_banks():
    """IST features channel-major [n, 256, 16, 16] are stored patch-major [n, 256 patches, 256] exactly, through
    bank_write and bank_write_ist (channel-major, and the channels-last view the trunk returns, stored as is); with
    ist_bank_global the slots are addressed by global template id.  Every other IST slot keeps its 0xFF bytes."""
    n = 2
    ist = _rand(n, 256, 16, 16, seed=70)
    want = ist.permute(0, 2, 3, 1).reshape(n, P, 256)
    view = ist.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)     # [n,16,16,256] memory seen as [n,256,16,16]
    zeros, ones = torch.zeros(n, P, 1024, device=DEV), torch.ones(n, 16, 16, device=DEV)

    def check_slots(eng, Ti, written):
        slots = _bank(eng)["ist"].view(torch.float32).view(eng.O * Ti, P, 256)
        for s in range(eng.O * Ti):
            if s in written:
                assert torch.equal(bits(slots[s]), bits(want[written[s]])), f"IST slot {s}"
            else:
                assert bool((bits(slots[s]) == -1).all()), f"IST slot {s} was written"

    eng = _prefilled_engine(2, 5, n, device=DEV)
    eng.bank_write(0, 3, zeros, ones, ist_feat=ist, norm_passes=0)         # slots 3, 4
    eng.bank_write_ist(1, 0, ist)                                         # slots 5, 6
    eng.bank_write_ist(1, 2, view)                                        # slots 7, 8 (patch-major, copied)
    torch.cuda.synchronize(DEV)
    check_slots(eng, 5, {3: 0, 4: 1, 5: 0, 6: 1, 7: 0, 8: 1})
    # shard 1 of 3 over 6 global templates: 2 descriptor slots per object, all 6 IST slots by global id
    g = _prefilled_engine(2, 2, n, device=DEV, shard_rank=1, shard_world=3, num_templates_global=6, ist_bank_global=True)
    g.bank_write_ist(0, 4, ist)
    g.bank_write_ist(1, 1, view)
    torch.cuda.synchronize(DEV)
    check_slots(g, 6, {4: 0, 5: 1, 7: 0, 8: 1})


def test_object_order_is_the_stable_argsort_of_the_clamped_ids():
    """gp_set_queries with B = 200 (two blocks of the object-order kernel), unsorted and repeated ids and ids outside
    [0, O) (-3, O + 5): perm is the stable argsort of the clamped ids, and q_obj holds the clamped ids."""
    O, B = 4, 200
    ids = torch.randint(-3, O + 6, (B,), generator=torch.Generator().manual_seed(80), dtype=torch.int32)
    ids[:4] = torch.tensor([O + 5, -3, O + 5, -3], dtype=torch.int32)
    assert (ids < 0).any() and (ids >= O).any()
    eng = Engine(O, 5, B, device=DEV, k=1)
    eng.set_queries(torch.zeros(B, P, 1024, device=DEV), torch.ones(B, 16, 16, device=DEV), ids, norm_passes=0)
    torch.cuda.synchronize(DEV)
    ws = _workspace(eng)
    clamped = ids.clamp(0, O - 1)
    assert torch.equal(ws["q_obj"].view(torch.int32).cpu(), clamped), "q_obj"
    assert torch.equal(ws["perm"].view(torch.int32).cpu(), torch.argsort(clamped, stable=True).to(torch.int32)), "perm"
