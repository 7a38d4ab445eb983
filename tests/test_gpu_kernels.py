"""-m gpu: the three tensor-core kernels alone -- vit_gemm_kernel, attention_tc_kernel and sim_search_kernel -- against a
plain fp64 statement of the same operation, at the shapes and edges where they would break.

The fp64 references are computed from the reconstructed split operands (hi + lo), so a measured error belongs to the
kernel and not to the rounding of its inputs.  GEMM errors are normalised per element by sum_k |a_k| |w_k| (+ the
magnitudes the epilogue adds): on that scale one dropped k-block or one missing split pass lands orders of magnitude
above the bars.  Each bar is about 4x the largest value measured on an H100 SXM (80 GB, 700 W power limit), stated
next to it.
Outputs are prefilled with sentinels (0xFFFF in bf16 / fp16 planes, NaN in fp32 rows); whatever a kernel must not
write has to keep them bit for bit."""
import ctypes as C

import pytest
import torch

from gigapose_b200 import _lib, synth
from gigapose_b200._lib import check
from oracle import port

from helpers import engine_from_case, write_report

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
SENT16 = -1                     # int16 0xFFFF: a NaN in bf16 and in fp16
NAN32 = 0x7FC00000              # bit pattern of torch's NaN fill

# --- bars: normalised errors, with the largest value measured on an H100 SXM (700 W limit) in brackets.  The GEMM's
# fp32 accumulation truncates, so the 3-pass rows sit near 1e-6 rather than at fp32 rounding.
BAR_ROWS = 2e-5                 # fp32 rows, 3 passes                             [4.6e-6]
BAR_PLANES_BF16 = 2.5e-5        # bf16 hi/lo output planes (+ ~2^-17 of the pair)  [6.5e-6]
BAR_PLANES_F16 = 2e-6           # fp16 hi/lo output planes (22-bit pairs)         [5.3e-7]
BAR_GELU = 3e-5                 # erf-GELU sweep, |err| / max(1, |GELU(x)|)       [7.5e-6]
# attention, |o - o64| / (P |v|).  The wgmma rows drop the lo*lo term of S = q k^T, an error that grows with the logit
# scale: x1 [6.5e-6], x8 [1.1e-4], x30 [3.9e-4].  Token 256 runs fp32 FMAs on the reconstructed planes: x1 [4.0e-6],
# x8 [7.1e-6]; at x30 its planted softmax is one-hot to fp32 precision [2.3e-15].
BAR_ATTN = {1: 2.5e-5, 8: 4.5e-4, 30: 1.5e-3}
BAR_ATTN_SIMT = {1: 1.6e-5, 8: 3e-5, 30: 1e-12}
BAR_TILES = 2e-5                # raw similarity tiles, fp32_split, K = 1024      [5.1e-6]


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV) * scale


def split(x, f16=False):
    """Caller-made operand planes: hi = round(x), lo = round(x - hi) in bf16 (or IEEE fp16)."""
    dt = torch.float16 if f16 else torch.bfloat16
    hi = x.to(dt)
    return hi.contiguous(), (x - hi.float()).to(dt).contiguous()


def joined(planes):
    return planes[0].double() + planes[1].double()


def sentinel_planes(shape, f16=False):
    dt = torch.float16 if f16 else torch.bfloat16
    return tuple(torch.full(shape, SENT16, dtype=torch.int16, device=DEV).view(dt) for _ in range(2))


def nan_rows(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def untouched(t):
    """Every element still holds its sentinel bit pattern."""
    if t.element_size() == 2:
        return bool((t.view(torch.int16) == SENT16).all())
    return bool((t.view(torch.int32) == NAN32).all())


def planes_untouched(planes):
    return untouched(planes[0]) and untouched(planes[1])


def bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def nerr(got, ref, den):
    return float(((got.double() - ref).abs() / den).max())


# ================================================================================================ GEMM
M_ = _lib
PLANE_MODES = (M_.GEMM_PLANES, M_.GEMM_PLANES_GELU, M_.GEMM_QKV_HEADS, M_.GEMM_PLANES_RELU, M_.GEMM_PLANES_ADD_RELU)
MODE_NAMES = {M_.GEMM_PLANES: "planes", M_.GEMM_PLANES_GELU: "gelu", M_.GEMM_SCALE_RESIDUAL: "scale_residual",
              M_.GEMM_PATCH_EMBED: "patch_embed", M_.GEMM_QKV_HEADS: "qkv_heads", M_.GEMM_PLANES_RELU: "relu",
              M_.GEMM_PLANES_ADD_RELU: "add_relu", M_.GEMM_ROWS_F32: "rows_f32", M_.GEMM_ROWS_F32_RELU: "rows_f32_relu"}


def run_gemm(a, w, bias, mode, *, out=None, x=None, bn=256, passes=3, swap=0, f16=0, acc_scale=0.0, gamma=None,
             pos=None, res=None, m_dev=None, tokens_per_img=0, patches_per_img=0, qkv_crop_stride=0):
    p = lambda t: None if t is None else t.data_ptr()
    out = out or (None, None)
    res = res or (None, None)
    g = _lib.GpDebugGemm(M=a[0].shape[0], N=w[0].shape[0], K=a[0].shape[1], bn=bn, passes=passes, mode=mode, swap=swap,
                         f16=f16, acc_scale=acc_scale, a_hi=p(a[0]), a_lo=p(a[1]), w_hi=p(w[0]), w_lo=p(w[1]),
                         out_hi=p(out[0]), out_lo=p(out[1]), bias=p(bias), gamma=p(gamma), x=p(x), pos=p(pos),
                         res_hi=p(res[0]), res_lo=p(res[1]), m_dev=p(m_dev), tokens_per_img=tokens_per_img,
                         patches_per_img=patches_per_img, qkv_crop_stride=qkv_crop_stride)
    check(_lib.load().gp_debug_gemm(C.byref(g), _stream()))
    torch.cuda.synchronize(DEV)


def product(a, w, bias, acc_scale=0.0, bias_per_row=False):
    """fp64 C = A W^T * scale + bias of the reconstructed planes, and the per-element scale sum_k |a||w| + |bias|."""
    A, W = joined(a), joined(w)
    s = acc_scale or 1.0
    b = bias.double()[:, None] if bias_per_row else bias.double()[None, :]
    return A @ W.T * s + b, A.abs() @ W.abs().T * s + b.abs()


def gelu64(v):
    return 0.5 * v * (1.0 + torch.special.erf(v / 2 ** 0.5))


def _operands(M, N, K, seed, f16=False):
    return split(_rand(M, K, seed=seed), f16), split(_rand(N, K, seed=seed + 1, scale=K ** -0.5), f16)


@pytest.mark.parametrize("bn", [192, 256])
@pytest.mark.parametrize("ntiles", [1, 3])
@pytest.mark.parametrize("K", [32, 160, 608, 4096])
@pytest.mark.parametrize("M", [1, 127, 129, 771])
def test_gemm_product_against_fp64(M, K, ntiles, bn):
    """The main loop at the edges of its tiling: M = 1 / 127 / 129 / 771 (partial 128-row tiles; the TMA zero-fills the
    missing A rows), K = 32 (one k-block, fewer than the 4 ring stages) to 4096, N = one or three bn-wide tiles.
    bn = 256 writes fp32 rows, bn = 192 (plane modes only) bf16 hi/lo planes.  Rows >= M keep their sentinels."""
    N = bn * ntiles
    a, w = _operands(M, N, K, seed=M * 7 + K)
    bias = _rand(N, seed=3, scale=0.5)
    ref, den = product(a, w, bias)
    if bn == 256:
        x = nan_rows(M + 64, N)
        run_gemm(a, w, bias, M_.GEMM_ROWS_F32, x=x, bn=bn)
        err, bar, tail_ok = nerr(x[:M], ref, den), BAR_ROWS, untouched(x[M:])
    else:
        out = sentinel_planes((M + 64, N))
        run_gemm(a, w, bias, M_.GEMM_PLANES, out=out, bn=bn)
        err, bar = nerr(joined(out)[:M], ref, den), BAR_PLANES_BF16
        tail_ok = planes_untouched((out[0][M:], out[1][M:]))
    write_report(f"kernels_gemm_product_M{M}_K{K}_N{N}_bn{bn}.json", {"err": err})
    assert tail_ok, "rows >= M were written"
    assert err < bar, f"normalised error {err:.3e}"


@pytest.mark.parametrize("bn,mode", [(256, M_.GEMM_ROWS_F32), (192, M_.GEMM_PLANES)])
def test_gemm_persistent_tiles_and_batch_invariance(bn, mode):
    """Enough rows for >= 3 tiles per persistent CTA on this device's SM count (the producer waits on ring_free_bar
    through several phases) and a last raster group with fewer than 16 m-tiles (tile_coords).  Row r of an M = 129 or
    M = 771 call is bit-identical to row r of the large call."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    num_m = sms + 1 if (sms + 1) % 16 else sms + 2
    M, N, K = (num_m - 1) * 128 + 77, 3 * bn, 608
    assert num_m * 3 >= 3 * sms and num_m % 16 != 0
    a, w = _operands(M, N, K, seed=11)
    bias = _rand(N, seed=12, scale=0.5)

    def run(m):
        sub = (a[0][:m], a[1][:m])
        if mode == M_.GEMM_ROWS_F32:
            x = nan_rows(m + 64, N)
            run_gemm(sub, w, bias, mode, x=x, bn=bn)
            assert untouched(x[m:])
            return x[:m]
        out = sentinel_planes((m + 64, N))
        run_gemm(sub, w, bias, mode, out=out, bn=bn)
        assert planes_untouched((out[0][m:], out[1][m:]))
        return torch.stack([bits(out[0][:m]), bits(out[1][:m])], -1)

    big = run(M)
    ref, den = product(a, w, bias)
    got = big if mode == M_.GEMM_ROWS_F32 else (big[..., 0].view(torch.bfloat16).double() + big[..., 1].view(torch.bfloat16).double())
    err = nerr(got, ref, den)
    write_report(f"kernels_gemm_persistent_bn{bn}.json", {"err": err, "M": M, "sms": sms})
    assert err < (BAR_ROWS if mode == M_.GEMM_ROWS_F32 else BAR_PLANES_BF16), f"normalised error {err:.3e}"
    for m in (129, 771):
        assert torch.equal(bits(run(m)), bits(big[:m])), f"rows of the M = {m} call differ from the large call"


# every (swap, bn, f16, mode) vit_gemm_kernel is instantiated for
COMBOS = ([(0, 256, 0, m) for m in MODE_NAMES] + [(0, 192, 0, m) for m in (M_.GEMM_PLANES, M_.GEMM_PLANES_RELU, M_.GEMM_PLANES_ADD_RELU)]
          + [(1, 256, 0, m) for m in (M_.GEMM_PLANES, M_.GEMM_PLANES_RELU, M_.GEMM_PLANES_ADD_RELU)]
          + [(0, 256, 1, m) for m in (M_.GEMM_PLANES_RELU, M_.GEMM_ROWS_F32_RELU)])


@pytest.mark.parametrize("swap,bn,f16,mode", COMBOS,
                         ids=[f"swap{s}-bn{b}-{'f16' if f else 'bf16'}-{MODE_NAMES[m]}" for s, b, f, m in COMBOS])
def test_gemm_epilogue_against_fp64(swap, bn, f16, mode):
    """Each instantiation against its epilogue formula in fp64: bias, erf-GELU, ReLU, residual planes + ReLU,
    x += gamma (acc + b), fp32 rows, the patch-embedding row remap + positional table (CLS rows untouched) and the
    head-major QKV scatter (checked against a reshape / permute).  swap = 1 writes the transposed planes [N, M]."""
    M, N, K = (256 if swap else 300), 2 * bn, 160
    if mode == M_.GEMM_QKV_HEADS:
        M, N = 3 * 257, 3072
    if mode == M_.GEMM_PATCH_EMBED:
        M, K = 2 * 256 + 100, 608
    a, w = _operands(M, N, K, seed=21 + mode, f16=bool(f16))
    bias = _rand(M if swap else N, seed=22, scale=0.5)
    ref, den = product(a, w, bias, bias_per_row=bool(swap))
    kw = dict(bn=bn, swap=swap, f16=f16)
    report = {}
    if mode in PLANE_MODES:
        oshape = (N + 64, M) if swap else (M + 64, N)
        if mode == M_.GEMM_QKV_HEADS:
            oshape = (3, 5, 16, 257, 64)
            kw.update(tokens_per_img=257, qkv_crop_stride=5)
        out = sentinel_planes(oshape, bool(f16))
        if mode == M_.GEMM_PLANES_ADD_RELU:
            res = split(_rand(*oshape, seed=23, scale=0.5))
            r = joined(res)
            r = r[:N].T if swap else r[:M]
            ref, den = ref + r, den + r.abs()
            kw["res"] = res
        run_gemm(a, w, bias, mode, out=out, **kw)
        if mode == M_.GEMM_PLANES_GELU:
            ref = gelu64(ref)
        if mode in (M_.GEMM_PLANES_RELU, M_.GEMM_PLANES_ADD_RELU):
            ref = ref.clamp(min=0)
        if mode == M_.GEMM_QKV_HEADS:
            want = ref.reshape(3, 257, 3, 16, 64).permute(2, 0, 3, 1, 4)
            scale = den.reshape(3, 257, 3, 16, 64).permute(2, 0, 3, 1, 4)
            got = joined((out[0][:, :3], out[1][:, :3]))
            err = nerr(got, want, scale)
            assert planes_untouched((out[0][:, 3:], out[1][:, 3:])), "crop slots >= 3 were written"
        else:
            got = joined(out)
            got = got[:N].T if swap else got[:M]
            err = nerr(got, ref, den)
            tail = (out[0][N:], out[1][N:]) if swap else (out[0][M:], out[1][M:])
            assert planes_untouched(tail), "rows beyond the output were written"
        bar = BAR_PLANES_F16 if f16 else BAR_PLANES_BF16
    elif mode == M_.GEMM_SCALE_RESIDUAL:
        x0 = _rand(M + 64, N, seed=24)
        gamma = _rand(N, seed=25, scale=0.3)
        x = x0.clone()
        run_gemm(a, w, bias, mode, x=x, gamma=gamma, **kw)
        g64 = gamma.double()[None, :]
        err = nerr(x[:M], x0[:M].double() + g64 * ref, g64.abs() * den + x0[:M].double().abs())
        assert torch.equal(bits(x[M:]), bits(x0[M:])), "rows >= M were written"
        bar = BAR_ROWS
    elif mode == M_.GEMM_PATCH_EMBED:
        pos = _rand(257, N, seed=26, scale=0.5)
        x = nan_rows(3 * 257, N)
        run_gemm(a, w, bias, mode, x=x, pos=pos, tokens_per_img=257, patches_per_img=256, **kw)
        m = torch.arange(M, device=DEV)
        rows = (m // 256) * 257 + 1 + m % 256
        p64 = pos.double()[1 + m % 256]
        err = nerr(x[rows], ref + p64, den + p64.abs())
        written = torch.zeros(3 * 257, dtype=torch.bool, device=DEV)
        written[rows] = True
        assert untouched(x[~written]), "CLS rows or rows past the last patch were written"
        bar = BAR_ROWS
    else:
        x = nan_rows(M + 64, N)
        run_gemm(a, w, bias, mode, x=x, **kw)
        if mode == M_.GEMM_ROWS_F32_RELU:
            ref = ref.clamp(min=0)
        err = nerr(x[:M], ref, den)
        assert untouched(x[M:]), "rows >= M were written"
        bar = BAR_ROWS
    report["err"] = err
    write_report(f"kernels_gemm_epilogue_swap{swap}_bn{bn}_f16{f16}_{MODE_NAMES[mode]}.json", report)
    assert err < bar, f"normalised error {err:.3e}"


@pytest.mark.parametrize("f16", [0, 1], ids=["bf16", "f16"])
def test_gemm_output_planes_are_the_rounded_value_and_residual(f16):
    """hi is the round-to-nearest bf16 (fp16) of the epilogue value and lo that of the residual, bit for bit; the
    value itself comes from the fp32-row form of the same GEMM.  The fp16 epilogue saturates |v| > 65504 to +-65504
    (not inf: the next layer's lo plane would turn it into NaN)."""
    M, N, K = 300, 512, 160
    a, w = _operands(M, N, K, seed=31, f16=bool(f16))
    bias = _rand(N, seed=32, scale=0.5)
    if f16:
        bias[:8], bias[8:16], bias[16:24] = 1e5, 7e4, 65519.0      # beyond the fp16 range (65519 still rounds to 65504)
    x = nan_rows(M, N)
    run_gemm(a, w, bias, M_.GEMM_ROWS_F32_RELU if f16 else M_.GEMM_ROWS_F32, x=x, f16=f16)
    dt = torch.float16 if f16 else torch.bfloat16
    modes = (M_.GEMM_PLANES_RELU,) if f16 else (M_.GEMM_PLANES, M_.GEMM_PLANES_RELU)
    for mode in modes:
        v = x.clamp(min=0) if mode == M_.GEMM_PLANES_RELU else x
        if f16:
            v = v.clamp(-65504.0, 65504.0)
        hi = v.to(dt)
        lo = (v - hi.float()).to(dt)
        out = sentinel_planes((M, N), bool(f16))
        run_gemm(a, w, bias, mode, out=out, f16=f16)
        assert torch.equal(bits(out[0]), bits(hi)), f"{MODE_NAMES[mode]}: hi plane is not round(v)"
        assert torch.equal(bits(out[1]), bits(lo)), f"{MODE_NAMES[mode]}: lo plane is not round(v - hi)"
        if f16:
            assert bool((out[0][:, :24].float() == 65504.0).all()) and bool((out[1][:, :24] == 0).all())


@pytest.mark.parametrize("rows", [0, 1, 299, 300, 400])
@pytest.mark.parametrize("f16,mode", [(0, M_.GEMM_ROWS_F32), (1, M_.GEMM_PLANES_RELU)], ids=["rows_f32", "f16_relu"])
def test_gemm_device_row_count(rows, f16, mode):
    """m_dev (the regressor's data-dependent row count, read on the device): rows < min(*m_dev, M) equal the
    unbounded call bit for bit, every other row keeps its sentinel."""
    M, N, K = 300, 512, 160
    a, w = _operands(M, N, K, seed=41, f16=bool(f16))
    bias = _rand(N, seed=42, scale=0.5)
    m_dev = torch.tensor([rows], dtype=torch.int32, device=DEV)

    def run(md):
        if mode == M_.GEMM_ROWS_F32:
            x = nan_rows(M, N)
            run_gemm(a, w, bias, mode, x=x, f16=f16, m_dev=md)
            return x
        out = sentinel_planes((M, N), bool(f16))
        run_gemm(a, w, bias, mode, out=out, f16=f16, m_dev=md)
        return torch.stack([bits(out[0]), bits(out[1])], -1)

    full, part = run(None), run(m_dev)
    n = min(rows, M)
    assert torch.equal(bits(part[:n]), bits(full[:n]))
    assert untouched(part[n:]) if mode == M_.GEMM_ROWS_F32 else bool((part[n:] == SENT16).all())


def test_gemm_acc_scale_undoes_a_scaled_weight():
    """acc_scale = 1/64 on a W scaled by 64 (the regressor's scheme, which keeps small fp16 weights out of the
    subnormal range): with bf16 planes the result equals the unscaled product bit for bit; with fp16 planes it stays
    within the fp32-row bar of the fp64 product."""
    M, N, K = 300, 512, 512
    A = _rand(M, K, seed=51)
    Wt = _rand(N, K, seed=52, scale=0.02)
    bias = _rand(N, seed=53, scale=0.1)
    x0, x1 = nan_rows(M, N), nan_rows(M, N)
    run_gemm(split(A), split(Wt), bias, M_.GEMM_ROWS_F32, x=x0)
    run_gemm(split(A), split(Wt * 64), bias, M_.GEMM_ROWS_F32, x=x1, acc_scale=1 / 64)
    assert torch.equal(bits(x0), bits(x1))
    a16, w16 = split(A, True), split(Wt * 64, True)
    x = nan_rows(M, N)
    run_gemm(a16, w16, bias, M_.GEMM_ROWS_F32_RELU, x=x, f16=1, acc_scale=1 / 64)
    ref, den = product(a16, w16, bias, acc_scale=1 / 64)
    err = nerr(x, ref.clamp(min=0), den)
    write_report("kernels_gemm_acc_scale_f16.json", {"err": err})
    assert err < BAR_ROWS, f"normalised error {err:.3e}"


def test_gemm_one_pass_is_bf16_and_three_passes_read_the_lo_planes():
    """passes = 1 (hi * hi only) lands within the bf16 bound (2^-8: each operand rounded to 2^-9) and at least 30x
    above passes = 3 [5.8e-4 against 1.0e-6]."""
    M, N, K = 300, 512, 1024
    a, w = _operands(M, N, K, seed=61)
    bias = _rand(N, seed=62, scale=0.5)
    ref, den = product(a, w, bias)
    errs = {}
    for passes in (1, 3):
        x = nan_rows(M, N)
        run_gemm(a, w, bias, M_.GEMM_ROWS_F32, x=x, passes=passes)
        errs[passes] = nerr(x, ref, den)
    write_report("kernels_gemm_passes.json", errs)
    assert errs[1] < 2 ** -8, errs
    assert errs[1] > 30 * errs[3], errs


def test_gemm_gelu_against_erf_over_minus_10_to_10():
    """erf-GELU epilogue against the exact function: A is an identity block, so the pre-activations are the W values,
    swept over [-10, 10].  Error = |hi + lo - GELU(x)| / max(1, |GELU(x)|)."""
    M = K = N = 256
    eye = torch.eye(K, device=DEV)
    a = split(eye)
    pre = torch.linspace(-10.0, 10.0, N * K, device=DEV).reshape(N, K)
    w = split(pre)
    bias = torch.zeros(N, device=DEV)
    out = sentinel_planes((M, N))
    run_gemm(a, w, bias, M_.GEMM_PLANES_GELU, out=out)
    ref = gelu64(joined(w).T)
    err = nerr(joined(out), ref, ref.abs().clamp(min=1.0))
    write_report("kernels_gemm_gelu_sweep.json", {"err": err})
    assert err < BAR_GELU, f"GELU error {err:.3e}"


# ============================================================================================ attention
PLANTED_ROWS = [0, 17, 63, 64, 130, 191, 200, 255, 256]       # rows whose maximum logit is key 256


def _qkv(b, stride, scale, seed, fill):
    """Head-major planes [3][stride][16][257][64]; crops >= b hold `fill` (+-1e30 with random signs, or 0)."""
    q = _rand(b, 16, 257, 64, seed=seed, scale=scale)
    k = _rand(b, 16, 257, 64, seed=seed + 1)
    v = _rand(b, 16, 257, 64, seed=seed + 2)
    k256 = k[:, :, 256:257]
    q[:, :, PLANTED_ROWS] = 0.5 * scale * k256 + _rand(b, 16, len(PLANTED_ROWS), 64, seed=seed + 3, scale=0.1 * scale)
    full = _rand(3, stride, 16, 257, 64, seed=seed + 4).sign() * fill
    full[:, :b] = torch.stack([q, k, v])
    return split(full)


def run_attention(b, stride, passes, planes):
    out = sentinel_planes((stride * 257, 1024))
    check(_lib.load().gp_debug_attention(b, stride, passes, planes[0].data_ptr(), planes[1].data_ptr(),
                                         out[0].data_ptr(), out[1].data_ptr(), _stream()))
    torch.cuda.synchronize(DEV)
    return out


def attention_ref(planes, b):
    x = joined(planes)
    q, k, v = x[0, :b], x[1, :b], x[2, :b]
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1)
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(b * 257, 1024)
    return rows(p @ v), rows(p @ v.abs()), p


def _attn_errs(out, ref, den, b):
    e = ((joined(out)[: b * 257] - ref).abs() / den).reshape(b, 257, 1024)
    return float(e[:, :256].max()), float(e[:, 256].max())


@pytest.mark.parametrize("scale", [1, 8, 30])
@pytest.mark.parametrize("b", [1, 3])
def test_attention_against_fp64(b, scale):
    """Softmax(q k^T / 8) v per (crop, head) against fp64, at logit scales x1, x8 and x30 (a peaked softmax), with
    rows whose maximum is key 256 (the n16 tail tile, masked down to its one real key).  Error = |o - o64| / (P |v|).
    The unused crop slots of the planes hold +-1e30: the last head of the last crop reads its 15 padding key / value
    rows from there, so the output must be bit-identical to the same call with those slots zeroed, and only the
    b crops' rows may be written."""
    stride = 5
    planes = _qkv(b, stride, scale, seed=70 + b, fill=1e30)
    zeroed = tuple(t.clone() for t in planes)
    for t in zeroed:
        t[:, b:] = 0
    out = run_attention(b, stride, 3, planes)
    out0 = run_attention(b, stride, 3, zeroed)
    ref, den, p = attention_ref(planes, b)
    assert bool((p[:, :, PLANTED_ROWS].argmax(-1) == 256).all())
    assert planes_untouched((out[0][b * 257:], out[1][b * 257:])), "rows of crops >= b were written"
    assert torch.equal(bits(out[0]), bits(out0[0])) and torch.equal(bits(out[1]), bits(out0[1])), \
        "the padding rows read past a head changed the result"
    e_tc, e_simt = _attn_errs(out, ref, den, b)
    write_report(f"kernels_attention_b{b}_x{scale}.json", {"tensor_rows": e_tc, "token256": e_simt})
    assert e_tc < BAR_ATTN[scale], f"tokens 0..255: {e_tc:.3e}"
    assert e_simt < BAR_ATTN_SIMT[scale], f"token 256: {e_simt:.3e}"


def test_attention_one_pass_is_bf16_and_three_passes_read_the_lo_planes():
    """passes = 1 (plain bf16 products) lands within the bf16 bound and at least 30x above passes = 3
    [tokens 0..255: 4.6e-3 against 7.0e-6]."""
    b, stride = 3, 5
    planes = _qkv(b, stride, 1, seed=90, fill=0.0)
    ref, den, _ = attention_ref(planes, b)
    errs = {p: _attn_errs(run_attention(b, stride, p, planes), ref, den, b) for p in (1, 3)}
    write_report("kernels_attention_passes.json", {str(k): v for k, v in errs.items()})
    assert errs[1][0] < 2 ** -6 and errs[1][1] < 2 ** -6, errs
    assert errs[1][0] > 30 * errs[3][0], errs


# =========================================================================================== similarity
ROW_TIES = ((4, 5, 5), (1, 202, 202))       # (s_lo, s_hi, query row t): template patches s_lo == s_hi, t's best match
COL_TIES = ((3, 11), (20, 100), (130, 250))  # query patches t_lo == t_hi, best match of template patch s = t_lo
CROSS_HALF = (50, 178)                       # t_lo in the first t-half, t_hi in the second (accumulated in reverse K order)


def _tie_case(cross_half=False):
    """B = 37 queries (one full and one partial 32-query chunk) over O = 2 objects (25 / 12 queries) x T = 9 templates,
    with planted exact ties.  Planted matches are ~0.99: far from every threshold tested."""
    labels = torch.tensor([1] * 25 + [2] * 12)[torch.randperm(37, generator=torch.Generator().manual_seed(5))]
    case = synth.make_feature_case(B=37, O=2, T=9, seed=8, labels=labels)
    g = torch.Generator().manual_seed(9)
    # template n carries noise 0.05 + 0.1 n / T: the per-template scores then differ by far more than the kernel error
    sig = (0.05 + 0.1 * torch.arange(case.T) / case.T)[None, :, None]
    noisy = lambda u, *shape, s=0.1: torch.nn.functional.normalize(u + s * torch.randn(*shape, 1024, generator=g) / 32, dim=-1)
    o = case.q_label - 1
    pairs = list(COL_TIES) + ([CROSS_HALF] if cross_half else [])
    for s_lo, s_hi, t in ROW_TIES:
        u = torch.nn.functional.normalize(torch.randn(case.O, 1024, generator=g), dim=-1)
        tmpl = noisy(u[:, None], case.O, case.T, s=sig)
        case.bank_feat[:, :, s_lo] = tmpl
        case.bank_feat[:, :, s_hi] = tmpl
        case.q_feat[:, t] = noisy(u[o], case.B)
        case.bank_mask16[:, :, [s_lo, s_hi]] = 1
        case.q_mask16[:, t] = 1
    for t_lo, t_hi in pairs:
        u = torch.nn.functional.normalize(torch.randn(case.O, 1024, generator=g), dim=-1)
        q = noisy(u[o], case.B)
        case.q_feat[:, t_lo] = q
        case.q_feat[:, t_hi] = q
        case.bank_feat[:, :, t_lo] = noisy(u[:, None], case.O, case.T, s=sig)
        case.q_mask16[:, [t_lo, t_hi]] = 1
        case.bank_mask16[:, :, t_lo] = 1
    return case


def test_similarity_tiles_against_fp64_over_two_query_chunks():
    """Raw fp32 tiles of B = 37 queries x 9 templates (333 items: more than two per CTA, so the reversed-K second
    t-half runs on a CTA's second and third item; the second query chunk is partial) against an fp64 einsum.
    Duplicate query rows 50 / 178 sit in different t-halves; whether the kernel keeps them equal is recorded, not
    asserted: the second half accumulates K in reverse order, and on the H100 84 589 of the 85 248 pairs came out
    unequal, by at most 1.5e-6."""
    case = _tie_case(cross_half=True)
    eng = engine_from_case(case)
    eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1)
    tiles = eng.debug_sim_tiles()
    order = torch.argsort(case.q_label, stable=True)
    q = torch.nn.functional.normalize(case.q_feat.to(DEV, torch.float64), dim=-1)[order.to(DEV)]
    bank = torch.nn.functional.normalize(case.bank_feat.to(DEV, torch.float64), dim=-1)
    err = 0.0
    for n in range(case.T):
        ref = torch.einsum("btc,bsc->bts", q, bank[(case.q_label[order] - 1).to(DEV), n])
        err = max(err, float((tiles[n].double() - ref).abs().max()))
    t_lo, t_hi = CROSS_HALF
    a, b = tiles[:, :, t_lo], tiles[:, :, t_hi]
    differ = (a != b)
    write_report("kernels_sim_tiles.json", {"err": err, "cross_half_pairs": int(differ.numel()),
                                            "cross_half_unequal": int(differ.sum()),
                                            "cross_half_max_diff": float((a - b).abs().max())})
    assert err < BAR_TILES, f"max |sim - fp64| = {err:.3e}"


@pytest.mark.parametrize("thr", [0.5, 0.0, -0.05, 0.95])
def test_similarity_outputs_exact_with_ties_and_thresholds(thr):
    """Every integer output of the similarity search (id_src, tar_pts, src_pts) equals port.similarity_search exactly
    on the B = 37 tie case: the lower s wins a row tie (s = 4 / 5 in one lane, s = 1 / 202 in different lanes), the
    lower t wins a column tie (t = 3 / 11: rows t0 and t0 + 8 of one lane; 20 / 100: two warpgroups; 130 / 250: second
    t-half).  Thresholds <= 0 let negative values and -0.0 (masked patches) through, which the column arg-max has to
    order like torch.max."""
    case = _tie_case()
    eng = engine_from_case(case, sim_threshold=thr)
    eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1)
    m = {k: v.cpu() for k, v in eng.sim_topk().items()}
    ri = synth.to_reference_layout(case)
    ref = port.similarity_search(ri["src_feats"], ri["tar_feat"], ri["src_masks"], ri["tar_mask"], sim_threshold=thr,
                                 return_intermediates=True)
    # the planted ties are live: the tie rows / columns pick the lower index in the reference itself
    for s_lo, _, t in ROW_TIES:
        assert bool((ref["idx_tar2src"][:, :, t] == s_lo).all())
    for t_lo, _ in COL_TIES:
        assert bool((ref["idx_src2tar"][:, :, t_lo] == t_lo).all())
    bad = {k: int((m[k] != ref[k]).sum()) for k in ("id_src", "tar_pts", "src_pts") if not torch.equal(m[k], ref[k])}
    assert not bad, f"entries differing from the oracle: {bad}"
    assert torch.allclose(m["score_src"], ref["score_src"], atol=2e-6)
    assert torch.allclose(m["score_pts"], ref["score_pts"], atol=2e-6)
