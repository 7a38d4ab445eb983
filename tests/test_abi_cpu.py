"""CPU-side checks of the drop-in boundary: the shared library builds/loads without a GPU and exports exactly the
symbols include/gigapose_b200.h declares; configuration errors are reported through the status/last-error channel."""
import ctypes as C
import os
import re

import pytest

from gigapose_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "gigapose_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gp_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree(lib):
    declared = _declared_functions()
    assert declared, "no functions parsed from the header"
    assert sorted(_lib.SYMBOLS) == declared
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/gigapose_b200.h but not exported"


def test_config_validation_needs_no_gpu(lib):
    cfg = _lib.GpConfig(abi_version=_lib.GP_ABI_VERSION, device=0, num_objects=8, num_templates=162,
                        num_templates_global=162, template_id_stride=1, template_id_offset=0, max_batch=32, top_k=5,
                        sim_threshold=0.5, patch_threshold=3, pixel_threshold=14, patch_size=14, precision=0)
    bank, ws = C.c_size_t(), C.c_size_t()
    assert lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws)) == 0
    # hi + lo bf16 planes == the fp32 bank of BASELINE.md (1.36 GB for 8 x 162) plus masks / IST features / poses
    assert bank.value >= 8 * 162 * 256 * 1024 * 4
    assert bank.value < 1.3 * (8 * 162 * 256 * (1024 * 4 + 256 * 4 + 4))
    cfg.top_k = 0
    assert lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws)) == -1
    assert b"top_k" in lib.gp_last_error()
    cfg.top_k = 5
    cfg.num_templates_global = 3
    assert lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws)) == -1
    cfg.num_templates_global = 162
    cfg.abi_version = 99
    assert lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws)) == -1
    assert b"ABI" in lib.gp_last_error()


def test_engine_refuses_cpu():
    from gigapose_b200.engine import Engine
    with pytest.raises(_lib.GigaPoseNativeError):
        Engine(1, 8, 1, device="cpu")


def test_product_code_never_imports_the_oracle():
    """oracle/ is test infrastructure; a product path routed through it would void every parity claim."""
    offenders = []
    for pkg in ("gigapose_b200", "src"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, pkg)):
            for f in files:
                if f.endswith(".py"):
                    txt = open(os.path.join(dirpath, f)).read()
                    if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M):
                        offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders


def test_every_kernel_launch_goes_through_the_counting_launcher():
    """gp_launch_count() (bench.py's `gpu_launches`) is kept by the one launcher in csrc/runtime.cu, so it cannot drift
    from the kernels really launched: no `<<<...>>>` launch in any source, and one place increments the counter."""
    csrc = os.path.join(ROOT, "gigapose_b200", "csrc")
    chevrons, increments = [], []
    for f in sorted(os.listdir(csrc)):
        txt = open(os.path.join(csrc, f)).read()
        if "<<<" in txt:
            chevrons.append(f)
        increments += [f] * len(re.findall(r"g_launches\s*(?:\+\+|\+=|\.fetch_add)|\+\+\s*g_launches", txt))
    assert not chevrons, chevrons
    assert increments == ["runtime.cu"], increments


def test_abi_v2_config_and_argument_checks_need_no_gpu(lib):
    """ABI 2: the replicated IST bank is sized by `ist_bank_global`; the multi-GPU and helper entry points reject bad
    arguments through the status channel without touching a device."""
    def sizes(**kw):
        cfg = _lib.GpConfig(abi_version=_lib.GP_ABI_VERSION, device=0, num_objects=21, num_templates=21,
                            num_templates_global=162, template_id_stride=8, template_id_offset=3, max_batch=128, top_k=5,
                            sim_threshold=0.5, patch_threshold=3, pixel_threshold=14, patch_size=14, precision=0, **kw)
        bank, ws = C.c_size_t(), C.c_size_t()
        rc = lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws))
        return rc, bank.value, ws.value
    rc0, bank_local, ws0 = sizes(ist_bank_global=0)
    rc1, bank_global, ws1 = sizes(ist_bank_global=1)
    assert rc0 == 0 and rc1 == 0 and ws0 == ws1
    extra = 21 * (162 - 21) * 256 * 256 * 4                       # the other shards' IST features, f32 patch-major
    assert extra <= bank_global - bank_local < extra + 4096
    assert sizes(ist_bank_global=2)[0] == -1 and b"ist_bank_global" in lib.gp_last_error()
    assert lib.gp_comm_init(None, None, 0, 1) == -1
    assert lib.gp_allgather(None, None, None, 0, None) == -1
    assert lib.gp_normalize_patch_tokens(0, None, None, None) == -1
    assert lib.gp_bank_write_ist(None, 0, 0, 1, None, 0, None) == -1


def test_nan_similarity_threshold_is_rejected(lib):
    """Every value fails `sim < NaN`, so a NaN threshold would silently keep every similarity; zero and negative
    thresholds are legal (the reference accepts any float)."""
    for thr, rc in ((float("nan"), -1), (0.0, 0), (-0.05, 0)):
        cfg = _lib.GpConfig(abi_version=_lib.GP_ABI_VERSION, device=0, num_objects=2, num_templates=9,
                            num_templates_global=9, template_id_stride=1, template_id_offset=0, max_batch=4, top_k=5,
                            sim_threshold=thr, patch_threshold=3, pixel_threshold=14, patch_size=14, precision=0)
        bank, ws = C.c_size_t(), C.c_size_t()
        assert lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws)) == rc, thr
        if rc:
            assert b"sim_threshold" in lib.gp_last_error()
            assert lib.gp_create(C.byref(cfg), None, None, None) == -1


def test_num_templates_beyond_the_topk_shared_memory_is_rejected(lib):
    """topk_select_kernel keeps one float per template in the default 48 KiB of shared memory: the largest accepted
    num_templates is MAX_NUM_TEMPLATES (12 032 = 47 KiB / 4), and one more fails at configuration time, naming
    num_templates, instead of at the first search."""
    for T, rc in ((_lib.MAX_NUM_TEMPLATES, 0), (_lib.MAX_NUM_TEMPLATES + 1, -1)):
        cfg = _lib.GpConfig(abi_version=_lib.GP_ABI_VERSION, device=0, num_objects=1, num_templates=T,
                            num_templates_global=T, template_id_stride=1, template_id_offset=0, max_batch=1, top_k=5,
                            sim_threshold=0.5, patch_threshold=3, pixel_threshold=14, patch_size=14, precision=0)
        bank, ws = C.c_size_t(), C.c_size_t()
        assert lib.gp_query_sizes(C.byref(cfg), C.byref(bank), C.byref(ws)) == rc, T
        if rc:
            assert b"num_templates" in lib.gp_last_error()
            assert lib.gp_create(C.byref(cfg), None, None, None) == -1
        else:
            assert bank.value >= T * 256 * 1024 * 4          # the two bf16 descriptor planes


def test_debug_kernel_entries_reject_bad_arguments_without_a_gpu(lib):
    """gp_debug_gemm / gp_debug_attention / gp_debug_layernorm check their arguments before they touch a device: an
    unsupported GEMM configuration fails with GP_ERR_INVALID and says why."""
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first

    def gemm(**kw):
        g = dict(M=256, N=512, K=64, bn=256, passes=3, mode=_lib.GEMM_ROWS_F32, swap=0, f16=0, acc_scale=0.0,
                 a_hi=fake, a_lo=fake, w_hi=fake, w_lo=fake, bias=fake, x=fake, out_hi=fake, out_lo=fake)
        g.update(kw)
        rc = lib.gp_debug_gemm(C.byref(_lib.GpDebugGemm(**g)), None)
        return rc, lib.gp_last_error()

    assert lib.gp_debug_gemm(None, None) == -1
    cases = [
        (dict(bn=128), b"bn"),                                            # the 128-column tiles are not instantiated
        (dict(bn=64), b"bn"),
        (dict(N=384), b"multiple of bn"),                                 # N % bn
        (dict(bn=192, N=576, mode=_lib.GEMM_ROWS_F32), b"192"),           # bn = 192 has the plane modes only
        (dict(K=48), b"K"),                                               # K % 32
        (dict(K=0), b"K"),
        (dict(passes=2), b"passes"),
        (dict(mode=9), b"mode"),
        (dict(swap=1, mode=_lib.GEMM_PLANES_GELU), b"swap"),              # swap with GELU
        (dict(swap=1, M=200, mode=_lib.GEMM_PLANES), b"swap"),            # swap needs whole 128-row tiles
        (dict(swap=1, f16=1, mode=_lib.GEMM_PLANES_RELU), b"swap"),
        (dict(f16=1, bn=192, N=576, mode=_lib.GEMM_PLANES_RELU), b"f16"),  # f16 with bn = 192
        (dict(f16=1, mode=_lib.GEMM_PLANES), b"f16"),
        (dict(M=0), b"M"),
        (dict(a_lo=None), b"null"),
        (dict(bias=None), b"null"),
        (dict(x=None), b"null output"),
        (dict(mode=_lib.GEMM_PLANES, out_lo=None), b"null output"),
        (dict(mode=_lib.GEMM_SCALE_RESIDUAL, gamma=None), b"gamma"),
        (dict(mode=_lib.GEMM_PLANES_ADD_RELU, res_hi=fake, res_lo=None), b"residual"),
        (dict(mode=_lib.GEMM_QKV_HEADS, N=1024, tokens_per_img=257, qkv_crop_stride=1), b"3072"),
        (dict(mode=_lib.GEMM_PATCH_EMBED, pos=fake, tokens_per_img=256, patches_per_img=256), b"patch"),
    ]
    for kw, word in cases:
        rc, msg = gemm(**kw)
        assert rc == -1 and word in msg, (kw, rc, msg)
    att = lambda b, stride, passes, hi=fake, lo=fake, oh=fake, ol=fake: lib.gp_debug_attention(b, stride, passes, hi, lo, oh, ol, None)
    assert att(0, 5, 3) == -1
    assert att(6, 5, 3) == -1 and b"crop_stride" in lib.gp_last_error()
    assert att(1, 5, 2) == -1 and b"passes" in lib.gp_last_error()
    for null in ("hi", "lo", "oh", "ol"):
        assert att(1, 5, 3, **{null: None}) == -1 and b"null" in lib.gp_last_error()
    ln = lambda M, x=fake, w=fake, b=fake, oh=fake, ol=fake: lib.gp_debug_layernorm(M, x, w, b, oh, ol, None)
    for null in ("x", "w", "b", "oh", "ol"):
        assert ln(8, **{null: None}) == -1 and b"null" in lib.gp_last_error()
    for M in (0, -5):
        assert ln(M) == -1 and b"M must be" in lib.gp_last_error()


def test_icp_debug_hooks_reject_bad_arguments_without_a_gpu(lib):
    """gp_debug_icp_select checks n, rank and its pointers, and gp_icp_refine checks the trace fields, before either
    touches a device; the trace record has the header's 456-byte layout."""
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first
    sel = lambda n, rank, bits=fake, out=fake: lib.gp_debug_icp_select(bits, n, rank, out, None)
    for n, rank, word in ((0, 0, b"n 0"), (-3, 0, b"n -3"), (5, 5, b"rank 5"), (5, -1, b"rank -1"),
                          (1, 1, b"rank 1")):
        assert sel(n, rank) == -1 and word in lib.gp_last_error(), (n, rank)
    for null in ("bits", "out"):
        assert sel(4, 0, **{null: None}) == -1 and b"null" in lib.gp_last_error()
    assert C.sizeof(_lib.GpIcpTrace) == 456 and _lib.GpIcpTrace.sums.offset == 80
    p = _lib.GpIcpParams(unit_per_m=1000.0, min_points=1000, num_levels=4, max_iters=100, rejection_scale=2.5,
                         max_residual=0.01, min_step_rad=1e-6, min_step_m=1e-6)
    for cap, count in ((0, fake), (-1, fake), (8, None)):
        p.debug = _lib.GpIcpDebug(trace=fake, trace_capacity=cap, trace_count=count)
        assert lib.gp_icp_refine(1, 1, 480, 640, *[fake] * 6, C.byref(p), *[fake] * 5, None) == -1, (cap, count)
        assert b"trace" in lib.gp_last_error()
