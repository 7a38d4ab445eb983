"""A/B comparison of two builds of libgigapose_b200.so in one process: outputs and speed of vit_gemm_kernel.

    python scripts/gemm_ab.py --a path/to/parent/libgigapose_b200.so [--b gigapose_b200/libgigapose_b200.so]
                              [--rounds 5]

1. For each of the 17 (swap, bn, f16, mode) instantiations: one gp_debug_gemm launch per build on the same seeded
   operands; the outputs must be byte-identical.
2. Timing with CUDA events, A and B alternating in every round: each instantiation (20 launches per sample),
   gp_vit_time_linears over 32 crops (ViT-L/14, random weights) and the IST trunk forward over 32 crops.  Prints
   medians and spreads (max - min) per build, and the A/A spread (the two halves of A's samples).
One JSON line; the card name, power limit and max SM clock are part of it.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from gigapose_b200 import _lib  # noqa: E402
from gemm_timeline import call, gpu_info, open_lib, planes  # noqa: E402

L = _lib
# (swap, bn, f16, mode): every instantiation vit_gemm.cu has
INSTANCES = [(0, 256, 0, m) for m in (L.GEMM_PLANES, L.GEMM_PLANES_GELU, L.GEMM_SCALE_RESIDUAL, L.GEMM_PATCH_EMBED,
                                      L.GEMM_QKV_HEADS, L.GEMM_PLANES_RELU, L.GEMM_PLANES_ADD_RELU, L.GEMM_ROWS_F32,
                                      L.GEMM_ROWS_F32_RELU)]
INSTANCES += [(0, 192, 0, m) for m in (L.GEMM_PLANES, L.GEMM_PLANES_RELU, L.GEMM_PLANES_ADD_RELU)]
INSTANCES += [(0, 256, 1, m) for m in (L.GEMM_PLANES_RELU, L.GEMM_ROWS_F32_RELU)]
INSTANCES += [(1, 256, 0, m) for m in (L.GEMM_PLANES, L.GEMM_PLANES_RELU, L.GEMM_PLANES_ADD_RELU)]
PLANE_MODES = (L.GEMM_PLANES, L.GEMM_PLANES_GELU, L.GEMM_QKV_HEADS, L.GEMM_PLANES_RELU, L.GEMM_PLANES_ADD_RELU)


def make_case(swap, bn, f16, mode, seed):
    """Seeded operands at a size the pipeline runs (a partial last row tile where the form allows one)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if swap:
        M, N, K = 128, 8192, 1152                      # 128 output channels x 8192 pixels, 3x3x128 filter taps
    elif mode == L.GEMM_PATCH_EMBED:
        M, N, K = 32 * 256, 1024, 608
    else:
        M, N, K = 32 * 257, (3072 if mode == L.GEMM_QKV_HEADS else 1152 if bn == 192 else 1024), 1024
    if f16:
        def pl(r, c, s=1.0):
            x = torch.randn(r, c, generator=gen, device="cuda") * s
            hi = x.half()
            return hi, (x - hi.float()).half()
    else:
        pl = lambda r, c, s=1.0: planes(r, c, gen, s)
    a, w = pl(M, K), pl(N, K, 0.03)
    bias = torch.randn(M if swap else N, generator=gen, device="cuda") * 0.1
    keep = {"a": a, "w": w, "bias": bias}
    g = dict(M=M, N=N, K=K, bn=bn, passes=3, mode=mode, swap=swap, f16=f16, a_hi=a[0].data_ptr(), a_lo=a[1].data_ptr(),
             w_hi=w[0].data_ptr(), w_lo=w[1].data_ptr(), bias=bias.data_ptr())
    out_shape = (N, M) if swap else (M, N)
    if mode in PLANE_MODES:
        dt = torch.float16 if f16 else torch.bfloat16
        keep["out"] = (torch.zeros(out_shape, dtype=dt, device="cuda"), torch.zeros(out_shape, dtype=dt, device="cuda"))
        g.update(out_hi=keep["out"][0].data_ptr(), out_lo=keep["out"][1].data_ptr())
    else:
        rows = 32 * 257 if mode == L.GEMM_PATCH_EMBED else M
        keep["x"] = torch.randn(rows, N, generator=gen, device="cuda")
        keep["x0"] = keep["x"].clone()
        g.update(x=keep["x"].data_ptr())
    if mode == L.GEMM_SCALE_RESIDUAL:
        keep["gamma"] = torch.rand(N, generator=gen, device="cuda")
        g.update(gamma=keep["gamma"].data_ptr())
    if mode == L.GEMM_PATCH_EMBED:
        keep["pos"] = torch.randn(257, N, generator=gen, device="cuda")
        g.update(pos=keep["pos"].data_ptr(), tokens_per_img=257, patches_per_img=256)
    if mode == L.GEMM_QKV_HEADS:
        g.update(tokens_per_img=257, qkv_crop_stride=32)
    if mode == L.GEMM_PLANES_ADD_RELU:
        keep["res"] = pl(*out_shape)
        g.update(res_hi=keep["res"][0].data_ptr(), res_lo=keep["res"][1].data_ptr())
    if acc_scale := (0.25 if f16 else 0.0):
        g.update(acc_scale=acc_scale)
    return keep, _lib.GpDebugGemm(**g)


def outputs(keep):
    if "out" in keep:
        return [t.clone() for t in keep["out"]]
    out = keep["x"].clone()
    keep["x"].copy_(keep["x0"])                        # the residual modes update x in place
    return [out]


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def stats(a, b):
    h = len(a) // 2
    med = statistics.median
    return {"a_ms": round(med(a), 4), "b_ms": round(med(b), 4), "a_spread": round(max(a) - min(a), 4),
            "b_spread": round(max(b) - min(b), 4), "aa_diff": round(abs(med(a[:h]) - med(a[h:])), 4),
            "speedup": round(med(a) / med(b), 4)}


def vit_and_trunk(lib):
    """(gp_vit_time_linears over 32 crops, IST trunk forward over 32 crops) engines built on `lib`."""
    from gigapose_b200.ist_trunk import NativeISTTrunk
    from gigapose_b200.vit import DinoVisionTransformer
    from gigapose_b200.vit_engine import NativeViT
    from src.models.network.resnet import ResNet
    _lib._lib = lib                                    # the engines bind the library _lib.load() returns
    torch.manual_seed(0)
    vit = NativeViT(DinoVisionTransformer(depth=24).cuda(), "cuda:0", max_crops=32)
    net = ResNet(dict(n_heads=0, input_dim=3, input_size=256, initial_dim=128, block_dims=[128, 192, 256, 512],
                      descriptor_size=256)).cuda().eval()
    trunk = NativeISTTrunk(net, "cuda:0", max_crops=32)
    crops = torch.randn(32, 3, 224, 224, device="cuda")
    _lib._lib = None
    return vit, trunk, crops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="library A (the parent build)")
    ap.add_argument("--b", default=_lib.LIB_PATH, help="library B (this tree's build)")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    libs = {"a": open_lib(os.path.abspath(args.a)), "b": open_lib(os.path.abspath(args.b))}
    result = {"gpu": gpu_info(), "rounds": args.rounds, "gemm": {}}

    identical = True
    times = {}
    for i, inst in enumerate(INSTANCES):
        name = "swap%d_bn%d_f16%d_mode%d" % inst
        keep, dbg = make_case(*inst, seed=100 + i)
        outs = {}
        for k, lib in libs.items():
            call(lib, lib.gp_debug_gemm(C.byref(dbg), None))
            torch.cuda.synchronize()
            outs[k] = outputs(keep)
        same = all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(outs["a"], outs["b"]))
        identical &= same
        result["gemm"][name] = {"identical": same}
        times[name] = {"a": [], "b": []}
        fns = {k: (lambda lib=lib: call(lib, lib.gp_debug_gemm(C.byref(dbg), None))) for k, lib in libs.items()}
        for _ in range(args.rounds):
            for k in ("a", "b"):
                times[name][k].append(timed(fns[k], 20))
        result["gemm"][name].update(stats(times[name]["a"], times[name]["b"]))
        del keep
    result["all_identical"] = identical

    engines = {k: vit_and_trunk(lib) for k, lib in libs.items()}
    lin, tr = {"a": [], "b": []}, {"a": [], "b": []}
    for k, (vit, trunk, crops) in engines.items():      # warm-up
        vit.time_linears(32, iters=2)
        trunk.forward(crops)
    for _ in range(args.rounds):
        for k, (vit, trunk, crops) in engines.items():
            lin[k].append(vit.time_linears(32, iters=5))
            tr[k].append(timed(lambda: trunk.forward(crops), 5))
    result["vit_time_linears_32"] = stats(lin["a"], lin["b"])
    result["ist_trunk_forward_32"] = stats(tr["a"], tr["b"])
    print(json.dumps(result))


if __name__ == "__main__":
    main()
