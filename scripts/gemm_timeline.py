"""Per-tile cycle timeline of vit_gemm_kernel (CTA 0) for the four ViT-L linears at M = 32 x 257 tokens.

    python scripts/gemm_timeline.py [--lib path/to/libgigapose_b200.so]

For each shape (qkv, proj, fc1, fc2) one stamped launch of gp_debug_gemm on seeded operands, then
gp_debug_gemm_timeline.  Prints one JSON line with, per shape and in SM clocks, the medians of
  mma_span      first k-block landed -> last MMA retired (MMA start -> retired where the library has no landing stamp)
  epilogue_span epilogue start -> end
  tile_gap      end of a tile's epilogue -> the next tile's first k-block landed (0 when it had landed already)
and idle_frac, the share of CTA 0's time (kernel start -> last epilogue end) with no MMA in flight, together with
the card name, its power limit and max SM clock.  A library without the `stamp` field only stamps its qkv launch.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gigapose_b200 import _lib  # noqa: E402

TOK, CROPS, DIM, MLP = 257, 32, 1024, 4096
M = TOK * CROPS
SHAPES = {   # name: (N, K, mode)
    "qkv": (3 * DIM, DIM, _lib.GEMM_QKV_HEADS),
    "proj": (DIM, DIM, _lib.GEMM_SCALE_RESIDUAL),
    "fc1": (MLP, DIM, _lib.GEMM_PLANES_GELU),
    "fc2": (DIM, MLP, _lib.GEMM_SCALE_RESIDUAL),
}
STAMP_TILES = 15


def open_lib(path: str) -> C.CDLL:
    lib = C.CDLL(path)
    for name, (res, args) in _lib.SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def call(lib, status):
    if status != 0:
        raise RuntimeError(lib.gp_last_error().decode())


def planes(rows, cols, gen, scale=1.0):
    x = torch.randn(rows, cols, generator=gen, device="cuda") * scale
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def make_case(name, seed=0):
    """Seeded operands and a GpDebugGemm for one ViT linear (tensors are returned to keep them alive)."""
    N, K, mode = SHAPES[name]
    gen = torch.Generator(device="cuda").manual_seed(seed)
    a, w = planes(M, K, gen), planes(N, K, gen, 0.03)
    bias = torch.randn(N, generator=gen, device="cuda") * 0.1
    keep = {"a": a, "w": w, "bias": bias}
    g = dict(M=M, N=N, K=K, bn=256, passes=3, mode=mode, a_hi=a[0].data_ptr(), a_lo=a[1].data_ptr(),
             w_hi=w[0].data_ptr(), w_lo=w[1].data_ptr(), bias=bias.data_ptr())
    if mode == _lib.GEMM_SCALE_RESIDUAL:
        keep["gamma"] = torch.rand(N, generator=gen, device="cuda")
        keep["x"] = torch.randn(M, N, generator=gen, device="cuda")
        g.update(gamma=keep["gamma"].data_ptr(), x=keep["x"].data_ptr())
    else:
        keep["out"] = (torch.empty(M, N, dtype=torch.bfloat16, device="cuda"),
                       torch.empty(M, N, dtype=torch.bfloat16, device="cuda"))
        g.update(out_hi=keep["out"][0].data_ptr(), out_lo=keep["out"][1].data_ptr())
    if mode == _lib.GEMM_QKV_HEADS:
        g.update(tokens_per_img=TOK, qkv_crop_stride=CROPS)
    return keep, g


def summarize(s, n_tiles):
    t = min(n_tiles, STAMP_TILES)
    start = [s[4 * i] for i in range(t)]
    done = [s[4 * i + 1] for i in range(t)]
    epi0 = [s[4 * i + 2] for i in range(t)]
    epi1 = [s[4 * i + 3] for i in range(t)]
    landed = [s[64 + i] for i in range(t)]
    has_landed = all(start[i] <= landed[i] <= done[i] for i in range(t))
    mma_from = landed if has_landed else start
    total = epi1[t - 1] - s[63]
    busy = sum(done[i] - mma_from[i] for i in range(t))
    out = {"tiles_cta0": n_tiles, "tiles_stamped": t,
           "mma_span": statistics.median(done[i] - mma_from[i] for i in range(t)),
           "epilogue_span": statistics.median(epi1[i] - epi0[i] for i in range(t)),
           "tile_gap": (statistics.median(max(0, landed[i] - epi1[i - 1]) for i in range(1, t))
                        if has_landed and t > 1 else None),
           "cta0_clocks": total, "idle_frac": round(1.0 - busy / total, 4) if t == n_tiles else None}
    return out


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timeline(lib, sms):
    res = {}
    for name in SHAPES:
        keep, g = make_case(name)
        stamps = (C.c_longlong * 128)()
        call(lib, lib.gp_debug_gemm_timeline(stamps))
        before = stamps[63]
        dbg = _lib.GpDebugGemm(**g, stamp=1)
        call(lib, lib.gp_debug_gemm(C.byref(dbg), None))          # warm-up (module load, attribute set-up)
        call(lib, lib.gp_debug_gemm(C.byref(dbg), None))
        call(lib, lib.gp_debug_gemm_timeline(stamps))
        if stamps[63] == before:
            res[name] = None                                        # this library does not stamp the shape
            continue
        N = SHAPES[name][0]
        tiles = ((M + 127) // 128) * (N // 256)
        grid = min(tiles, sms)
        res[name] = summarize(list(stamps), len(range(0, tiles, grid)))
        del keep
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=_lib.LIB_PATH)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    lib = open_lib(os.path.abspath(args.lib))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps({"gpu": gpu_info(), "lib": os.path.relpath(os.path.abspath(args.lib), ROOT), "M": M,
                      "shapes": timeline(lib, sms)}))


if __name__ == "__main__":
    main()
