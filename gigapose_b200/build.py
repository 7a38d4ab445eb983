"""Builds libgigapose_b200.so in-tree with nvcc for sm_90a (no JIT cache: the library is built in place by build())."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgigapose_b200.so")
SOURCES = ["runtime.cu", "api.cu", "sim_search.cu", "prep.cu", "ist_mlp.cu", "ransac_pose.cu", "vit_gemm.cu", "vit_ops.cu", "vit_attention_tc.cu", "vit_api.cu", "ist_trunk.cu", "preprocess.cu", "render.cu", "depth_icp.cu", "depth_score.cu", "bop_eval.cu", "depth_teaser.cu", "vis.cu", "onboard.cu", "reconstruct.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
# sources whose contract states every floating-point operation rounds once (no multiply-add contraction)
SOURCE_FLAGS = {"depth_teaser.cu": ["-fmad=false"], "onboard.cu": ["-fmad=false"],
                "reconstruct.cu": ["-fmad=false"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(HERE), "include", "gigapose_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, *SOURCE_FLAGS.get(src, []), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, pr in procs:
        out, _ = pr.communicate()
        if verbose or pr.returncode != 0:
            print(out)
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-lcudart"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
