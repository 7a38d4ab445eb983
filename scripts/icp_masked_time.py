"""Depth refinement with and without the detection masks (row f11) on the LM-O- and HOPE-shaped images of
scripts/bop_refine_time.py (640 x 480 with 8 instances, 1920 x 1080 with 18; the same meshes, poses and perturbations,
generated from a seed, kept on the device instead of a PNG).  Each instance's mask is its visible pixels, given as COCO
run-length encoding.  Per image, for H = 1 and 5 hypotheses per instance:
  maskless  bop_run's default: gp_icp_prepare_scene + gp_icp_refine with the threshold rule
  masked    gp_icp_masked_decode (decode), gp_icp_prepare_masked_scene (scene), gp_icp_refine_masked (icp)
with CUDA events, medians of 5 repetitions after a warm-up; the renders of the coarse poses are made once, outside the
timed stages.  Also: the mean iterations per ICP level, the accepted (status OK) counts, and the peak device memory of
one refinement above what the inputs hold.  Prints the card's name, power limit and maximum SM clock.

    python scripts/icp_masked_time.py [--out results/icp_masked_time.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bop_refine_time import SHAPES  # noqa: E402
from gigapose_b200 import icp, render  # noqa: E402
from icp_time import bumpy, perturbed, rodrigues  # noqa: E402
from oracle import bop_run_port  # noqa: E402

DEV = "cuda:0"
REPS = 5


def make_image(shape, meshes, rng):
    """Depth f32 [1,H,W] of the shape's grid in front of a plane at 1 m, labels, truth, visible masks [n,H,W]."""
    H, W = shape["size"]
    K = np.array(shape["K"], np.float32)
    depth = torch.zeros(H, W, device=DEV)
    owner = torch.full((H, W), -1, dtype=torch.int64, device=DEV)
    labels, truth = [], []
    for j, (x, y) in enumerate(shape["grid"]):
        o = j % len(meshes)
        T = np.eye(4, dtype=np.float32)
        T[:3, :3] = rodrigues(rng.normal(size=3))
        T[:3, 3] = (x, y, rng.uniform(750, 850))
        d = render.render_templates(meshes[o], torch.as_tensor(T)[None], K, size=(H, W), device=DEV)["depth"][0]
        front = (d > 0) & ((depth == 0) | (d < depth))
        depth = torch.where(front, d, depth)
        owner = torch.where(front, torch.full_like(owner, j), owner)
        labels.append(o)
        truth.append(T)
    depth = torch.where(depth > 0, depth, torch.full_like(depth, 1000.0)).round()
    masks = torch.stack([owner == j for j in range(len(labels))])
    return depth[None].contiguous(), np.array(labels), np.stack(truth), masks


def _stats(iters, status, L):
    it = iters.cpu().numpy()
    return dict(mean_iterations_per_level={str(lv): float(it[:, lv].mean()) for lv in range(L)},
                at_max_iters_per_level={str(lv): int((it[:, lv] == 100).sum()) for lv in range(L)},
                accepted=int((status == 0).sum()), statuses=np.bincount(status.cpu().numpy(), minlength=6).tolist())


def time_image(dm, labels, truth, depth, K, masks, hyp, rng):
    H, W = depth.shape[1:]
    n_det = len(labels)
    T0 = torch.as_tensor(perturbed(truth, hyp, rng)).to(DEV)
    n = T0.shape[0]
    lab = torch.as_tensor(np.repeat(labels, hyp))
    R, boxes = icp.render_hypotheses(dm, lab, T0, K, torch.zeros(n, dtype=torch.int64), H, W)
    counts = [bop_run_port.binary_mask_to_rle(m)["counts"] for m in masks.cpu().numpy()]
    rle = (np.concatenate(counts).astype(np.int32), np.concatenate([[0], np.cumsum([len(c) for c in counts])]))
    fi = torch.zeros(n, dtype=torch.int32, device=DEV)
    di = torch.as_tensor(np.repeat(np.arange(n_det), hyp), dtype=torch.int32).to(DEV)
    iters = torch.zeros(n, 4, dtype=torch.int32, device=DEV)
    out = {}
    torch.cuda.synchronize()
    # maskless
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ms_list = []
    for rep in range(REPS + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ws = torch.empty(icp.workspace_bytes(1, n, H, W), dtype=torch.uint8, device=DEV)
        ev[0].record()
        icp.prepare_scene(depth, K, ws)
        _, status, _, _ = icp.refine_rendered(depth, K, fi, R, boxes, T0, None, ws, debug=dict(iterations=iters))
        ev[1].record()
        torch.cuda.synchronize()
        if rep:
            ms_list.append(ev[0].elapsed_time(ev[1]))
        del ws
    out["maskless"] = dict(ms=dict(icp=float(np.median(ms_list))), peak_mb=(torch.cuda.max_memory_allocated() - base) / 2**20,
                           **_stats(iters, status, 4))
    # masked, run-length masks
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    stages = {"decode": [], "scene": [], "icp": []}
    from gigapose_b200 import _lib
    lib = _lib.load()
    import ctypes as C
    for rep in range(REPS + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        cnt = torch.as_tensor(rle[0]).to(DEV, non_blocking=True)
        ms = icp.MaskSet(np.zeros(n_det), icp.rle_boxes(rle[0], rle[1], H, W), rle[1])
        nbytes, px = ms.query(1, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.gp_icp_masked_decode(1, H, W, C.byref(ms.c), None, cnt.data_ptr(), ws.data_ptr(), stream))
        ev[1].record()
        _lib.check(lib.gp_icp_prepare_masked_scene(1, H, W, C.byref(ms.c), depth.data_ptr(), K.data_ptr(), 1000.0,
                                                   ws.data_ptr(), stream))
        ev[2].record()
        _, status, _, _ = icp.refine_rendered_masked(ms, ws, px, depth, K, di, R, boxes, T0, debug=dict(iterations=iters))
        ev[3].record()
        torch.cuda.synchronize()
        if rep:
            for k, (a, b) in zip(stages, zip(ev[:-1], ev[1:])):
                stages[k].append(a.elapsed_time(b))
        del ws
    out["masked"] = dict(ms={k: float(np.median(v)) for k, v in stages.items()},
                         peak_mb=(torch.cuda.max_memory_allocated() - base) / 2**20,
                         box_pixels=int(px), **_stats(iters, status, 4))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "icp_masked_time.py measures on the GPU"
    torch.cuda.set_device(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi[:1], repetitions=REPS)
    meshes = [bumpy(o) for o in range(8)]
    dm = icp.device_meshes(meshes, DEV)
    for name, shape in SHAPES.items():
        rng = np.random.default_rng(len(name))
        K = torch.as_tensor(np.array(shape["K"], np.float32)).to(DEV)[None].contiguous()
        depth, labels, truth, masks = make_image(shape, meshes, rng)
        result[name] = {f"hypotheses_{h}": time_image(dm, labels, truth, depth, K, masks, h, rng) for h in (1, 5)}
        print(name, json.dumps(result[name]), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=2)


if __name__ == "__main__":
    main()
