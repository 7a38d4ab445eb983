"""Per-image stage times of the depth refinement of row f10 (`bop_run --refine-depth H`) on synthetic BOP-shaped test
images: LM-O-shaped (640 x 480, 8 instances per image) and HOPE-shaped (1920 x 1080, 18 instances per image), generated
from a seed into a temporary directory.  The depth images are 16-bit PNGs rendered from the planted ground truth (eight
10^4-face meshes of scripts/icp_time.py) in front of a plane; the coarse predictions are the truth perturbed by 2-6
degrees and up to 8 mm per axis, as scripts/icp_time.py plants them.  For H = 1 and 5 hypotheses per instance, per image:
  decode        host wall clock: the depth PNG to f32 [H,W] (`bop_eval.load_depth`)
  render        `icp.render_hypotheses` of the coarse poses
  icp           gp_icp_prepare_scene + gp_icp_refine
  score_render  `icp.render_hypotheses` of the final poses
  depth_score   gp_depth_score (depth_score_kernel alone)
the GPU stages with CUDA events, the median of 7 repetitions after a warm-up over all images.  The retrieval time of
the same image shapes is what scripts/bop_run_time.py reports.  Prints the card's name, power limit and maximum SM clock.

    python scripts/bop_refine_time.py [--images 2] [--out results/bop_refine_time.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gigapose_b200 import _lib, bop_eval, icp, render  # noqa: E402
from icp_time import bumpy, perturbed, rodrigues  # noqa: E402

DEV = "cuda:0"
SHAPES = {"lmo": dict(size=(480, 640), K=[[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]],
                      grid=[(-240 + 160 * (j % 4), -90 + 180 * (j // 4)) for j in range(8)]),
          "hope": dict(size=(1080, 1920), K=[[1390.53, 0, 964.957], [0, 1386.99, 522.586], [0, 0, 1]],
                       grid=[(-450 + 180 * (j % 6), -180 + 180 * (j // 6)) for j in range(18)])}
REPS = 7
TOLERANCE_MM = 15.0


def make_image(root, shape, meshes, index, rng):
    """One depth PNG (mm) of the shape's grid of instances in front of a plane at 1 m -> (labels, truth [n,4,4])."""
    from PIL import Image
    H, W = shape["size"]
    K = np.array(shape["K"], np.float32)
    depth = torch.zeros(H, W, device=DEV)
    labels, truth = [], []
    for j, (x, y) in enumerate(shape["grid"]):
        o = (3 * index + j) % len(meshes)
        T = np.eye(4, dtype=np.float32)
        T[:3, :3] = rodrigues(rng.normal(size=3))
        T[:3, 3] = (x, y, rng.uniform(750, 850))
        d = render.render_templates(meshes[o], torch.as_tensor(T)[None], K, size=(H, W), device=DEV)["depth"][0]
        depth = torch.where((d > 0) & ((depth == 0) | (d < depth)), d, depth)
        labels.append(o)
        truth.append(T)
    depth = torch.where(depth > 0, depth, torch.full_like(depth, 1000.0))
    d = os.path.join(root, "test", "000001", "depth")
    os.makedirs(d, exist_ok=True)
    Image.fromarray(depth.round().cpu().numpy().astype(np.uint16)).save(os.path.join(d, f"{index:06d}.png"))
    return np.array(labels), np.stack(truth)


def time_image(dm, labels, T0, depth, K, hyp):
    """-> ({stage: [ms] * REPS}, ICP status counts, mean over the instances of the best hypothesis' depth score)."""
    H, W = depth.shape[1:]
    n = len(T0)
    T0 = torch.as_tensor(T0).to(DEV)
    lab, fr = torch.as_tensor(np.repeat(labels, hyp)), torch.zeros(n, dtype=torch.int64)
    fi = torch.zeros(n, dtype=torch.int32, device=DEV)
    ws = torch.empty(icp.workspace_bytes(1, n, H, W), dtype=torch.uint8, device=DEV)
    counts = torch.empty(n, 4, dtype=torch.int32, device=DEV)
    score = torch.empty(n, device=DEV)
    best = torch.empty(n // hyp, dtype=torch.int32, device=DEV)
    ms = {"render": [], "icp": [], "score_render": [], "depth_score": []}
    for rep in range(REPS + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        ev[0].record()
        R, boxes = icp.render_hypotheses(dm, lab, T0, K, fr, H, W)
        ev[1].record()
        icp.prepare_scene(depth, K, ws)
        out, status, _, _ = icp.refine_rendered(depth, K, fi, R, boxes, T0, None, ws)
        ev[2].record()
        R2, boxes2 = icp.render_hypotheses(dm, lab, out, K, fr, H, W)
        ev[3].record()
        _lib.check(_lib.load().gp_depth_score(1, n // hyp, hyp, H, W, fi.data_ptr(), depth.data_ptr(), R2.data_ptr(),
                                              boxes2.data_ptr(), TOLERANCE_MM, counts.data_ptr(), score.data_ptr(),
                                              best.data_ptr(), torch.cuda.current_stream().cuda_stream))
        ev[4].record()
        torch.cuda.synchronize()
        if rep:
            for k, (a, b) in zip(ms, zip(ev[:-1], ev[1:])):
                ms[k].append(a.elapsed_time(b))
    return ms, np.bincount(status.cpu().numpy(), minlength=6).tolist(), float(score.reshape(-1, hyp).max(1).values.mean())


def measure(name, images):
    shape = SHAPES[name]
    meshes = [bumpy(o) for o in range(8)]
    dm = icp.device_meshes(meshes, DEV)
    K = torch.as_tensor(np.array(shape["K"], np.float32)).to(DEV)[None].contiguous()
    rng = np.random.default_rng(len(name))
    out = dict(size=list(shape["size"]), instances=len(shape["grid"]))
    with tempfile.TemporaryDirectory() as root:
        planted = [make_image(root, shape, meshes, i, rng) for i in range(images)]
        decode = []
        for hyp in (1, 5):
            stages, statuses, scores = {}, np.zeros(6, np.int64), []
            for i, (labels, truth) in enumerate(planted):
                t0 = time.perf_counter()
                d = bop_eval.load_depth(root, "test", 1, i, 1.0)
                decode.append((time.perf_counter() - t0) * 1e3)
                depth = torch.as_tensor(d).to(DEV)[None].contiguous()
                ms, st, sc = time_image(dm, labels, perturbed(truth, hyp, rng), depth, K, hyp)
                for k, v in ms.items():
                    stages.setdefault(k, []).extend(v)
                statuses += st
                scores.append(sc)
            out[f"hypotheses_{hyp}"] = dict(
                ms_per_image={k: float(np.median(v)) for k, v in stages.items()},
                status_counts=dict(zip(["ok", "too_few_points", "degenerate", "residual", "invalid", "lost"], statuses.tolist())),
                mean_best_depth_score=float(np.mean(scores)))
        out["decode_ms"] = float(np.median(decode))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bop_refine_time.py measures on the GPU"
    torch.cuda.set_device(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi[:1], repetitions=REPS, images=a.images)
    for name in SHAPES:
        result[name] = measure(name, a.images)
        print(name, json.dumps(result[name]), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=2)


if __name__ == "__main__":
    main()
