"""Times the depth refiner (row f6) on a c2-shaped case: 32 detections of 8 objects (10^4-face meshes) in 4 frames at
640 x 480, refining 1 and 5 hypotheses per detection.  Reports milliseconds per detection for the render, scene and ICP
stages (CUDA events, median of 5 after a warm-up) and the mean iterations per level, with the card's name and power
limit.  Prints one JSON object; writes it to --out when given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gigapose_b200 import icp, render  # noqa: E402

H, W = 480, 640
K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]], np.float32)


def bumpy(seed, n_lat=50, n_lon=100):
    """An asymmetric bumpy ellipsoid of ~10^4 faces (mm)."""
    rng = np.random.default_rng(seed)
    r = rng.uniform([50, 35, 20], [90, 60, 40])
    th = np.linspace(0, np.pi, n_lat)[:, None]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)[None]
    k = rng.integers(2, 6, 2)
    bump = 1 + 0.08 * np.sin(k[0] * th) * np.cos(k[1] * ph + rng.uniform(0, 6))
    V = np.stack([r[0] * np.sin(th) * np.cos(ph) * bump, r[1] * np.sin(th) * np.sin(ph) * bump,
                  r[2] * np.cos(th) * bump + 0 * ph], -1).reshape(-1, 3).astype(np.float32)
    F = [[i * n_lon + j, (i + 1) * n_lon + j, i * n_lon + (j + 1) % n_lon] for i in range(n_lat - 1) for j in range(n_lon)]
    F += [[i * n_lon + (j + 1) % n_lon, (i + 1) * n_lon + j, (i + 1) * n_lon + (j + 1) % n_lon]
          for i in range(n_lat - 1) for j in range(n_lon)]
    return dict(vertices=V, faces=np.array(F, np.int32))


def rodrigues(w):
    th = np.linalg.norm(w)
    Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    return np.eye(3) + np.sin(th) / th * Wx + (1 - np.cos(th)) / th ** 2 * Wx @ Wx


def make_case(dev, seed=0):
    rng = np.random.default_rng(seed)
    meshes = [bumpy(o) for o in range(8)]
    dm = icp.device_meshes(meshes, dev)
    labels, frames, truth = [], [], []
    depth = torch.zeros(4, H, W, device=dev)
    Kt = torch.as_tensor(K).to(dev).expand(4, 3, 3).contiguous()
    for f in range(4):
        for j in range(8):                                  # 8 detections per frame on a 4 x 2 grid
            o = (f * 3 + j) % 8
            T = np.eye(4, dtype=np.float32)
            T[:3, :3] = rodrigues(rng.normal(size=3))
            T[:3, 3] = (-240 + 160 * (j % 4), -90 + 180 * (j // 4), rng.uniform(750, 850))
            d = render.render_templates(meshes[o], torch.as_tensor(T)[None], K, size=(H, W), device=dev)["depth"][0]
            depth[f] = torch.where((d > 0) & ((depth[f] == 0) | (d < depth[f])), d, depth[f])
            labels.append(o)
            frames.append(f)
            truth.append(T)
    plane = torch.full((H, W), 1000.0, device=dev)
    depth = torch.where(depth > 0, depth, plane)
    return dm, np.array(labels), np.array(frames), np.stack(truth), depth, Kt


def perturbed(truth, hyp, rng):
    out = []
    for T in truth:
        for _ in range(hyp):
            P = T.copy()
            P[:3, :3] = rodrigues(np.deg2rad(rng.uniform(2, 6)) * rng.normal(size=3) / np.sqrt(3)) @ T[:3, :3]
            P[:3, 3] += rng.uniform(-8, 8, 3)
            out.append(P)
    return np.stack(out).astype(np.float32)


def time_case(dm, labels, frames, T0, depth, Kt, reps=5):
    dev = depth.device
    n = len(T0)
    F = depth.shape[0]
    T0 = torch.as_tensor(T0).to(dev)
    lab, fr = torch.as_tensor(labels), torch.as_tensor(frames)
    ws = torch.empty(icp.workspace_bytes(F, n, H, W), dtype=torch.uint8, device=dev)
    fi = fr.to(dev, torch.int32)
    iters = torch.zeros(n, 4, dtype=torch.int32, device=dev)
    ms = {"render": [], "scene": [], "icp": []}
    for rep in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        R, boxes = icp.render_hypotheses(dm, lab, T0, Kt, fr, H, W)
        ev[1].record()
        icp.prepare_scene(depth, Kt, ws)
        ev[2].record()
        out = icp.refine_rendered(depth, Kt, fi, R, boxes, T0, None, ws, debug=dict(iterations=iters))
        ev[3].record()
        torch.cuda.synchronize()
        if rep:
            for k, (a, b) in zip(ms, zip(ev[:-1], ev[1:])):
                ms[k].append(a.elapsed_time(b))
    status = out[1].cpu().numpy()
    return ({k: float(np.median(v)) for k, v in ms.items()}, iters.float().mean(0).tolist(),
            np.bincount(status, minlength=6).tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "icp_time.py measures on a GPU"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    dm, labels, frames, truth, depth, Kt = make_case(dev)
    rng = np.random.default_rng(1)
    result = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi[0] if smi else None, detections=len(truth),
                  frames=4, size=[H, W], faces_per_mesh=int(dm[0]["faces"].shape[0]), cases={})
    for hyp in (1, 5):
        T0 = perturbed(truth, hyp, rng)
        ms, it, st = time_case(dm, np.repeat(labels, hyp), np.repeat(frames, hyp), T0, depth, Kt)
        per_det = {k: v / len(truth) for k, v in ms.items()}
        result["cases"][f"hypotheses_{hyp}"] = dict(
            ms_total=ms, ms_per_detection=per_det, ms_per_detection_all=sum(per_det.values()),
            mean_iterations_per_level=dict(zip(["level0", "level1", "level2", "level3"], it)),
            status_counts=dict(zip(["ok", "too_few_points", "degenerate", "residual", "invalid", "lost"], st)))
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
