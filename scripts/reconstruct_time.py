"""Times row f17's reconstruction on a HOPE-shaped object (a 90 x 60 x 180 mm bumpy ellipsoid, an up and a down
sequence of 150 frames each at 1920 x 1080) and an LM-O-shaped one (70 x 45 x 60 mm, 2 x 150 frames at 640 x 480), at
R = 128 and 256: the host decode of the depth and mask PNGs (on the decode threads), the upload, the box (order
statistics), gp_tsdf_fuse and the extraction (CUDA events, median of 3 after a warm-up), the vertex and face counts and
the peak device memory of `reconstruct.reconstruct`.  It also times the ICP refinement of row f10 (5 hypotheses of one
image, CUDA events, median of 5 after a warm-up) with the reconstructed mesh against the true mesh, since render time
grows with the faces.  The frames are synthetic renders written to a temporary directory as 16-bit PNG depth (1 mm
units); the card name and power limit are read in the same run.  The sequence lengths are assumptions.

    python scripts/reconstruct_time.py [--frames 150] [--out results.json]
"""
import argparse
import concurrent.futures
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gigapose_b200 import icp, onboarding, reconstruct, render  # noqa: E402
from rgbd_static_tree import look_at_pose, up_down_directions  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def ellipsoid(radii, n_lat=96, n_lon=192):
    th = np.linspace(0, np.pi, n_lat)[:, None]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)[None]
    bump = 1 + 0.06 * np.sin(3 * th) * np.cos(2 * ph) + 0.04 * np.cos(5 * ph + 1.0) * np.sin(th) ** 2
    V = np.stack([radii[0] * np.sin(th) * np.cos(ph) * bump, radii[1] * np.sin(th) * np.sin(ph) * bump,
                  radii[2] * np.cos(th) * bump + 0 * ph], -1).reshape(-1, 3).astype(np.float32)
    F = [[a, a + n_lon, b] for i in range(n_lat - 1) for j in range(n_lon)
         for a, b in [(i * n_lon + j, i * n_lon + (j + 1) % n_lon)]]
    F += [[b, a + n_lon, b + n_lon] for i in range(n_lat - 1) for j in range(n_lon)
          for a, b in [(i * n_lon + j, i * n_lon + (j + 1) % n_lon)]]
    return dict(vertices=V, faces=np.array(F, np.int32))


def write_frames(mesh, n, H, W, K, dist, d, seed):
    """n frames (half up, half down) as 16-bit PNG depth (mm) and PNG masks under d -> onboarding.Frames."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    os.makedirs(d, exist_ok=True)
    poses, jobs = [], []
    pool = concurrent.futures.ThreadPoolExecutor(8)
    for i, cam in enumerate(up_down_directions(n, rng)):
        P = look_at_pose(cam, dist)
        r = render.render_templates(mesh, torch.as_tensor(P, dtype=torch.float32)[None], K, size=(H, W), device=DEV)
        depth = r["depth"][0].cpu().numpy()
        bg = np.float32(dist + 200.0)
        raw = np.round(np.where(depth > 0, depth, bg)).astype(np.uint16)
        mask = (depth > 0).astype(np.uint8) * 255
        jobs.append(pool.submit(Image.fromarray(raw).save, os.path.join(d, f"d{i:06d}.png")))
        jobs.append(pool.submit(Image.fromarray(mask).save, os.path.join(d, f"m{i:06d}.png")))
        poses.append(P)
    for j in jobs:
        j.result()
    pool.shutdown()
    return onboarding.Frames([None] * n, [os.path.join(d, f"m{i:06d}.png") for i in range(n)],
                             np.repeat(np.asarray(K, np.float64)[None], n, 0), np.stack(poses),
                             depths=[os.path.join(d, f"d{i:06d}.png") for i in range(n)], depth_scale=1.0)


def events(fn, reps=3):
    fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out)), r


def stages(frames, R):
    """Each stage of `reconstruct` on its own: decode + upload (wall), box, fusion and extraction (CUDA events)."""
    pool = concurrent.futures.ThreadPoolExecutor(reconstruct.DECODE_THREADS)
    t0 = time.perf_counter()
    kept = list(reconstruct._chunks(frames, torch.device(DEV), pool))
    torch.cuda.synchronize()
    load_s = time.perf_counter() - t0
    pool.shutdown()
    # the upload alone: pinned host copies of one chunk, timed with events
    h_d, h_m = kept[0][1].cpu().pin_memory(), kept[0][2].cpu().pin_memory()
    upload_ms_per_chunk, _ = events(lambda: (h_d.to(DEV, non_blocking=True), h_m.to(DEV, non_blocking=True)))

    def box():
        pts = torch.cat([reconstruct.object_points(d[j], m[j], frames.K[i], frames.poses[i])
                         for ids, d, m in kept for j, i in enumerate(ids)])
        return reconstruct.order_statistics(pts)
    box_ms, (lo, hi) = events(box, reps=1)
    b = reconstruct.grid_box(lo, hi, R)

    def fuse():
        g = reconstruct.new_grid(b["dims"], DEV)
        for ids, d, m in kept:
            reconstruct.fuse(g, d, m, frames.K[ids], frames.poses[ids], b["origin"], b["voxel"], b["trunc"])
        return g
    fuse_ms, grid = events(fuse)
    extract_ms, (V, F) = events(lambda: reconstruct.extract(grid, b["origin"], b["voxel"]))
    del kept, grid
    torch.cuda.empty_cache()
    return dict(decode_and_upload_s=load_s, upload_ms_per_chunk=upload_ms_per_chunk, chunk=reconstruct.CHUNK,
                box_ms=box_ms, fuse_ms=fuse_ms, extract_ms=extract_ms, dims=list(b["dims"]), voxel_mm=float(b["voxel"]),
                vertices=int(V.shape[0]), faces=int(F.shape[0]))


def hypotheses(T):
    """5 hypotheses of pose T, each 3 deg and up to 6 mm per axis off."""
    rng = np.random.default_rng(0)
    T0 = []
    for _ in range(5):
        a = rng.normal(size=3)
        a *= np.radians(3.0) / np.linalg.norm(a)
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        th = np.linalg.norm(a)
        Ra = np.eye(3) + np.sin(th) / th * Kx + (1 - np.cos(th)) / th ** 2 * Kx @ Kx
        P = T.copy()
        P[:3, :3] = Ra @ T[:3, :3]
        P[:3, 3] += rng.uniform(-6, 6, 3)
        T0.append(P)
    return T0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=150, help="frames per sequence (up and down)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), frames_per_sequence=a.frames, objects={})
    cases = {"hope": (ellipsoid((45.0, 30.0, 90.0)), 1080, 1920,
                      np.array([[1390.0, 0, 961.5], [0, 1390.0, 538.5], [0, 0, 1]]), 450.0),
             "lmo": (ellipsoid((35.0, 22.5, 30.0)), 480, 640,
                     np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]]), 700.0)}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (mesh, H, W, K, dist) in cases.items():
            frames = write_frames(mesh, 2 * a.frames, H, W, K, dist, os.path.join(tmp, name), seed=len(name))
            # the host decode of one frame (depth + mask PNG), single-threaded
            t0 = time.perf_counter()
            for i in range(8):
                reconstruct._load(frames, i)
            decode_ms = (time.perf_counter() - t0) / 8 * 1e3
            out = dict(size=[H, W], frames=len(frames), decode_ms_per_frame_one_thread=decode_ms, R={})
            T = look_at_pose([0.3, -0.4, 0.8], dist)
            scene = render.render_templates(mesh, torch.as_tensor(T, dtype=torch.float32)[None], K, size=(H, W),
                                            device=DEV)["depth"]
            T0 = torch.as_tensor(np.stack(hypotheses(T))).float().to(DEV)
            Kt = torch.as_tensor(K, dtype=torch.float32)[None]

            def icp_ms(m):
                dm = icp.device_meshes([m], DEV)
                ms, r = events(lambda: icp.refine_icp(dm, np.zeros(5, np.int64), T0, scene, Kt, np.zeros(5, np.int64)),
                               reps=5)
                return ms, int((r[1] == 0).sum())
            out["icp_true_mesh"] = dict(faces=len(mesh["faces"]), ms=icp_ms(mesh))
            for R in (128, 256):
                st = stages(frames, R)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(DEV)
                base = torch.cuda.memory_allocated(DEV)
                t0 = time.perf_counter()
                rec = reconstruct.reconstruct(frames, resolution=R, device=DEV)
                torch.cuda.synchronize()
                st["reconstruct_s"] = time.perf_counter() - t0
                st["peak_mib"] = (torch.cuda.max_memory_allocated(DEV) - base) / 2 ** 20
                st["icp_reconstructed_ms"] = icp_ms(rec)
                out["R"][R] = st
                print(name, R, json.dumps(st), flush=True)
            res["objects"][name] = out
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
