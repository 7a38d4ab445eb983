"""Times the template renderer (row f5) on the GPU: `gp_render_templates` for the 162 level-1 template views at
640 x 480 on meshes of about 10^4 and 10^6 faces, and `GigaPose.onboard_meshes` in seconds per object (render + crop +
both encoders + bank write).  CUDA events after warm-up; the card name and power limit are read in the same run.

    python scripts/render_time.py [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gigapose_b200 import render, synth  # noqa: E402


def uv_sphere(n_lat, n_lon, radius=60.0, seed=0):
    """Bumpy latitude / longitude sphere with 2 * n_lon * (n_lat - 1) faces and random vertex colours."""
    g = np.random.default_rng(seed)
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    d = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    d = np.concatenate([[[0, 0, 1]], d, [[0, 0, -1]]])
    r = radius * (1 + 0.05 * np.sin(7 * d[:, 0]) * np.cos(5 * d[:, 1]))
    V = (d * r[:, None]).astype(np.float32)
    idx = lambda i, j: 1 + i * n_lon + (j % n_lon)
    faces = []
    j = np.arange(n_lon)
    faces.append(np.stack([np.zeros(n_lon, int), idx(0, j), idx(0, j + 1)], 1))
    for i in range(n_lat - 2):
        a, b, c, e = idx(i, j), idx(i, j + 1), idx(i + 1, j + 1), idx(i + 1, j)
        faces += [np.stack([a, e, c], 1), np.stack([a, c, b], 1)]
    last = len(V) - 1
    faces.append(np.stack([np.full(n_lon, last), idx(n_lat - 2, j + 1), idx(n_lat - 2, j)], 1))
    F = np.concatenate(faces).astype(np.int32)
    return dict(vertices=V, faces=F, vertex_color=g.uniform(0, 1, (len(V), 3)).astype(np.float32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def time_render(mesh, poses, K, H, W, iters=5):
    dev = torch.device("cuda:0")
    dm = render._device_mesh(mesh, dev)
    P = torch.as_tensor(poses, dtype=torch.float32, device=dev).contiguous()
    Kt = torch.as_tensor(K, dtype=torch.float32, device=dev)
    n = P.shape[0]
    per_view = H * W * 4 * 8
    chunk = max(1, min(n, render.WORKSPACE_BYTES // per_view))
    ws = torch.empty(chunk * per_view, dtype=torch.uint8, device=dev)
    rgba = torch.empty(n, 4, H, W, device=dev)
    depth = torch.empty(n, H, W, device=dev)
    boxes = torch.empty(n, 4, dtype=torch.int64, device=dev)

    def run():
        for v0 in range(0, n, chunk):
            v1 = min(n, v0 + chunk)
            render.render_chunk(dm, P[v0:v1], Kt, H, W, 100.0, ws, rgba[v0:v1], depth[v0:v1], boxes[v0:v1])
    run()
    run()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return dict(views=n, faces=int(len(mesh["faces"])), chunk_views=chunk, ms_median=float(np.median(ms)),
                ms_min=float(np.min(ms)), ms_max=float(np.max(ms)), covered_px_view0=int(rgba[0, 3].sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--objects", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "render_time.py measures on the GPU; there is no CPU path"
    torch.cuda.set_device(0)
    poses = synth.fibonacci_view_poses(162, distance=400.0).numpy()
    H, W = render.TEMPLATE_SIZE
    res = dict(card=card(), size=[H, W])
    meshes = {"1e4": uv_sphere(51, 100), "1e6": uv_sphere(501, 1000)}
    for name, mesh in meshes.items():
        res[f"render_162_views_{name}_faces"] = time_render(mesh, poses, render.TEMPLATE_K, H, W)
        print(name, res[f"render_162_views_{name}_faces"], flush=True)
    import bench
    model = bench.build_models(torch.device("cuda:0"))
    objs = [uv_sphere(51, 100, seed=o) for o in range(args.objects)]
    model.onboard_meshes("warmup", objs[:1], poses)
    model.onboard_meshes("timed", objs, poses)
    res["onboard_meshes_s_per_object"] = model.onboarding_s_per_object
    res["onboard_meshes_objects"] = args.objects
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
