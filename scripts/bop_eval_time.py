"""Times gigapose_b200.bop_eval.evaluate() per stage on an LM-O-shaped synthetic evaluation: 200 frames at 640 x 480,
8 objects of about 10^4 faces, about 1 450 targets with perturbed estimates.  GPU stages (renders, VSD, MSSD/MSPD) from
CUDA events, matching from the host clock; median of 5 runs after a warm-up.  Also times the fp64 numpy port of the
three errors on a subset of pairs, on the host (a CPU number).  Prints one JSON line and writes it to --out."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from bop_tree import rot, write_tree  # noqa: E402
from gigapose_b200 import bop_eval, icp  # noqa: E402
from oracle import bop_port  # noqa: E402

H, W = 480, 640
K = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]])


def bumpy_spheroid(seed, n_lat=52, n_lon=100):
    """~10^4 faces; object k is a lumpy ellipsoid of its own size."""
    rng = np.random.default_rng(seed)
    a, b, c = rng.uniform(30, 60, 3)
    th = np.linspace(0, np.pi, n_lat)[1:-1, None]
    ph = np.arange(n_lon)[None] * (2 * np.pi / n_lon)
    bump = 1 + 0.1 * np.sin(3 * th + seed) * np.cos(2 * ph)
    ring = np.stack([a * np.sin(th) * np.cos(ph) * bump, b * np.sin(th) * np.sin(ph) * bump,
                     c * np.cos(th) * bump + 0 * ph], -1).reshape(-1, 3)
    V = np.concatenate([ring, [[0, 0, c], [0, 0, -c]]]).astype(np.float32)
    F, L = [], n_lat - 2
    for i in range(L - 1):
        for j in range(n_lon):
            p, q = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            F += [[p, p + n_lon, q], [q, p + n_lon, q + n_lon]]
    for j in range(n_lon):
        F += [[len(V) - 2, j, (j + 1) % n_lon], [len(V) - 1, (L - 1) * n_lon + (j + 1) % n_lon, (L - 1) * n_lon + j]]
    return V, np.array(F, np.int32), 2 * max(a, b, c) * 1.1


def build_tree(root, frames=200, objects=8, seed=0):
    rng = np.random.default_rng(seed)
    models, info = {}, {}
    for o in range(1, objects + 1):
        V, F, d = bumpy_spheroid(o)
        models[o] = (V, F)
        info[o] = dict(diameter=float(d))
    info[objects]["symmetries_discrete"] = [np.diag([-1.0, -1, 1, 1]).ravel().tolist()]
    dm = icp.device_meshes([dict(vertices=models[o][0], faces=models[o][1]) for o in models], "cuda")
    ws = torch.empty(8 * H * W, dtype=torch.uint8, device="cuda")
    Kd = torch.as_tensor(K, dtype=torch.float32, device="cuda")
    scenes, targets, results = {1: {}}, [], []
    for im in range(frames):
        present = sorted(rng.choice(np.arange(1, objects + 1), size=7 + (im % 4 == 0), replace=False))
        gts, depth = [], np.full((H, W), 1200.0, np.float32)
        for k, o in enumerate(present):
            R = rot(rng.normal(size=3), rng.uniform(0, 180))
            t = np.array([(k % 4 - 1.5) * 120 + rng.normal() * 10, (k // 4 - 0.5) * 150, rng.uniform(700, 1000)])
            gts.append((int(o), R, t))
            T = np.eye(4, dtype=np.float32)
            T[:3, :3], T[:3, 3] = R, t
            d = torch.empty(1, H, W, device="cuda")
            b = torch.empty(1, 4, dtype=torch.int64, device="cuda")
            bop_eval.render_depth(dm[o - 1], torch.as_tensor(T, device="cuda")[None], Kd, H, W, 10.0, ws, d, b)
            d = d[0].cpu().numpy()
            depth = np.where((d > 0) & (d < depth), d, depth)
            for rep in range(2):
                dR = rot(rng.normal(size=3), rng.uniform(0, 10))
                results.append(dict(scene_id=1, im_id=im, obj_id=int(o), score=float(rng.random()), R=dR @ R,
                                    t=(t + rng.normal(size=3) * [5, 5, 20]).reshape(3, 1), time=0.05))
        depth[rng.random((H, W)) < 0.02] = 0
        scenes[1][im] = dict(gt=gts, visib=rng.uniform(0.05, 1.0, len(gts)).tolist(), K=K, depth_scale=0.1,
                             png=np.round(depth / 0.1).astype(np.uint16))
        targets += [(1, im, int(o), 1) for o in present]
    write_tree(root, models, info, scenes, targets)
    return results, len(targets)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--port-pairs", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    with tempfile.TemporaryDirectory() as root:
        results, n_targets = build_tree(root, a.frames)
        faces = [int(len(bumpy_spheroid(o)[1])) for o in range(1, 9)]
        setup = bop_eval.prepare(results, root)
        bop_eval.compute_errors(setup)                                    # warm-up
        stages, total, match = [], [], []
        for _ in range(a.runs):
            ms = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            err = bop_eval.compute_errors(setup, stage_ms=ms)
            t1 = time.perf_counter()
            rec = bop_eval.recalls(bop_eval.error_groups(setup, err), n_targets, r=W / 640)
            t2 = time.perf_counter()
            stages.append(ms)
            total.append((t1 - t0) * 1e3)
            match.append((t2 - t1) * 1e3)
        t0 = time.perf_counter()
        out = bop_eval.evaluate(results, root)
        evaluate_ms = (time.perf_counter() - t0) * 1e3
        # fp64 port on the first pairs, on the host, from depth rendered by the GPU
        n = min(a.port_pairs, len(err["group"]))
        dms = icp.device_meshes([bop_eval.read_ply(os.path.join(setup["mdir"], f"obj_{o:06d}.ply"))
                                 for o in sorted(setup["info"])], "cuda")
        Kd = torch.as_tensor(K, dtype=torch.float32, device="cuda")
        ws = torch.empty(8 * H * W, dtype=torch.uint8, device="cuda")
        port_s = 0.0
        for p in range(n):
            g = setup["groups"][int(err["group"][p])]
            o, im = g["obj_id"], g["im_id"]
            sc = setup["scenes"][1]
            gt = sc["gt"][im][int(err["gt"][p])]
            e = setup["results"][int(err["est"][p])]
            Pe, Pg = bop_eval._pose(e["R"], e["t"]), bop_eval._pose(gt["R"], gt["t"])
            dep = []
            for P in (Pe, Pg):
                d = torch.empty(1, H, W, device="cuda")
                b = torch.empty(1, 4, dtype=torch.int64, device="cuda")
                bop_eval.render_depth(dms[o - 1], torch.as_tensor(P, dtype=torch.float32, device="cuda")[None], Kd, H, W,
                                      10.0, ws, d, b)
                dep.append(d[0].cpu().numpy())
            d_test = bop_eval.load_depth(root, "test", 1, im, 0.1)
            V = bop_eval.read_ply(os.path.join(setup["mdir"], f"obj_{o:06d}.ply"))["vertices"]
            S = bop_eval.symmetry_transforms(setup["info"][o])
            t0 = time.perf_counter()
            bop_port.vsd_fp64(d_test, K, dep[0], dep[1], setup["info"][o]["diameter"], bop_eval.DELTA, bop_eval.TAUS)
            bop_port.mssd_mspd_fp64(V, S, Pe, Pg, K)
            port_s += time.perf_counter() - t0
    med = lambda xs: float(np.median(xs))
    rep = dict(card=card(), frames=a.frames, targets=n_targets, pairs=int(len(err["group"])), faces_per_object=faces,
               renders_ms=med([s.get("renders", 0.0) for s in stages]), vsd_ms=med([s.get("vsd", 0.0) for s in stages]),
               mssd_mspd_ms=med([s.get("mssd_mspd", 0.0) for s in stages]), compute_errors_wall_ms=med(total),
               matching_host_ms=med(match), evaluate_wall_ms_once=evaluate_ms, ar=out["ar"], ar_vsd=out["ar_vsd"],
               ar_mssd=out["ar_mssd"], ar_mspd=out["ar_mspd"],
               cpu_fp64_port_ms_per_pair=1e3 * port_s / max(n, 1), cpu_fp64_port_pairs=n,
               recall_check=float(rec["vsd"].mean()))
    line = json.dumps(rep)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
