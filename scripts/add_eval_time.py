"""Times row f12 (gp_bop_add and bop_eval.evaluate_add) on synthetic evaluations generated from a seed:
  - LM-O-shaped: 200 frames, 8 objects of 10 002 vertices, one instance of about 7 objects per frame, one estimate per
    target (about 1 450 pairs);
  - HOPE-shaped: the tree of scripts/bop24_eval_time.py (200 images, 28 objects of 10 002 vertices), gp_bop_add timed
    on the 24 134 (estimate, ground truth) pairs of its BOP 2024 evaluation, evaluate_add on BOP 2019 targets listing
    every object of every image;
  - N^2 scaling: pairs of one 100 000-vertex object.
gp_bop_add from CUDA events (median of --runs after a warm-up), evaluate_add's wall time and its host share (wall minus
the device stage), the card's name, power limit and max SM clock read in the same run, and scipy's cKDTree ADD-S on
--kdtree-pairs pairs (a CPU number).  Prints one JSON line and writes it to --out."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import bop24_eval_time  # noqa: E402
from bop_eval_time import bumpy_spheroid, card  # noqa: E402
from bop_tree import rot, write_tree  # noqa: E402
from gigapose_b200 import bop_eval  # noqa: E402

DEV = "cuda"
K_LMO = np.array([[572.4, 0, 325.3], [0, 573.6, 242.0], [0, 0, 1]])


def lmo_tree(root, frames=200, objects=8, seed=0):
    rng = np.random.default_rng(seed)
    models, info = {}, {}
    for o in range(1, objects + 1):
        V, F, d = bumpy_spheroid(o, n_lat=102, n_lon=100)
        models[o] = (V, F)
        info[o] = dict(diameter=float(d))
    info[1]["symmetries_discrete"] = [np.diag([-1.0, -1, 1, 1]).ravel().tolist()]
    scenes, targets, results = {1: {}}, [], []
    png = np.zeros((480, 640), np.uint16)
    for im in range(frames):
        present = rng.choice(np.arange(1, objects + 1), size=int(rng.integers(6, 9)), replace=False)
        gts = [(int(o), rot(rng.normal(size=3), rng.uniform(0, 180)),
                np.array([rng.uniform(-200, 200), rng.uniform(-150, 150), rng.uniform(700, 1200)])) for o in present]
        scenes[1][im] = dict(gt=gts, visib=[float(rng.uniform(0.05, 1)) for _ in gts], K=K_LMO, depth_scale=1.0,
                             png=png)
        for o, R, t in gts:
            results.append(dict(scene_id=1, im_id=im, obj_id=o, score=float(rng.random()),
                                R=rot(rng.normal(size=3), rng.uniform(0, 15)) @ R, t=t + rng.normal(size=3) * 10,
                                time=0.1))
        targets += [(1, im, int(o), 1) for o in present]
    write_tree(root, models, info, scenes, targets)
    return results


def hope_targets(root, results):
    """BOP 2019 targets over every object of every image of the bop24 tree (inst_count = its instances)."""
    with open(os.path.join(root, "test_targets_bop24.json")) as f:
        images = [(d["scene_id"], d["im_id"]) for d in json.load(f)]
    out = []
    for s, im in images:
        with open(os.path.join(root, "test", f"{s:06d}", "scene_gt.json")) as f:
            gts = json.load(f)[str(im)]
        count = {}
        for g in gts:
            count[g["obj_id"]] = count.get(g["obj_id"], 0) + 1
        out += [dict(scene_id=s, im_id=im, obj_id=o, inst_count=n) for o, n in sorted(count.items())]
    with open(os.path.join(root, "test_targets_bop19.json"), "w") as f:
        json.dump(out, f)


def pair_tensors(setup, groups, pairs, obj_ids):
    """Device inputs of gp_bop_add for `pairs` (a _pair_rows dict over `groups`)."""
    res, scenes = setup["results"], setup["scenes"]
    _, vertices, _, vo, _ = bop_eval._object_tables(setup, obj_ids, DEV)
    oidx = {o: i for i, o in enumerate(obj_ids)}
    K = torch.as_tensor(np.stack([scenes[s]["K"][im] for s, im in setup["images"]]), dtype=torch.float32,
                        device=DEV).contiguous()
    gl, el, kl = pairs["group"].tolist(), pairs["est"].tolist(), pairs["gt"].tolist()
    pe = np.stack([bop_eval._pose(res[e]["R"], res[e]["t"]) for e in el]).astype(np.float32)
    gts = [scenes[groups[g]["scene_id"]]["gt"][groups[g]["im_id"]][k] for g, k in zip(gl, kl)]
    pg = np.stack([bop_eval._pose(g["R"], g["t"]) for g in gts]).astype(np.float32)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    obj = t(np.array([oidx[groups[g]["obj_id"]] for g in gl], np.int32))
    return dict(obj=obj, vo=vo, vertices=vertices, K=K, frame=t(pairs["frame"].astype(np.int32)), pe=t(pe), pg=t(pg))


def time_kernel(a, runs):
    call = lambda: bop_eval.add_errors(a["obj"], a["vo"], a["vertices"], a["K"], a["frame"], a["pe"], a["pg"])
    out = call()                                                               # warm-up
    ms = []
    for _ in range(runs):
        ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev[0].record()
        call()
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ms)), out


def time_evaluate(results, root, runs):
    bop_eval.evaluate_add(results, root)                                       # warm-up
    wall, dev, out = [], [], None
    for _ in range(runs):
        stage = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = bop_eval.evaluate_add(results, root, stage_ms=stage)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(stage.get("add", 0.0))
    w, d = float(np.median(wall)), float(np.median(dev))
    return dict(evaluate_add_wall_ms=w, evaluate_add_device_ms=d, evaluate_add_host_share=(w - d) / w,
                evaluate_add_pairs=int(len(out["errors"]["group"])), n_targets=out["n_targets"], recall=out["recall"],
                auc=out["auc"])


def kdtree_ms(a, n):
    from scipy.spatial import cKDTree
    V = a["vertices"].cpu().numpy().astype(np.float64)
    obj, pe, pg = a["obj"].cpu().numpy(), a["pe"].cpu().numpy().astype(np.float64), a["pg"].cpu().numpy().astype(np.float64)
    t0 = time.perf_counter()
    for p in range(n):
        X = V[a["vo"][obj[p]]:a["vo"][obj[p] + 1]]
        e, g = X @ pe[p, :3, :3].T + pe[p, :3, 3], X @ pg[p, :3, :3].T + pg[p, :3, 3]
        cKDTree(e).query(g, k=1)
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--kdtree-pairs", type=int, default=20)
    ap.add_argument("--big-pairs", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    rep = dict(card=card())
    with tempfile.TemporaryDirectory() as root:                                # LM-O-shaped
        results = lmo_tree(root)
        setup = bop_eval.prepare(results, root)
        groups = setup["groups"]
        pairs = bop_eval._pair_rows(groups, range(len(groups)), setup["images"])
        args = pair_tensors(setup, groups, pairs, sorted({g["obj_id"] for g in groups}))
        ms, _ = time_kernel(args, a.runs)
        rep["lmo"] = dict(pairs=int(len(pairs["group"])), vertices_per_object=args["vo"][1], gp_bop_add_ms=ms,
                          kdtree_adds_cpu_ms_per_pair=kdtree_ms(args, a.kdtree_pairs), **time_evaluate(results, root,
                                                                                                      a.runs))
    with tempfile.TemporaryDirectory() as root:                                # HOPE-shaped
        results, _ = bop24_eval_time.build_tree(root)
        setup = bop_eval.prepare_detection(results, root)
        pairs = bop_eval.detection_pairs(setup)
        args = pair_tensors(setup, setup["groups"], pairs, setup["objects"])
        ms, _ = time_kernel(args, a.runs)
        hope = dict(pairs=int(len(pairs["group"])), vertices_per_object=args["vo"][1], gp_bop_add_ms=ms,
                    kdtree_adds_cpu_ms_per_pair=kdtree_ms(args, a.kdtree_pairs))
        hope_targets(root, results)
        hope["bop19_targets"] = time_evaluate(results, root, a.runs)
        rep["hope"] = hope
    # N^2: one 100 000-vertex object
    rng = np.random.default_rng(1)
    V = (rng.normal(size=(100000, 3)) * [60, 40, 30]).astype(np.float32)
    n = a.big_pairs
    P = np.tile(np.eye(4, dtype=np.float32), (n, 1, 1))
    P[:, :3, 3] = [0, 0, 1000]
    Q = P.copy()
    Q[:, :3, 3] += rng.normal(size=(n, 3)).astype(np.float32) * 5
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=DEV)
    big = dict(obj=t(np.zeros(n, np.int32)), vo=[0, len(V)], vertices=t(V), K=t(K_LMO.astype(np.float32)[None]),
               frame=t(np.zeros(n, np.int32)), pe=t(Q), pg=t(P))
    ms, _ = time_kernel(big, a.runs)
    rep["big"] = dict(vertices=len(V), pairs=n, gp_bop_add_ms=ms, ms_per_pair=ms / n,
                      kdtree_adds_cpu_ms_per_pair=kdtree_ms(big, min(a.kdtree_pairs, 5)))
    line = json.dumps(rep)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
