"""Times gigapose_b200.bop_eval.evaluate_detection() (row f8, BOP 2024 6D detection) per stage on a HOPE-shaped synthetic
evaluation: 200 images at 1920 x 1080, 28 objects of about 10^4 vertices (one with a discrete and one with a continuous
symmetry), about 10 ground truths per image with repeated objects and about 10 % ignored, 100 estimates per image
(perturbed ground truths, duplicates and wrong-object estimates).  GPU stages (MSSD/MSPD, matching, AP) from CUDA events,
host wall times of prepare_detection and evaluate_detection; median of 5 runs after a warm-up.  Also times the numpy
port's matching + AP on the same errors, on the host (a CPU number).  Prints one JSON line and writes it to --out."""
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

from bop_eval_time import bumpy_spheroid, card  # noqa: E402
from bop_tree import rot, write_tree  # noqa: E402
from gigapose_b200 import bop_eval  # noqa: E402
from oracle import bop24_port  # noqa: E402

H, W = 1080, 1920
K = np.array([[1386.0, 0, 960.0], [0, 1386.0, 540.0], [0, 0, 1]])


def build_tree(root, images=200, objects=28, seed=0):
    rng = np.random.default_rng(seed)
    models, info = {}, {}
    for o in range(1, objects + 1):
        V, F, d = bumpy_spheroid(o, n_lat=102, n_lon=100)
        models[o] = (V, F)
        info[o] = dict(diameter=float(d))
    info[1]["symmetries_discrete"] = [np.diag([-1.0, -1, 1, 1]).ravel().tolist()]
    info[2]["symmetries_continuous"] = [dict(axis=[0, 0, 1], offset=[0, 0, 0])]
    scenes, results = {}, []
    png = np.zeros((H, W), np.uint16)
    for im in range(images):
        s = 1 + im // 40                                   # 5 scenes of 40 images
        present = rng.choice(np.arange(1, objects + 1), size=8, replace=False)
        objs = list(present) + list(rng.choice(present, size=2))          # two repeats
        gts = []
        for k, o in enumerate(objs):
            t = np.array([(k % 5 - 2) * 250 + rng.normal() * 10, (k // 5 - 0.5) * 300, rng.uniform(700, 1200)])
            gts.append((int(o), rot(rng.normal(size=3), rng.uniform(0, 180)), t))
        visib = [0.05 if rng.random() < 0.1 else float(rng.uniform(0.1, 1.0)) for _ in gts]
        scenes.setdefault(s, {})[im] = dict(gt=gts, visib=visib, K=K, depth_scale=1.0, png=png)
        ests = []
        for o, R, t in gts:                                # perturbed ground truths and duplicates: 8 per instance
            for rep in range(8):
                dR = rot(rng.normal(size=3), rng.uniform(0, 4 + 6 * rep))
                ests.append((o, dR @ R, t + rng.normal(size=3) * [3, 3, 10] * (1 + rep)))
        while len(ests) < 100:                             # wrong objects at ground-truth poses
            o, R, t = gts[int(rng.integers(len(gts)))]
            ests.append((int(rng.integers(1, objects + 1)), R, t + rng.normal(size=3) * 5))
        for o, R, t in ests:
            results.append(dict(scene_id=s, im_id=im, obj_id=int(o), score=float(rng.random()), R=R, t=t.reshape(3, 1),
                                time=0.2))
    write_tree(root, models, info, scenes, [(s, im, g[0], 1) for s in scenes for im in scenes[s]
                                            for g in scenes[s][im]["gt"][:1]])
    with open(os.path.join(root, "test_targets_bop24.json"), "w") as f:
        json.dump([dict(scene_id=s, im_id=im) for s in scenes for im in scenes[s]], f)
    return results, [len(models[o][0]) for o in models]


def port_inputs(setup, out):
    """The port's estimates / ground truths / errors from the GPU's per-pair errors."""
    res, scenes = setup["results"], setup["scenes"]
    kept = sorted({e for g in setup["groups"] for e in g["est"]})
    pos = {e: i for i, e in enumerate(kept)}
    estimates = [dict(image=(res[e]["scene_id"], res[e]["im_id"]), obj=res[e]["obj_id"], score=res[e]["score"])
                 for e in kept]
    gts, gpos = [], {}
    for s, im in setup["images"]:
        for k, (g, v) in enumerate(zip(scenes[s]["gt"][im], scenes[s]["visib"][im])):
            gpos[(s, im, k)] = len(gts)
            gts.append(dict(image=(s, im), obj=g["obj_id"], valid=v >= bop_eval.VISIB_GT_MIN))
    err = out["errors"]
    errors = {}
    for p in range(len(err["group"])):
        g = setup["groups"][int(err["group"][p])]
        errors[(pos[int(err["est"][p])], gpos[(g["scene_id"], g["im_id"], int(err["gt"][p]))])] = (err["mssd"][p],
                                                                                                   err["mspd"][p])
    return estimates, gts, errors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=200)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    with tempfile.TemporaryDirectory() as root:
        results, verts = build_tree(root, a.images)
        t0 = time.perf_counter()
        setup = bop_eval.prepare_detection(results, root)
        prepare_ms = (time.perf_counter() - t0) * 1e3
        bop_eval.evaluate_detection(results, root)                             # warm-up
        stages, wall = [], []
        for _ in range(a.runs):
            ms = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = bop_eval.evaluate_detection(results, root, stage_ms=ms)
            wall.append((time.perf_counter() - t0) * 1e3)
            stages.append(ms)
        estimates, gts, errors = port_inputs(setup, out)
        diam = {o: setup["info"][o]["diameter"] for o in setup["info"]}
        t0 = time.perf_counter()
        port = bop24_port.detection_scores(estimates, gts, errors, bop_eval.THETA_MSSD, bop_eval.THETA_MSPD, diam, W / 640)
        port_ms = (time.perf_counter() - t0) * 1e3
    med = lambda xs: float(np.median(xs))
    n_ign = sum(int((~g["valid"]).sum()) for g in setup["groups"])
    n_gt = sum(len(g["valid"]) for g in setup["groups"])
    rep = dict(card=card(), images=a.images, objects=len(verts), vertices_per_object=int(np.median(verts)),
               kept_estimates=int(len(out["rows"])), ground_truths=n_gt, ignored_ground_truths=n_ign,
               pairs=int(len(out["errors"]["group"])), mssd_mspd_ms=med([s["mssd_mspd"] for s in stages]),
               match_ms=med([s["match"] for s in stages]), ap_ms=med([s["ap"] for s in stages]),
               prepare_detection_wall_ms=prepare_ms, evaluate_detection_wall_ms=med(wall),
               cpu_numpy_port_match_ap_ms=port_ms, map=out["map"], map_mssd=out["map_mssd"], map_mspd=out["map_mspd"],
               port_map_bit_identical=bool(np.float64(port["map"]).view(np.uint64) ==
                                           np.float64(out["map"]).view(np.uint64)))
    line = json.dumps(rep)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
