"""Row f14: time `render_results` per image on LM-O-shaped (640 x 480, 8 targets) and HOPE-shaped (1920 x 1080, 18
targets) synthetic images with two csvs each (a coarse one and a refined one), by stage: renders, vertex errors (with
the ADD(-S) pairing and the heat colours), overlay (CUDA events) and PNG encode (wall clock), plus the wall clock of
the whole call, in ms per image.

    python scripts/vis_time.py [--images 4] [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import bop_tree  # noqa: E402
from gigapose_b200 import vis  # noqa: E402


def make_tree(root, H, W, n_targets, n_images, rng):
    """n_images images with n_targets objects each (distinct ids), a 6 000-face spheroid (symmetric) and tetrahedra."""
    from PIL import Image
    models = {o: (bop_tree.spheroid(n_lat=40, n_lon=80) if o % 3 == 0 else bop_tree.tetra(60.0)) for o in
              range(1, n_targets + 1)}
    info = {o: dict(diameter=80.0, **({"symmetries_continuous": [dict(axis=[0, 0, 1], offset=[0, 0, 0])]}
                                     if o % 3 == 0 else {})) for o in models}
    f = 0.9 * W
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
    ims, targets, coarse, refined = {}, [], [], []
    for im in range(n_images):
        gt = []
        for o in models:
            t = [rng.uniform(-200, 200), rng.uniform(-120, 120), rng.uniform(700, 1400)]
            R = bop_tree.rot(rng.normal(size=3), rng.uniform(0, 360))
            gt.append((o, R, t))
            targets.append((1, im, o, 1))
            for rows, err in ((coarse, 12.0), (refined, 2.0)):
                rows.append(dict(scene_id=1, im_id=im, obj_id=o, score=0.5, R=bop_tree.rot(rng.normal(size=3), 1.5) @ R,
                                 t=np.add(t, rng.normal(0, err, 3)), time=1.0))
        ims[im] = dict(gt=gt, visib=[1.0] * len(gt), K=K, depth_scale=1.0, png=np.zeros((H, W), np.uint16))
    bop_tree.write_tree(root, models, info, {1: ims}, targets)
    d = os.path.join(root, "test", "000001", "rgb")
    os.makedirs(d, exist_ok=True)
    for im in ims:
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(d, f"{im:06d}.png"))
    return coarse, refined


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    rng = np.random.default_rng(0)
    report = {"gpu": torch.cuda.get_device_name(0)}
    for name, (H, W, n) in {"lmo_640x480_8": (480, 640, 8), "hope_1920x1080_18": (1080, 1920, 18)}.items():
        with tempfile.TemporaryDirectory() as tmp:
            coarse, refined = make_tree(tmp, H, W, n, a.images + 1, rng)
            out = os.path.join(tmp, "vis")
            vis.render_results([coarse, refined], tmp, out, max_images=1)          # warm-up: loads, first launches
            stages = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            paths = vis.render_results([coarse, refined], tmp, out, max_images=a.images + 1, stage_ms=stages)
            wall = (time.perf_counter() - t0) * 1e3
            k = len(paths)
            report[name] = dict(images=k, wall_ms_per_image=round(wall / k, 2),
                                **{f"{s}_ms_per_image": round(v / k, 3) for s, v in sorted(stages.items())})
        print(json.dumps({name: report[name]}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vis_time.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
