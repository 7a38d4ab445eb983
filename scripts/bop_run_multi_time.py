"""Wall time per image of `python -m gigapose_b200.bop_run` (row f15) under `torchrun --nproc-per-node N`, on synthetic
LM-O-shaped (640 x 480 JPEG, 50 detections per image) and HOPE-shaped (1920 x 1080 PNG, 100 detections per image) test
splits of 8 objects, onboarded from the generated level-1 templates (8 x 162), detection setting, seeded weights.

Per run, the time per image is (last prediction file written - first) / (images - ranks): every rank writes its first
file after its first image, so the span covers the other images of all ranks, and excludes start-up, model build and
onboarding.  Ranks take cuda:LOCAL_RANK; N is limited to the visible devices unless --share-device puts every rank on
cuda:0, which measures ranks sharing one GPU, not scaling.

    python scripts/bop_run_multi_time.py [--ranks 1 2 4 8] [--images 32] [--share-device] [--out results/x.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bop_run_time import SHAPES, box_mesh, make_images  # noqa: E402
from gigapose_b200 import bop_run  # noqa: E402

OBJECTS = [1, 5, 6, 8, 9, 10, 11, 12]       # LM-O's object ids; the HOPE-shaped tree numbers them 1 .. 8


def write_ply(path, mesh):
    V, F, C = mesh["vertices"], mesh["faces"], (mesh["vertex_color"] * 255).round().astype(int)
    with open(path, "w") as f:
        f.write(f"ply\nformat ascii 1.0\nelement vertex {len(V)}\nproperty float x\nproperty float y\nproperty float z\n"
                f"property uchar red\nproperty uchar green\nproperty uchar blue\nelement face {len(F)}\n"
                f"property list uchar int vertex_indices\nend_header\n")
        for v, c in zip(V, C):
            f.write(" ".join(repr(float(x)) for x in v) + " " + " ".join(str(x) for x in c) + "\n")
        for t in F:
            f.write("3 " + " ".join(str(int(i)) for i in t) + "\n")


def make_tree(root, shape, images):
    """<root>/<shape> as a BOP test split with its default CNOS detection file; -> the dataset directory."""
    H, W, n, ext = SHAPES[shape]
    ds = os.path.join(root, shape)
    scene = os.path.join(ds, "test", "000001")
    os.makedirs(os.path.join(scene, "rgb"))
    os.makedirs(os.path.join(ds, "models"))
    ids = OBJECTS if shape == "lmo" else list(range(1, 9))
    rng = np.random.default_rng(4)
    for o in ids:
        write_ply(os.path.join(ds, "models", f"obj_{o:06d}.ply"), box_mesh(*rng.uniform(20, 50, 3)))
    with open(os.path.join(ds, "models", "models_info.json"), "w") as f:
        json.dump({str(o): dict(diameter=100.0) for o in ids}, f)
    dets, cams = [], {}
    for im, (path, ds_dets) in enumerate(make_images(os.path.join(scene, "rgb"), H, W, n, ext, images, seed=len(shape))):
        for d in ds_dets:
            dets.append(dict(d, scene_id=1, image_id=im, category_id=ids[int(rng.integers(len(ids)))]))
        cams[str(im)] = dict(cam_K=[600.0, 0, W / 2, 0, 600.0, H / 2, 0, 0, 1], depth_scale=1.0)
    with open(os.path.join(scene, "scene_camera.json"), "w") as f:
        json.dump(cams, f)
    year, model = bop_run.detection_year(shape)
    d = os.path.join(root, "default_detections", f"core{year}_model_based_unseen", model)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, f"{model}_{shape}-test.json"), "w") as f:
        json.dump(dets, f)
    return ds


def run(ds, ckpt, out, ranks, share_device):
    cmd = [sys.executable, "-m", "gigapose_b200.bop_run", "--dataset-dir", ds, "--checkpoint", ckpt, "--out", out,
           "--setting", "detection"] + (["--device", "cuda:0"] if share_device else [])
    if ranks > 1:
        cmd[1:1] = ["-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(ranks)]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    pred = os.path.join(out, "predictions")
    times = sorted(os.path.getmtime(os.path.join(pred, f)) for f in os.listdir(pred) if f.endswith(".npz"))
    return dict(images=len(times), wall_per_image_ms=(times[-1] - times[0]) / (len(times) - ranks) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--share-device", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bop_run_multi_time.py measures on the GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ranks = [n for n in a.ranks if a.share_device or n <= torch.cuda.device_count()]
    result = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi, gpus=torch.cuda.device_count(),
                  share_device=a.share_device, not_measured=[n for n in a.ranks if n not in ranks])
    with tempfile.TemporaryDirectory() as root:
        ckpt = os.path.join(root, "seeded.ckpt")
        torch.save({"state_dict": bop_run.build_model("cuda:0", root, seed=7).state_dict()}, ckpt)
        torch.cuda.empty_cache()
        for shape in SHAPES:
            ds = make_tree(root, shape, a.images)
            result[shape] = {}
            for n in ranks:
                result[shape][n] = run(ds, ckpt, os.path.join(root, f"out_{shape}_{n}"), n, a.share_device)
                print(shape, n, json.dumps(result[shape][n]), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=2)


if __name__ == "__main__":
    main()
