"""Per-image stage times of the row f9 runner on synthetic BOP-shaped test images, and the RLE crop against the dense-mask
crop it replaces, in the same process and alternating per image.

Two shapes, generated from a seed into a temporary directory: LM-O-shaped (640 x 480 JPEG, 50 detections per image) and
HOPE-shaped (1920 x 1080 PNG, 100 detections per image).  Per image:
  decode     host: the image file to u8 [H,W,3] (`bop_run.read_image`)
  rle        host RLE read (`bop_run.image_inputs`), upload of the image and runs, gp_crop_resize_pad_rle (CUDA events)
  dense      host decode of every mask to f32 [n,H,W], upload of image and masks, gp_crop_resize_pad (CUDA events)
  retrieval  `GigaPose.eval_retrieval` on the RLE crops (seeded weights, 2 objects x 162 templates)
and the peak allocated device memory of each crop path.  Medians over the images after the first.

    python scripts/bop_run_time.py [--images 8] [--out results/bop_run_time.json]
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
from gigapose_b200 import bop_run  # noqa: E402
from gigapose_b200.preprocess import crop_detections_rle, preprocess_queries  # noqa: E402
from gigapose_b200.synth import fibonacci_view_poses  # noqa: E402

DEV = "cuda:0"
SHAPES = {"lmo": (480, 640, 50, "jpg"), "hope": (1080, 1920, 100, "png")}


def _encode(m):
    flat = m.reshape(-1, order="F")
    bounds = np.concatenate([[0], np.flatnonzero(flat[1:] != flat[:-1]) + 1, [flat.size]])
    c = np.diff(bounds).tolist()
    return [0] + c if flat[0] else c


def make_images(root, H, W, n, ext, count, seed):
    """Smooth random images (so that JPEG / PNG sizes are realistic) with n elliptical detections each."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W]
    out = []
    for i in range(count):
        low = rng.integers(0, 256, (H // 16 + 1, W // 16 + 1, 3)).astype(np.uint8)
        img = np.asarray(Image.fromarray(low).resize((W, H), Image.BILINEAR))
        path = os.path.join(root, f"{i:06d}.{ext}")
        Image.fromarray(img).save(path, quality=95) if ext == "jpg" else Image.fromarray(img).save(path)
        dets = []
        for _ in range(n):
            cy, cx = rng.uniform(0, H), rng.uniform(0, W)
            ry, rx = rng.uniform(10, H / 6), rng.uniform(10, W / 6)
            m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
            dets.append(dict(category_id=int(rng.integers(1, 3)), score=float(rng.random()), time=0.1,
                             bbox=[cx - rx, cy - ry, 2 * rx, 2 * ry], segmentation=dict(size=[H, W], counts=_encode(m))))
        out.append((path, dets))
    return out


def dense_masks(counts, offsets, H, W):
    n = len(offsets) - 1
    out = np.zeros((n, H * W), np.float32)
    for i in range(n):
        c = counts[offsets[i]:offsets[i + 1]].astype(np.int64)
        v = np.repeat((np.arange(len(c)) % 2).astype(np.float32), c)[:H * W]
        out[i, :len(v)] = v
    return out.reshape(n, W, H).transpose(0, 2, 1)


def _events():
    return [torch.cuda.Event(enable_timing=True) for _ in range(3)]


def run_rle(rgb, x):
    ev = _events()
    ev[0].record()
    img = rgb.to(DEV, non_blocking=True)[None]
    cnt = torch.as_tensor(x["counts"]).to(DEV, non_blocking=True)
    ev[1].record()
    out = crop_detections_rle(img, cnt, x["offsets"], x["boxes"], np.zeros(len(x["labels"]), np.int64))
    ev[2].record()
    return out, ev


def run_dense(rgb, masks, x):
    ev = _events()
    ev[0].record()
    img = rgb.to(DEV, non_blocking=True)[None].permute(0, 3, 1, 2)
    m = torch.as_tensor(masks).to(DEV, non_blocking=True)
    ev[1].record()
    out = preprocess_queries(img, m, x["boxes"], torch.zeros(len(x["labels"]), dtype=torch.int64))
    ev[2].record()
    return out, ev


def measure(shape, model, images):
    H, W, n, ext = SHAPES[shape]
    rows = []
    with tempfile.TemporaryDirectory() as root:
        for i, (path, dets) in enumerate(make_images(root, H, W, n, ext, images, seed=len(shape))):
            t0 = time.perf_counter()
            rgb = torch.from_numpy(bop_run.read_image(path)).pin_memory()
            t1 = time.perf_counter()
            row = dict(decode_ms=(t1 - t0) * 1e3)
            order = ("rle", "dense") if i % 2 == 0 else ("dense", "rle")
            for path_name in order:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                h0 = time.perf_counter()
                x = bop_run.image_inputs(dets, [], "hope", (H, W), str(i))
                if path_name == "rle":
                    out, ev = run_rle(rgb, x)
                else:
                    masks = dense_masks(x["counts"], x["offsets"], H, W)
                    out, ev = run_dense(rgb, masks, x)
                h1 = time.perf_counter()
                ev[2].synchronize()
                row[f"{path_name}_host_ms"] = (h1 - h0) * 1e3
                row[f"{path_name}_upload_ms"] = ev[0].elapsed_time(ev[1])
                row[f"{path_name}_crop_ms"] = ev[1].elapsed_time(ev[2])
                row[f"{path_name}_peak_mb"] = (torch.cuda.max_memory_allocated() - base) / 1e6
                if path_name == "rle":
                    crops = out
                else:
                    dense = out
            assert all(torch.equal(crops[k], dense[k]) for k in crops), "RLE and dense crops differ"
            import pandas as pd
            import src.megapose.utils.tensor_collection as tc
            nd = len(dets)
            labels = [str(d["category_id"]) for d in dets]
            batch = tc.PandasTensorCollection(
                infos=pd.DataFrame(dict(label=labels, scene_id=[1] * nd, view_id=[i] * nd)),
                tar_img=crops["tar_img"], tar_mask=crops["tar_mask"],
                tar_K=torch.eye(3, device=DEV).expand(nd, 3, 3).contiguous(), tar_M=crops["tar_M"])
            model.eval_retrieval(batch, idx_batch=i, dataset_name="timing")
            row["retrieval_ms"] = model.last_times["retrieval"] * 1e3
            rows.append(row)
    keys = rows[0].keys()
    return {k: float(np.median([r[k] for r in rows[1:]])) for k in keys}


def box_mesh(a, b, c):
    V = np.array([[x, y, z] for x in (-a, a) for y in (-b, b) for z in (-c, c)], np.float32)
    F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                  [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    return dict(vertices=V, faces=F, vertex_color=np.random.default_rng(1).uniform(0, 1, (8, 3)).astype(np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bop_run_time.py measures on the GPU"
    torch.cuda.set_device(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi[:1])
    with tempfile.TemporaryDirectory() as log:
        model = bop_run.build_model(DEV, log, seed=7)
        model.onboard_meshes("timing", [box_mesh(40, 30, 20), box_mesh(25, 50, 35)], fibonacci_view_poses(162, 400.0))
        for shape in SHAPES:
            result[shape] = measure(shape, model, a.images)
            print(shape, json.dumps(result[shape]), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=2)


if __name__ == "__main__":
    main()
