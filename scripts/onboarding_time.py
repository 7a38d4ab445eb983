"""Times model-free onboarding (row f16) per object on a HOPE-shaped case: 1920 x 1080 JPEG frames, about 300 per
object over an up and a down sequence, 162 template views (level 1) of which each takes its nearest frame.  Reports the
host decode (JPEG + PNG mask, on the decode threads), the upload, gp_recentre_boxes and gp_recentre_crop (CUDA events),
both encoders and the bank write, `GigaPose.onboard_images` end to end, and `onboard_meshes` on 10^4-face meshes for
comparison.  The frames are synthetic renders written to a temporary directory; the card name and power limit are read
in the same run.

    python scripts/onboarding_time.py [--objects 2] [--frames 300] [--out results.json]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gigapose_b200 import onboarding, render  # noqa: E402
from gigapose_b200.template_poses import template_poses  # noqa: E402

K_HOPE = np.array([[1390.0, 0, 961.5], [0, 1390.0, 538.5], [0, 0, 1]])
H, W = 1080, 1920


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def frames_of(mesh, n, d, seed):
    """n frames around the object (half above, half below), 350-600 mm away, the object up to 15 deg off the axis,
    written as JPEG + PNG mask under d -> onboarding.Frames."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    images, masks, poses = [], [], []
    os.makedirs(d, exist_ok=True)
    for i in range(n):
        z = (1 if i < n // 2 else -1) * rng.uniform(0.05, 0.95)
        ph = rng.uniform(0, 2 * np.pi)
        cam = np.array([np.sqrt(1 - z * z) * np.cos(ph), np.sqrt(1 - z * z) * np.sin(ph), z])
        fwd = -cam
        x = np.cross([0.0, 0.0, 1.0], fwd)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(fwd, x), fwd])
        a = rng.normal(size=3)
        a *= np.radians(rng.uniform(0, 15)) / np.linalg.norm(a)
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        th = np.linalg.norm(a)
        Ra = np.eye(3) + np.sin(th) / th * Kx + (1 - np.cos(th)) / th ** 2 * Kx @ Kx
        P = np.eye(4)
        P[:3, :3] = Ra @ R
        P[:3, 3] = P[:3, :3] @ (-cam * rng.uniform(350, 600))
        r = render.render_templates(mesh, torch.as_tensor(P, dtype=torch.float32)[None], K_HOPE, size=(H, W))
        rgb = (r["rgba"][0, :3].permute(1, 2, 0) * 255).round().byte().cpu().numpy()
        m = (r["rgba"][0, 3] > 0).byte().cpu().numpy() * 255
        Image.fromarray(rgb).save(os.path.join(d, f"{i:06d}.jpg"), quality=95)
        Image.fromarray(m).save(os.path.join(d, f"{i:06d}_000000.png"))
        images.append(os.path.join(d, f"{i:06d}.jpg"))
        masks.append(os.path.join(d, f"{i:06d}_000000.png"))
        poses.append(P)
    return onboarding.Frames(images, masks, np.stack([K_HOPE] * n), np.stack(poses))


def stages(frames, tpl, device):
    """The stages of one object's onboarding, timed one after another."""
    ids, gaps = onboarding.select_frames(frames, tpl)
    uniq = np.unique(ids)
    t0 = time.perf_counter()
    loaded = [frames.load(int(i)) for i in uniq]
    decode_s = time.perf_counter() - t0
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    hinv = np.stack([onboarding.recentre(frames.K[i], frames.poses[i])[2] for i in uniq])
    src = np.stack([frames.boxes[int(i)] for i in uniq])
    rgb_h = torch.from_numpy(np.stack([x[0] for x in loaded])).pin_memory()
    mask_h = torch.from_numpy(np.stack([x[1] for x in loaded])).pin_memory()
    ev[0].record()
    rgb, mask = rgb_h.to(device, non_blocking=True), mask_h.to(device, non_blocking=True)
    ev[1].record()
    boxes = onboarding.recentre_boxes(mask, hinv, src)
    ev[2].record()
    crop = onboarding.recentre_crop(rgb, mask, hinv, boxes)
    ev[3].record()
    torch.cuda.synchronize()
    return dict(selected_frames=int(len(uniq)), gap_max_deg=float(gaps.max()), decode_s=decode_s,
                upload_ms=ev[0].elapsed_time(ev[1]), boxes_ms=ev[1].elapsed_time(ev[2]),
                crop_ms=ev[2].elapsed_time(ev[3]), crops=crop)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=2)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "onboarding_time.py measures on the GPU; there is no CPU path"
    torch.cuda.set_device(0)
    device = torch.device("cuda:0")
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from render_time import uv_sphere
    import bench
    tpl = template_poses(1, "all")
    meshes = [uv_sphere(51, 100, seed=o) for o in range(args.objects)]
    res = dict(card=card(), frame_size=[H, W], frames_per_object=args.frames, views=len(tpl))
    with tempfile.TemporaryDirectory() as tmp:
        objs = [frames_of(m, args.frames, os.path.join(tmp, f"obj{o}"), o) for o, m in enumerate(meshes)]
        model = bench.build_models(device)
        per = [stages(objs[0], tpl, device)]                               # warm-up
        per = [stages(f, tpl, device) for f in objs]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        enc = []
        for p in per:
            ev[0].record()
            model.ae_net.raw_tokens(p["crops"]["images"][:64])
            model.ist_net.forward_by_chunk(p["crops"]["images"][:64])
            ev[1].record()
            torch.cuda.synchronize()
            enc.append(ev[0].elapsed_time(ev[1]) / 64 * len(tpl))
            del p["crops"]
        res["per_object"] = per
        res["encoders_ms_per_object_est"] = float(np.mean(enc))
        model.onboard_images("warmup", objs[:1], tpl)
        objs = [onboarding.Frames(f.images, f.masks, f.K, f.poses) for f in objs]      # masks decoded afresh
        model.onboard_images("timed", objs, tpl)
        res["onboard_images_s_per_object"] = model.onboarding_s_per_object
        model.onboard_meshes("mesh_warmup", meshes[:1], tpl)
        model.onboard_meshes("mesh_timed", meshes, tpl)
        res["onboard_meshes_s_per_object"] = model.onboarding_s_per_object
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
