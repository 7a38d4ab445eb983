"""BOP onboarding_static/ scenes with depth, for the row f17 tests (tests/test_reconstruct_cpu.py,
tests/test_gpu_reconstruct.py): rgb/{im:06d}.png, mask_visib/{im:06d}_000000.png, depth/{im:06d}.png (16-bit),
scene_gt.json and scene_camera.json with cam_K and depth_scale, one object per scene."""
import json
import os

import numpy as np


def write_scene(ds, name, obj, frames, depth_scale=1.0, skip_depth=(), skip_scale=()):
    """frames: [(rgb u8 [H,W,3], mask [H,W], depth raw u16 [H,W], pose [4,4], K [3,3])]; the depth PNG of the images in
    `skip_depth` and the depth_scale of those in `skip_scale` are left out."""
    from PIL import Image
    d = os.path.join(ds, "onboarding_static", name)
    for sub in ("rgb", "mask_visib", "depth"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    gt, cam = {}, {}
    for im, (rgb, mask, depth, P, K) in enumerate(frames):
        Image.fromarray(np.asarray(rgb, np.uint8)).save(os.path.join(d, "rgb", f"{im:06d}.png"))
        Image.fromarray((np.asarray(mask) != 0).astype(np.uint8) * 255).save(
            os.path.join(d, "mask_visib", f"{im:06d}_000000.png"))
        if im not in skip_depth:
            Image.fromarray(np.asarray(depth, np.uint16)).save(os.path.join(d, "depth", f"{im:06d}.png"))
        P = np.asarray(P, np.float64)
        gt[str(im)] = [dict(obj_id=obj, cam_R_m2c=P[:3, :3].reshape(-1).tolist(), cam_t_m2c=P[:3, 3].tolist())]
        cam[str(im)] = dict(cam_K=np.asarray(K, np.float64).reshape(-1).tolist())
        if im not in skip_scale:
            cam[str(im)]["depth_scale"] = depth_scale
    for fname, v in (("scene_gt.json", gt), ("scene_camera.json", cam)):
        with open(os.path.join(d, fname), "w") as f:
            json.dump(v, f)
    return d


def look_at_pose(cam, dist, tilt=None):
    """Object -> camera pose of a camera at unit direction `cam` x dist looking at the object origin; `tilt` [3,3]
    rotates the camera about its centre afterwards (an off-centre view)."""
    cam = np.asarray(cam, np.float64) / np.linalg.norm(cam)
    fwd = -cam
    up = np.array([0.0, 0.0, 1.0]) if abs(fwd[2]) < 0.99 else np.array([0.0, 1.0, 0.0])
    x = np.cross(up, fwd)
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(fwd, x), fwd])
    if tilt is not None:
        R = tilt @ R
    P = np.eye(4)
    P[:3, :3] = R
    P[:3, 3] = R @ (-cam * dist)
    return P


def up_down_directions(n, rng):
    """n camera directions, half above the object's xy plane and half below (the up and down sequences)."""
    out = []
    for k in range(n):
        z = (1.0 if k < n // 2 else -1.0) * rng.uniform(0.15, 0.9)
        ph = rng.uniform(0, 2 * np.pi)
        out.append(np.array([np.sqrt(1 - z * z) * np.cos(ph), np.sqrt(1 - z * z) * np.sin(ph), z]))
    return out
