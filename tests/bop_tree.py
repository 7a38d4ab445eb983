"""Synthetic BOP dataset trees for the evaluation tests (tests/test_bop_eval_cpu.py, tests/test_gpu_bop_eval.py): ascii
PLY models, models_info.json, test_targets_bop19.json and per scene scene_gt.json, scene_gt_info.json,
scene_camera.json and 16-bit PNG depth, in the layout of a BOP dataset directory."""
import json
import os

import numpy as np


def write_ply(path, V, F):
    with open(path, "w") as f:
        f.write(f"ply\nformat ascii 1.0\nelement vertex {len(V)}\nproperty float x\nproperty float y\nproperty float z\n"
                f"element face {len(F)}\nproperty list uchar int vertex_indices\nend_header\n")
        for v in V:
            f.write(" ".join(repr(float(x)) for x in v) + "\n")
        for t in F:
            f.write("3 " + " ".join(str(int(i)) for i in t) + "\n")


def write_png16(path, a):
    from PIL import Image
    Image.fromarray(np.asarray(a, np.uint16)).save(path)


def write_tree(root, models, info, scenes, targets, split="test"):
    """models {obj_id: (V, F)}; info {obj_id: models_info entry}; scenes {scene_id: {im_id: dict(gt=[(obj_id, R [3,3],
    t [3])], visib=[float], K [3,3], depth_scale, png uint16 [H,W])}}; targets [(scene, im, obj, inst_count)]."""
    mdir = os.path.join(root, "models")
    os.makedirs(mdir, exist_ok=True)
    for o, (V, F) in models.items():
        write_ply(os.path.join(mdir, f"obj_{o:06d}.ply"), V, F)
    with open(os.path.join(mdir, "models_info.json"), "w") as f:
        json.dump({str(o): v for o, v in info.items()}, f)
    with open(os.path.join(root, "test_targets_bop19.json"), "w") as f:
        json.dump([dict(scene_id=s, im_id=i, obj_id=o, inst_count=n) for s, i, o, n in targets], f)
    for s, ims in scenes.items():
        d = os.path.join(root, split, f"{s:06d}")
        os.makedirs(os.path.join(d, "depth"), exist_ok=True)
        gt, gi, cam = {}, {}, {}
        for im, v in ims.items():
            gt[str(im)] = [dict(cam_R_m2c=np.asarray(R, float).reshape(-1).tolist(),
                                cam_t_m2c=np.asarray(t, float).reshape(-1).tolist(), obj_id=o) for o, R, t in v["gt"]]
            gi[str(im)] = [dict(visib_fract=float(x)) for x in v["visib"]]
            cam[str(im)] = dict(cam_K=np.asarray(v["K"], float).reshape(-1).tolist(), depth_scale=v["depth_scale"])
            write_png16(os.path.join(d, "depth", f"{im:06d}.png"), v["png"])
        for name, obj in (("scene_gt.json", gt), ("scene_gt_info.json", gi), ("scene_camera.json", cam)):
            with open(os.path.join(d, name), "w") as f:
                json.dump(obj, f)


def tetra(size=50.0):
    V = np.array([[0, 0, 0], [size, 0, 0], [0, size, 0], [0, 0, size]], np.float32)
    return V, np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)


def spheroid(a=40.0, c=25.0, n_lat=24, n_lon=96):
    """An ellipsoid of revolution about z with radii (a, a, c), n_lon segments: exactly symmetric under rotations by
    multiples of 2 pi / n_lon about z (as a vertex set)."""
    th = np.linspace(0, np.pi, n_lat)[1:-1, None]
    ph = np.arange(n_lon)[None] * (2 * np.pi / n_lon)
    ring = np.stack([a * np.sin(th) * np.cos(ph), a * np.sin(th) * np.sin(ph), c * np.cos(th) + 0 * ph], -1).reshape(-1, 3)
    V = np.concatenate([ring, [[0, 0, c], [0, 0, -c]]]).astype(np.float32)
    F, L = [], n_lat - 2
    for i in range(L - 1):
        for j in range(n_lon):
            p, q = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            F += [[p, p + n_lon, q], [q, p + n_lon, q + n_lon]]
    top, bot = len(V) - 2, len(V) - 1
    for j in range(n_lon):
        F += [[top, j, (j + 1) % n_lon], [bot, (L - 1) * n_lon + (j + 1) % n_lon, (L - 1) * n_lon + j]]
    return V, np.array(F, np.int32)


def rot(axis, deg):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    t = np.deg2rad(deg)
    return np.eye(3) + np.sin(t) * k + (1 - np.cos(t)) * (k @ k)
