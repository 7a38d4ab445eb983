"""Row f16: onboarding from real frames with known poses, for objects without a CAD model (the BOP 2024 model-free
tasks, whose datasets ship `onboarding_static/` sequences of RGB frames with a visible mask, `cam_K` and the object
pose).  GigaPose is template based, so real views with known poses are all it needs, once each view meets the template
contract that pose lifting (src/models/poses.py) assumes: a camera that looks at the object origin, one K per object
(`render.TEMPLATE_K`), and a rotation that composes as R = R_inplane R_template.

`recentre` gives the exact fix: a virtual camera at the frame's centre, rotated by R_v so that its axis passes
through the object origin, sees the frame through H = K_t R_v K_f^-1 and has the pose [R_v R | (0, 0, |t|)].
`select_views` picks, for every template viewpoint, the frame that sees the object from the nearest direction, and
`recentre_boxes` / `recentre_crop` (csrc/onboard.cu) turn the chosen frames into template crops on the GPU.
Everything on the host is fp64 numpy; `read_onboarding_static` reads a dataset's onboarding_static/ tree.
"""
from __future__ import annotations

import concurrent.futures
import ctypes as C
import json
import os

import numpy as np
import torch

from . import _lib
from ._lib import check

TARGET_SIZE = 224
DECODE_THREADS = 8           # frames decoded at once on the host
CHUNK = 16                   # frames uploaded and cropped per launch pair


class OnboardingError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------- geometry
def _skew(a):
    return np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])


def recentre(K, pose, K_template=None):
    """K [3,3] of the frame, pose [4,4] (or [3,4]) object -> camera, both fp64 -> (R_v [3,3], virtual pose [4,4],
    H^-1 [3,3] virtual pixel -> frame pixel), with K_template = `render.TEMPLATE_K` by default.

    R_v is the minimal rotation taking the viewing ray t / |t| to +z (Rodrigues about t^ x z^, in the form
    I + [a]x + [a]x^2 / (1 + c) with a = t^ x z^ and c = t^ . z^), exactly I when t_x = t_y = 0; the virtual pose is
    [R_v R | (0, 0, |t|)] and H^-1 = K_f R_v^T K_t^-1.  A pose with t_z <= 0 (object not in front) is refused."""
    from .render import TEMPLATE_K
    Kf = np.asarray(K, np.float64).reshape(3, 3)
    Kt = np.asarray(TEMPLATE_K if K_template is None else K_template, np.float64).reshape(3, 3)
    P = np.asarray(pose, np.float64)
    R, t = P[:3, :3], P[:3, 3]
    if not np.all(np.isfinite(P[:3])) or not t[2] > 0:
        raise OnboardingError(f"pose translation {t.tolist()} is not in front of the camera (t_z must be > 0)")
    norm = float(np.linalg.norm(t))
    d = t / norm
    if t[0] == 0 and t[1] == 0:
        Rv = np.eye(3)
    else:
        a = np.array([d[1], -d[0], 0.0])                       # d x (0, 0, 1)
        A = _skew(a)
        Rv = np.eye(3) + A + (A @ A) / (1.0 + d[2])
    virtual = np.eye(4)
    virtual[:3, :3] = Rv @ R
    virtual[:3, 3] = (0.0, 0.0, norm)
    Hinv = Kf @ Rv.T @ np.linalg.inv(Kt)
    return Rv, virtual, Hinv


def view_directions(poses):
    """Unit camera directions in the object frame, -R^T t / |t|, of poses [n,4,4] -> [n,3] fp64.  Re-centring leaves
    them unchanged (R_v is a rotation about the camera centre)."""
    P = np.asarray(poses, np.float64).reshape(-1, 4, 4)
    c = -np.einsum("nji,nj->ni", P[:, :3, :3], P[:, :3, 3])
    return c / np.linalg.norm(c, axis=1, keepdims=True)


def select_views(frame_poses, template_poses, valid=None):
    """For every template pose, the frame whose camera direction in the object frame is nearest (largest cosine; a tie
    goes to the lowest frame index), among the frames with valid[i] (default all) -> (frame ids i64 [T], angular gaps
    f64 [T] in degrees)."""
    f = view_directions(frame_poses)
    t = view_directions(template_poses)
    ok = np.ones(len(f), bool) if valid is None else np.asarray(valid, bool).reshape(-1)
    if ok.shape != (len(f),):
        raise OnboardingError(f"valid has {ok.shape[0]} entries for {len(f)} frames")
    if not ok.any():
        raise OnboardingError("no frame has a non-empty mask")
    cos = t @ f.T                                               # [T, n]
    cos[:, ~ok] = -np.inf
    ids = np.argmax(cos, axis=1)                                # first maximum: the lowest frame index
    gaps = np.degrees(np.arccos(np.clip(cos[np.arange(len(t)), ids], -1.0, 1.0)))
    return ids.astype(np.int64), gaps


def mask_box(mask):
    """xyxy box (exclusive max) of the non-zero pixels of a [H,W] mask; (0, 0, 0, 0) when it has none."""
    m = np.asarray(mask) != 0
    rows, cols = np.flatnonzero(m.any(1)), np.flatnonzero(m.any(0))
    if not len(rows):
        return np.zeros(4, np.int64)
    return np.array([cols[0], rows[0], cols[-1] + 1, rows[-1] + 1], np.int64)


# ---------------------------------------------------------------------------------------------------- GPU launches
@torch.no_grad()
def recentre_boxes(masks, hinv, src_boxes):
    """masks u8 [n,H,W] on a CUDA device, hinv [n,3,3] and src_boxes [n,4] (`mask_box`) on the host -> boxes i64 [n,4]
    on the device: the xyxy boxes of the re-centred masks on the unbounded virtual grid (gp_recentre_boxes)."""
    if not masks.is_cuda or masks.dtype != torch.uint8 or masks.dim() != 3:
        raise _lib.GigaPoseNativeError("recentre_boxes takes u8 [n,H,W] CUDA masks (no CPU fallback)")
    n, H, W = masks.shape
    h = np.ascontiguousarray(np.asarray(hinv, np.float64).reshape(n, 9))
    b = np.ascontiguousarray(np.asarray(src_boxes, np.int64).reshape(n, 4))
    out = torch.empty(n, 4, dtype=torch.int64, device=masks.device)
    masks = masks.contiguous()
    with torch.cuda.device(masks.device):
        check(_lib.load().gp_recentre_boxes(n, H, W, masks.data_ptr(), h.ctypes.data_as(C.POINTER(C.c_double)),
                                            b.ctypes.data_as(C.POINTER(C.c_int64)), out.data_ptr(),
                                            torch.cuda.current_stream(masks.device).cuda_stream))
    return out


@torch.no_grad()
def recentre_crop(images, masks, hinv, boxes, target_size=TARGET_SIZE):
    """images u8 [n,H,W,3] and masks u8 [n,H,W] on a CUDA device, hinv [n,3,3] on the host, boxes i64 [n,4] (device)
    -> dict(images f32 [n,3,T,T] masked and CLIP-normalised, mask f32 [n,T,T], M f32 [n,3,3]) (gp_recentre_crop)."""
    if not images.is_cuda or images.dtype != torch.uint8 or images.dim() != 4 or images.shape[-1] != 3:
        raise _lib.GigaPoseNativeError("recentre_crop takes u8 [n,H,W,3] CUDA images (no CPU fallback)")
    n, H, W, _ = images.shape
    dev = images.device
    if tuple(masks.shape) != (n, H, W) or masks.dtype != torch.uint8:
        raise ValueError(f"masks must be u8 [{n},{H},{W}], got {masks.dtype} {tuple(masks.shape)}")
    h = np.ascontiguousarray(np.asarray(hinv, np.float64).reshape(n, 9))
    boxes = torch.as_tensor(boxes, device=dev).long().contiguous()
    T = int(target_size)
    out = torch.empty(n, 3, T, T, device=dev)
    out_mask = torch.empty(n, T, T, device=dev)
    M = torch.empty(n, 3, 3, device=dev)
    images, masks = images.contiguous(), masks.to(dev).contiguous()
    with torch.cuda.device(dev):
        check(_lib.load().gp_recentre_crop(n, H, W, T, images.data_ptr(), masks.data_ptr(),
                                           h.ctypes.data_as(C.POINTER(C.c_double)), boxes.data_ptr(), out.data_ptr(),
                                           out_mask.data_ptr(), M.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return {"images": out, "mask": out_mask, "M": M}


# ---------------------------------------------------------------------------------------------------- frames
def read_rgb(x):
    """Path -> u8 [H,W,3] as decoded (gray repeated); a u8 array / tensor passes through."""
    if isinstance(x, (str, os.PathLike)):
        from .bop_run import read_image
        return read_image(x)
    a = x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise OnboardingError(f"an onboarding image must be u8 [H,W,3], got {a.dtype} {a.shape}")
    return a


def read_mask(x):
    """Path (PNG) -> u8 [H,W] with 1 where the mask is non-zero; arrays / tensors likewise."""
    if isinstance(x, (str, os.PathLike)):
        from PIL import Image
        with Image.open(x) as im:
            a = np.asarray(im)
    else:
        a = x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    if a.ndim == 3:
        a = a[..., 0]
    if a.ndim != 2:
        raise OnboardingError(f"an onboarding mask must be [H,W], got shape {a.shape}")
    return (a != 0).astype(np.uint8)


def read_depth(x, depth_scale):
    """Path (16-bit PNG) or array / tensor [H,W] -> f32 [H,W] in the unit of the poses: the raw values x depth_scale
    in fp64, rounded once to f32 (`bop_eval.load_depth`'s rule); 0 = missing."""
    if isinstance(x, (str, os.PathLike)):
        from PIL import Image
        with Image.open(x) as im:
            a = np.asarray(im)
    else:
        a = x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    if a.ndim != 2:
        raise OnboardingError(f"an onboarding depth image must be [H,W], got shape {a.shape}")
    return (a.astype(np.float64) * float(depth_scale)).astype(np.float32)


class Frames:
    """One object's onboarding frames: images and masks (paths, or u8 arrays / tensors [H,W,3] and [H,W]), K [n,3,3]
    and poses [n,4,4] object -> camera.  Masks are decoded once, when first asked for (`valid`, `load`).  Optional
    depths (16-bit PNG paths or arrays [H,W]) with depth_scale (one value, or one per frame; default 1) hold the
    depth images of row f17's reconstruction (`load_depth`)."""

    def __init__(self, images, masks, K, poses, depths=None, depth_scale=None):
        self.images, self.masks = list(images), list(masks)
        n = len(self.images)
        self.K = np.asarray(K, np.float64).reshape(-1, 3, 3)
        self.poses = np.asarray(poses, np.float64).reshape(-1, 4, 4)
        if len(self.masks) != n or self.K.shape[0] != n or self.poses.shape[0] != n:
            raise OnboardingError(f"{n} images, {len(self.masks)} masks, {self.K.shape[0]} K and "
                                  f"{self.poses.shape[0]} poses: one of each per frame")
        if n == 0:
            raise OnboardingError("an object has no onboarding frames")
        self.depths = None if depths is None else list(depths)
        if self.depths is not None and len(self.depths) != n:
            raise OnboardingError(f"{n} frames and {len(self.depths)} depth images: one per frame")
        scale = np.broadcast_to(np.asarray(1.0 if depth_scale is None else depth_scale, np.float64), (n,)).copy()
        if not np.all(np.isfinite(scale) & (scale > 0)):
            raise OnboardingError("depth_scale must be positive and finite")
        self.depth_scale = scale
        self.boxes = {}                                         # frame -> source mask box, once decoded

    def __len__(self):
        return len(self.images)

    def mask(self, i):
        m = read_mask(self.masks[i])
        self.boxes[i] = mask_box(m)
        return m

    def load(self, i):
        """-> (rgb u8 [H,W,3], mask u8 [H,W]) of frame i."""
        rgb, m = read_rgb(self.images[i]), self.mask(i)
        if rgb.shape[:2] != m.shape:
            raise OnboardingError(f"frame {i}: image {rgb.shape[:2]} and mask {m.shape} differ in size"
                                  + (f" ({self.images[i]})" if isinstance(self.images[i], (str, os.PathLike)) else ""))
        return rgb, m

    def load_depth(self, i):
        """-> depth f32 [H,W] of frame i in the unit of the poses (0 = missing)."""
        if self.depths is None:
            raise OnboardingError("these frames carry no depth images")
        return read_depth(self.depths[i], self.depth_scale[i])


def select_frames(frames, template_poses, pool=None):
    """`select_views` over the frames whose masks are not empty.  Only the masks of frames that win a template view
    are decoded: a chosen frame whose mask turns out empty leaves the candidates and the selection is repeated, which
    ends in the selection over all non-empty frames.  -> (ids [T], gaps in degrees [T])."""
    valid = np.ones(len(frames), bool)
    while True:
        ids, gaps = select_views(frames.poses, template_poses, valid)
        todo = [int(i) for i in np.unique(ids) if int(i) not in frames.boxes]
        if todo:
            list((pool.map if pool is not None else map)(frames.mask, todo))
        empty = [i for i in np.unique(ids) if frames.boxes[int(i)][2] <= frames.boxes[int(i)][0]]
        if not empty:
            return ids, gaps
        valid[empty] = False


def recentre_frames(frames, ids, device, pool=None):
    """Re-centred template crops of frames `ids` (repeats allowed): the unique frames are decoded on `pool`'s threads
    CHUNK at a time, a chunk ahead of the one on the GPU, uploaded and cropped -> dict(images [n,3,T,T], mask [n,T,T],
    M [n,3,3], poses f64 [n,4,4] the virtual poses, boxes i64 [n,4] the virtual boxes)."""
    ids = np.asarray(ids, np.int64).reshape(-1)
    uniq, inv = np.unique(ids, return_inverse=True)
    own = pool is None
    pool = pool or concurrent.futures.ThreadPoolExecutor(DECODE_THREADS)
    try:
        futures = {}

        def submit(c0):
            for i in uniq[c0:c0 + CHUNK]:
                futures[int(i)] = pool.submit(frames.load, int(i))

        submit(0)
        parts = []
        for c0 in range(0, len(uniq), CHUNK):
            if c0 + CHUNK < len(uniq):
                submit(c0 + CHUNK)
            chunk = [int(i) for i in uniq[c0:c0 + CHUNK]]
            loaded = [futures.pop(i).result() for i in chunk]
            shapes = {rgb.shape for rgb, _ in loaded}
            if len(shapes) != 1:
                raise OnboardingError(f"frames {chunk} have different sizes {sorted(shapes)}; one object's frames share "
                                      f"one size")
            maps = [recentre(frames.K[i], frames.poses[i]) for i in chunk]
            hinv = np.stack([m[2] for m in maps])
            rgb = torch.from_numpy(np.stack([x[0] for x in loaded])).pin_memory().to(device, non_blocking=True)
            mask = torch.from_numpy(np.stack([x[1] for x in loaded])).pin_memory().to(device, non_blocking=True)
            src = np.stack([frames.boxes[i] for i in chunk])
            boxes = recentre_boxes(mask, hinv, src)
            b = boxes.cpu().numpy()
            empty = [chunk[j] for j in range(len(chunk)) if b[j, 2] <= b[j, 0] or b[j, 3] <= b[j, 1]]
            if empty:
                raise OnboardingError(f"frames {empty}: the re-centred mask is empty (the mask is too small to sample)")
            crop = recentre_crop(rgb, mask, hinv, boxes)
            parts.append((crop, np.stack([m[1] for m in maps]), b))
    finally:
        if own:
            pool.shutdown(wait=True)
    cat = lambda k: torch.cat([p[0][k] for p in parts])
    sel = torch.as_tensor(inv, device=device)
    return dict(images=cat("images")[sel], mask=cat("mask")[sel], M=cat("M")[sel],
                poses=np.concatenate([p[1] for p in parts])[inv], boxes=np.concatenate([p[2] for p in parts])[inv])


# ---------------------------------------------------------------------------------------------------- dataset reader
def _load_json(path):
    if not os.path.exists(path):
        raise OnboardingError(f"{path} not found")
    with open(path) as f:
        return json.load(f)


def read_onboarding_static(dataset_dir, depth=False):
    """The dataset's onboarding_static/ tree (the layout of the BOP 2024 H3 datasets: one directory per scene, e.g.
    obj_000001_up and obj_000001_down, each with rgb/{im:06d}.jpg (or .png), mask_visib/{im:06d}_000000.png,
    scene_gt.json and scene_camera.json, one object per scene) -> {obj_id: Frames} with the up and down scenes of each
    object together, in scene then image order.  Refuses, naming the file or scene: a scene whose scene_gt holds more
    than one object, a missing mask or image, object ids that are not 1 .. N, and, when models/models_info.json exists,
    an id set that differs from it.  With `depth` (row f17) the frames also carry depth/{im:06d}.png and the image's
    `depth_scale` from scene_camera.json; a missing depth image or depth_scale is refused, naming it."""
    root = os.path.join(dataset_dir, "onboarding_static")
    if not os.path.isdir(root):
        raise OnboardingError(f"{root} not found: model-free onboarding reads the onboarding_static sequences")
    scenes = sorted(d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d)))
    if not scenes:
        raise OnboardingError(f"{root} holds no scene directories")
    per_obj = {}
    for sc in scenes:
        d = os.path.join(root, sc)
        gt = _load_json(os.path.join(d, "scene_gt.json"))
        cam = _load_json(os.path.join(d, "scene_camera.json"))
        ids = {int(e["obj_id"]) for v in gt.values() for e in v}
        if len(ids) != 1 or any(len(v) != 1 for v in gt.values()):
            raise OnboardingError(f"{os.path.join(d, 'scene_gt.json')}: scene {sc} must show one object once per image, "
                                  f"found objects {sorted(ids)}")
        obj = ids.pop()
        acc = per_obj.setdefault(obj, dict(images=[], masks=[], K=[], poses=[], depths=[], depth_scale=[]))
        for im in sorted(int(k) for k in gt):
            e = gt[str(im)][0]
            if str(im) not in cam:
                raise OnboardingError(f"{os.path.join(d, 'scene_camera.json')}: no camera for image {im}")
            rgb = next((p for p in (os.path.join(d, "rgb", f"{im:06d}.{x}") for x in ("jpg", "png")) if os.path.exists(p)),
                       None)
            if rgb is None:
                raise OnboardingError(f"{os.path.join(d, 'rgb', f'{im:06d}.jpg')} not found (nor .png)")
            mask = os.path.join(d, "mask_visib", f"{im:06d}_000000.png")
            if not os.path.exists(mask):
                raise OnboardingError(f"{mask} not found")
            pose = np.eye(4)
            pose[:3, :3] = np.asarray(e["cam_R_m2c"], np.float64).reshape(3, 3)
            pose[:3, 3] = np.asarray(e["cam_t_m2c"], np.float64).reshape(3)
            acc["images"].append(rgb)
            acc["masks"].append(mask)
            acc["K"].append(np.asarray(cam[str(im)]["cam_K"], np.float64).reshape(3, 3))
            acc["poses"].append(pose)
            if depth:
                dpath = os.path.join(d, "depth", f"{im:06d}.png")
                if not os.path.exists(dpath):
                    raise OnboardingError(f"{dpath} not found: reconstruction fuses the onboarding depth images")
                if "depth_scale" not in cam[str(im)]:
                    raise OnboardingError(f"{os.path.join(d, 'scene_camera.json')}: image {im} has no depth_scale")
                acc["depths"].append(dpath)
                acc["depth_scale"].append(float(cam[str(im)]["depth_scale"]))
    found = sorted(per_obj)
    if found != list(range(1, len(found) + 1)):
        raise OnboardingError(f"{root}: object ids {found} are not 1 .. {len(found)}: labels index the template bank")
    info = os.path.join(dataset_dir, "models", "models_info.json")
    if os.path.exists(info):
        listed = sorted(int(k) for k in _load_json(info))
        if listed != found:
            raise OnboardingError(f"{info} lists objects {listed} but {root} has objects {found}")
    return {o: Frames(v["images"], v["masks"], np.stack(v["K"]), np.stack(v["poses"]),
                      v["depths"] if depth else None, v["depth_scale"] if depth else None)
            for o, v in sorted(per_obj.items())}

