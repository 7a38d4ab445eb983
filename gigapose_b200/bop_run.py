"""Row f9: GigaPose on a BOP test split, from the dataset directory and its default CNOS detections to the results csv
(and, with --evaluate, to scores_bop19.json / scores_bop24.json) -- the reference's `test.py` with its test dataloader
(dataloader/test.py, utils/inout.py:370-492) and Lightning loop, without Hydra, Lightning, webdataset or the BOP toolkit.

Each image is one step, as in test.py:55-60: its CNOS masks stay COCO run-length encodings and are cropped on the GPU
(`preprocess.crop_detections_rle`, gp_crop_resize_pad_rle), then `GigaPose.eval_retrieval` writes the step's
predictions/{idx}.npz, and `save_predictions_from_batched_predictions` writes the csv at the end.  A background thread
decodes the next image into pinned memory while the current one runs.  INTEGRATION.md lists every deviation from
test.py.

Row f10, `--refine-depth H`: the reference's second stage (refine.py -> pose_estimator.run_inference_pipeline,
src/megapose/inference/pose_estimator.py:580-623) on the depth images of the split.  The first H hypotheses of every
instance that reaches the coarse csv are refined with the point-to-plane ICP (`GigaPose.refine_depth`, no masks, as
run_depth_refiner passes none, pose_estimator.py:501-503), the refined hypotheses are scored against the depth image
(gp_depth_score) and the best one per instance goes to refined_predictions/{idx}.npz and a second csv,
`..._{run_id}_icp.csv`.  The depth PNG is decoded on the thread that decodes the next RGB image.

Row f11, `--refine-masks` with `--refine-depth H`: each kept instance is refined with its own CNOS mask, the run-length
encoding decoded on the GPU over the mask's box, as the target set and as the region its target normals are smoothed
in (`GigaPose.refine_depth(mask_normals=True)`); the csv is `..._{run_id}_icp_masked.csv`.

Row f13, `--depth-refiner teaserpp` with `--refine-depth H`: the hypotheses go through MegaPose's TEASER++ refiner
(`GigaPose.refine_depth(refiner="teaserpp")`) instead of the ICP, with the same ranking; the csv is
`..._{run_id}_teaserpp.csv`.  Usage:

    python -m gigapose_b200.bop_run --dataset-dir D --checkpoint gigaPose_v1.ckpt
        [--template-poses P.npy | [--template-level 0|1|2] [--pose-distribution all|upper]]
        [--setting localization|detection] [--detections FILE] [--out DIR]
        [--refine-depth H [--refine-masks | --depth-refiner teaserpp]] [--onboarding models|static [--reconstruct]]
        [--evaluate]

Row f15: without --template-poses the templates are the reference's test templates, generated
(`template_poses.template_poses`, level 1 and all views by default).

Row f16, `--onboarding static`: objects without CAD models.  The templates are built from the dataset's
onboarding_static/ frames (`onboard_static`, `GigaPose.onboard_images`) for the same template viewpoints; models/ is
not read, except models_info.json when it exists (to check the object ids) and by --evaluate, whose BOP metrics need
the models.  The depth refiners render the CAD model, so --refine-depth is refused unless --reconstruct builds one;
the default run id is `bop_run_static`.

Row f17, `--onboarding static --refine-depth H --reconstruct`: every object is reconstructed from its onboarding depth
images (`reconstruct.reconstruct`), written to <out>/reconstructed/obj_{id:06d}.ply and attached for the depth
refiners, which then run as with CAD models.  Under `torchrun --nproc-per-node N -m
gigapose_b200.bop_run ...` each rank runs its share of the images on its own GPU (`main_ranks`).
"""
from __future__ import annotations

import argparse
import concurrent.futures
import copy
import glob
import json
import os
import pickle
import types

import numpy as np
import torch

from .bop_eval import load_cameras, load_depth
from .teaser import REFINERS

CAP_PER_TARGET = 16             # localization: detections kept per target (dataloader/test.py:110-114)
CAP_PER_TARGET_ICBIN = 32
TOP_K = 5                       # hypotheses per detection (configs/model/large.yaml)
LMO_INDEX_TO_ID = [1, 5, 6, 8, 9, 10, 11, 12]      # src/utils/dataset.py: the LM-O labels the model is indexed with
LMO_ID_TO_INDEX = {o: i + 1 for i, o in enumerate(LMO_INDEX_TO_ID)}


class BopRunError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------- dataset layout
def split_name(dataset_name):
    """(split, model directory) of a dataset's test images (`get_split_name`, dataloader/test.py:155-165)."""
    split = "test_primesense" if dataset_name in ("hb", "tless") else "test"
    return split, "models_cad" if dataset_name == "tless" else "models"


def detection_year(dataset_name):
    """(BOP year, CNOS variant) of the default detections (utils/inout.py:408-417)."""
    if dataset_name in ("lmo", "tless", "tudl", "icbin", "itodd", "hb", "ycbv"):
        return "19", "cnos-fastsam"
    if dataset_name == "hope":
        return "24", "cnos-sam"
    raise BopRunError(f"dataset {dataset_name!r} has no default detections; pass --detections")


def default_detections(dataset_dir):
    """<parent of dataset_dir>/default_detections/core{19,24}_model_based_unseen/cnos-*/ : the first file (by name)
    whose name contains the dataset name (utils/inout.py:418-424, which takes the first in directory order)."""
    name = os.path.basename(os.path.normpath(dataset_dir))
    year, model = detection_year(name)
    d = os.path.join(os.path.dirname(os.path.abspath(dataset_dir)), "default_detections",
                     f"core{year}_model_based_unseen", model)
    found = sorted(f for f in os.listdir(d) if name in f) if os.path.isdir(d) else []
    if not found:
        raise BopRunError(f"no detection file for {name!r} in {d}")
    return os.path.join(d, found[0])


def image_path(dataset_dir, split, scene_id, im_id):
    """rgb/*.jpg, else rgb/*.png, else gray/*.tif (web_scene_dataset.py:38-45)."""
    d = os.path.join(dataset_dir, split, f"{scene_id:06d}")
    for sub, ext in (("rgb", "jpg"), ("rgb", "png"), ("gray", "tif")):
        p = os.path.join(d, sub, f"{im_id:06d}.{ext}")
        if os.path.exists(p):
            return p
    raise BopRunError(f"no image {im_id:06d}.jpg/.png under {d}/rgb nor .tif under {d}/gray")


def read_image(path):
    """-> u8 [H,W,3] as decoded; a gray image is repeated to three channels.  Refuses anything but 8-bit data."""
    from PIL import Image
    with Image.open(path) as im:
        a = np.asarray(im)
    if a.dtype != np.uint8:
        raise BopRunError(f"{path} holds {a.dtype} pixels; only 8-bit images are supported")
    if a.ndim == 2:
        a = np.stack([a, a, a], axis=-1)
    if a.ndim != 3 or a.shape[2] != 3:
        raise BopRunError(f"{path} has shape {a.shape}; expected [H,W] gray or [H,W,3] RGB")
    return a


# ---------------------------------------------------------------------------------------------------- RLE
def rle_from_string(s):
    """COCO's compressed RLE string (`rleFrString` of the COCO mask API) -> list of run lengths."""
    counts, p = [], 0
    data = s.encode() if isinstance(s, str) else bytes(s)
    while p < len(data):
        x, k, more = 0, 0, True
        while more:
            if p >= len(data):
                raise BopRunError("truncated compressed RLE string")
            c = data[p] - 48
            if not 0 <= c < 64:
                raise BopRunError(f"byte {data[p]!r} is not a compressed RLE character")
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return counts


def rle_counts(segmentation, shape, where):
    """A detection's `segmentation` (dict(size [H, W], counts: list or compressed string)) -> i32 run lengths, after
    checking that its size is the image's (H, W) and that no run is negative; `where` names the detection in errors."""
    size = [int(v) for v in segmentation.get("size", ())]
    if size != list(shape):
        raise BopRunError(f"{where}: mask size {size} differs from the image's {list(shape)}")
    c = segmentation.get("counts")
    if isinstance(c, (str, bytes)):
        c = rle_from_string(c)
    c = np.asarray(c, np.int64).reshape(-1)
    if c.size and c.min() < 0:
        raise BopRunError(f"{where}: negative run length {int(c.min())}")
    if c.size and c.max() > np.iinfo(np.int32).max:
        raise BopRunError(f"{where}: run length {int(c.max())} does not fit 32 bits")
    return c.astype(np.int32)


# ---------------------------------------------------------------------------------------------------- detections
def _key(scene_id, im_id):
    return f"{int(scene_id):06d}_{int(im_id):06d}"


def _by_image(dets, image_key):
    """`group_by_image_level` (utils/inout.py:109-123): {"scene_im": [det]} in order of first appearance."""
    out = {}
    for d in dets:
        out.setdefault(_key(d["scene_id"], d[image_key]), []).append(d)
    return out


def select_detections(dets, dataset_name, setting, targets=None):
    """`load_test_list_and_cnos_detections` + `generate_test_list` (utils/inout.py:370-492) with the caps of
    `GigaPoseTestSet.load_detections` (dataloader/test.py:110-114).  dets: the CNOS list; targets: the
    test_targets_bop*.json list (localization).  -> (test_list {key: [dict(scene_id, im_id, obj_id, inst_count)]},
    detections {key: [det]}).  Localization: per target, its object's detections of the image (all of the image's,
    relabelled, when it has none), by descending score (stable), at most 16 (32 for icbin); detection: every detection
    of each image, one target per object with its count.  The detections are deep copies of the input's."""
    per_image = _by_image(dets, "image_id")
    if setting == "detection":
        test_list = {}
        for key, im_dets in per_image.items():
            counts = {}
            for d in im_dets:
                counts[d["category_id"]] = counts.get(d["category_id"], 0) + 1
            s, im = (int(v) for v in key.split("_"))
            test_list[key] = [dict(scene_id=s, im_id=im, obj_id=o, inst_count=n) for o, n in counts.items()]
        return test_list, {k: copy.deepcopy(v) for k, v in per_image.items()}
    if setting != "localization":
        raise BopRunError(f"setting {setting!r} is neither 'localization' nor 'detection'")
    if targets is None:
        raise BopRunError("the localization setting needs the test targets")
    cap = CAP_PER_TARGET_ICBIN if dataset_name == "icbin" else CAP_PER_TARGET
    selected = []
    for t in targets:
        key = _key(t["scene_id"], t["im_id"])
        if key not in per_image:
            raise BopRunError(f"target image {key} (object {t['obj_id']}) has no detection")
        chosen = [d for d in per_image[key] if d["category_id"] == t["obj_id"]]
        if not chosen:                                   # MegaPose's fallback: every detection of the image
            chosen = copy.deepcopy(per_image[key])
            for d in chosen:
                d["category_id"] = t["obj_id"]
        chosen = sorted(chosen, key=lambda d: d["score"], reverse=True)[:cap]
        selected.extend(copy.deepcopy(chosen))
    return _by_image(targets, "im_id"), _by_image(selected, "image_id")


def xywh_to_xyxy(bbox):
    """CNOS xywh -> i64 xyxy as the reference's collate makes it: float32 x, y, x + w, y + h truncated toward zero
    (scene_dataset.py:337, bbox.py:6-22,116-130)."""
    b = np.asarray(bbox, np.float32).reshape(-1, 4)
    return np.stack([b[:, 0], b[:, 1], b[:, 0] + b[:, 2], b[:, 1] + b[:, 3]], 1).astype(np.int64)


def image_inputs(dets, targets, dataset_name, shape, key, target_size=224):
    """One image's host inputs: labels (object ids, LM-O indices for lmo), i64 xyxy boxes, concatenated i32 RLE counts
    and their offsets [n+1], the test list rows and the image's detection time (its first detection's).  A box whose
    crop has no rows or columns once resized to target_size (a mask more than target_size times longer than it is
    wide, or no pixel inside the image) is refused: the reference cannot crop it, and a crop of zeros would pass into
    retrieval unnoticed."""
    from .preprocess import empty_crops
    remap = (lambda o: LMO_ID_TO_INDEX[int(o)]) if "lmo" in dataset_name else int
    counts = [rle_counts(d["segmentation"], shape, f"image {key}, detection {i}") for i, d in enumerate(dets)]
    boxes = xywh_to_xyxy([d["bbox"] for d in dets])
    bad = empty_crops(boxes, shape[0], shape[1], target_size)
    if len(bad):
        i = int(bad[0])
        raise BopRunError(f"image {key}, detection {i}: bbox {list(dets[i]['bbox'])} (xyxy {boxes[i].tolist()}) has "
                          f"no rows or columns once resized to {target_size} x {target_size}; it cannot be cropped")
    return dict(labels=np.array([remap(d["category_id"]) for d in dets], np.int64),
                boxes=boxes,
                counts=np.concatenate(counts) if counts else np.zeros(0, np.int32),
                offsets=np.concatenate([[0], np.cumsum([len(c) for c in counts])]).astype(np.int64),
                obj_id=[remap(t["obj_id"]) for t in targets], inst_count=[int(t["inst_count"]) for t in targets],
                detection_time=float(dets[0].get("time", 0.0)))


# ---------------------------------------------------------------------------------------------------- model
_SAFE_BUILTINS = {"set", "frozenset", "slice", "range", "complex", "bytearray", "list", "dict", "tuple", "int", "float",
                  "bool", "str", "bytes", "object"}


class _Inert:
    """Stands in for a pickled class this process does not have (Hydra / omegaconf hyper-parameters): it takes any
    arguments and state and does nothing."""

    def __init__(self, *args, **kwargs):
        pass

    def __setstate__(self, state):
        self.__dict__["_state"] = state


class _Unpickler(pickle.Unpickler):
    """Resolves torch, numpy, collections and plain builtin types; every other class becomes an `_Inert` subclass of
    the same name, so unpickling runs no code from other modules."""

    def find_class(self, module, name):
        root = module.split(".")[0]
        if root in ("torch", "numpy", "collections", "_codecs") or (module == "builtins" and name in _SAFE_BUILTINS) \
                or (module == "copyreg" and name == "_reconstructor"):
            try:
                return super().find_class(module, name)
            except (ImportError, AttributeError):
                pass
        return type(name, (_Inert,), {"__module__": module})


_pickle = types.ModuleType("gigapose_b200_checkpoint_pickle")
_pickle.Unpickler = _Unpickler
_pickle.load = lambda f, **kw: _Unpickler(f, **kw).load()


def load_state_dict(path):
    """The `state_dict` of a Lightning checkpoint (tensors on the CPU); its other entries are unpickled inertly."""
    ckpt = torch.load(path, map_location="cpu", pickle_module=_pickle, weights_only=False)
    if not isinstance(ckpt, dict) or not isinstance(ckpt.get("state_dict"), dict):
        raise BopRunError(f"{path} has no state_dict (not a Lightning checkpoint)")
    return ckpt["state_dict"]


def load_checkpoint(model, path):
    """Loads a Lightning checkpoint's state_dict into `model` strictly; a missing or unexpected key is named."""
    state = load_state_dict(path)
    own = set(model.state_dict())
    missing, unexpected = sorted(own - set(state)), sorted(set(state) - own)
    if missing or unexpected:
        raise BopRunError(f"{path} does not fit the model: missing keys {missing}, unexpected keys {unexpected}")
    model.load_state_dict(state, strict=True)
    return model


def build_model(device, log_dir, checkpoint=None, seed=None):
    """The `GigaPose` of configs/model/large.yaml (DINOv2 ViT-L/14 descriptors, ResNet IST trunk, k = TOP_K), built in code
    as bench.build_models builds it.  With `checkpoint`, its state_dict is loaded strictly (a missing or unexpected
    key is named); `seed` seeds the initial weights (tests), otherwise they are the constructors' defaults."""
    from gigapose_b200.vit import DinoVisionTransformer
    from src.models.gigaPose import GigaPose
    from src.models.matching import LocalSimilarity
    from src.models.network.ae_net import AENet
    from src.models.network.ist_net import ISTNet, Regressor
    from src.models.network.resnet import ResNet

    vit = DinoVisionTransformer(init_seed=seed)
    ae = AENet("dinov2_vitl14", dinov2_model=vit, descriptor_size=1024, max_batch_size=64)
    if seed is not None:
        torch.manual_seed(seed + 1)
    backbone = ResNet(dict(n_heads=0, input_dim=3, input_size=256, initial_dim=128, block_dims=[128, 192, 256, 512],
                           descriptor_size=256))
    reg = Regressor(descriptor_size=256, hidden_dim=256, use_tanh_act=True, normalize_output=True)
    ist = ISTNet("resnet", backbone, reg, max_batch_size=64)
    metric = LocalSimilarity(k=TOP_K, sim_threshold=0.5, patch_threshold=3)
    model = GigaPose("large", ae, ist, training_loss=None, testing_metric=metric, optim_config=None, log_interval=1000,
                     log_dir=log_dir, max_num_dets_per_forward=None)
    if checkpoint is not None:
        load_checkpoint(model, checkpoint)
    return model.to(device).eval()


def object_ids(dataset_dir, dataset_name):
    """Object ids in the model's label order (label i is object_ids[i - 1]): the LM-O order for lmo, else 1 .. N."""
    _, mname = split_name(dataset_name)
    with open(os.path.join(dataset_dir, mname, "models_info.json")) as f:
        ids = sorted(int(k) for k in json.load(f))
    if "lmo" in dataset_name:
        if sorted(LMO_INDEX_TO_ID) != ids:
            raise BopRunError(f"lmo models_info.json lists objects {ids}, not {LMO_INDEX_TO_ID}")
        return list(LMO_INDEX_TO_ID)
    if ids != list(range(1, len(ids) + 1)):
        raise BopRunError(f"object ids {ids} are not 1 .. {len(ids)}: labels index the template bank")
    return ids


def read_meshes(dataset_dir, dataset_name):
    """The dataset's meshes (models/ or models_cad/) as `read_ply` dicts, in object_ids order."""
    from gigapose_b200.render import read_ply
    _, mname = split_name(dataset_name)
    return [read_ply(os.path.join(dataset_dir, mname, f"obj_{o:06d}.ply"))
            for o in object_ids(dataset_dir, dataset_name)]


def onboard(model, dataset_dir, template_poses, dataset_name=None, meshes=None):
    """`GigaPose.onboard_meshes` on the dataset's meshes (`read_meshes`, unless the caller already holds them) with the
    [T,4,4] template poses of INTEGRATION.md (an .npy path or an array)."""
    name = dataset_name or os.path.basename(os.path.normpath(dataset_dir))
    poses = np.load(template_poses) if isinstance(template_poses, (str, os.PathLike)) else np.asarray(template_poses)
    if poses.ndim != 3 or poses.shape[1:] != (4, 4):
        raise BopRunError(f"template poses must be [T,4,4], got {poses.shape}")
    meshes = read_meshes(dataset_dir, name) if meshes is None else meshes
    return model.onboard_meshes(name, meshes, torch.as_tensor(poses, dtype=torch.float32))


def onboard_static(model, dataset_dir, template_poses, dataset_name=None, frames=None):
    """`GigaPose.onboard_images` on the dataset's onboarding_static/ frames (`onboarding.read_onboarding_static`,
    unless the caller already holds them) for the [T,4,4] template poses (an .npy path or an array)."""
    from .onboarding import read_onboarding_static
    name = dataset_name or os.path.basename(os.path.normpath(dataset_dir))
    poses = np.load(template_poses) if isinstance(template_poses, (str, os.PathLike)) else np.asarray(template_poses)
    if poses.ndim != 3 or poses.shape[1:] != (4, 4):
        raise BopRunError(f"template poses must be [T,4,4], got {poses.shape}")
    frames = read_onboarding_static(dataset_dir) if frames is None else frames
    return model.onboard_images(name, [frames[o] for o in sorted(frames)], poses)


# ---------------------------------------------------------------------------------------------------- the loop
def depth_path(dataset_dir, split, scene_id, im_id):
    """The depth PNG `bop_eval.load_depth` reads."""
    return os.path.join(dataset_dir, split, f"{scene_id:06d}", "depth", f"{im_id:06d}.png")


def plan(dataset_dir, setting="localization", detections=None, dataset_name=None, depth=False):
    """Everything the loop needs from the host: dict(name, split, images [(scene, im)] in sorted order, test_list,
    detections, cameras {scene: {im: K}}, depth_scale {scene: {im: float}}).  With `depth`, every image's depth PNG must
    exist: a missing one is named here, before any GPU work."""
    name = dataset_name or os.path.basename(os.path.normpath(dataset_dir))
    split, _ = split_name(name)
    path = detections or default_detections(dataset_dir)
    with open(path) as f:
        dets = json.load(f)
    targets = None
    if setting == "localization":
        year = "24" if name == "hope" else "19"
        tpath = os.path.join(dataset_dir, f"test_targets_bop{year}.json")
        if not os.path.exists(tpath):
            raise BopRunError(f"{tpath} not found: the localization setting needs the test targets")
        with open(tpath) as f:
            targets = json.load(f)
    test_list, selected = select_detections(dets, name, setting, targets)
    images = sorted({tuple(int(v) for v in k.split("_")) for k in test_list})
    cams, scales = {}, {}
    for s in sorted({s for s, _ in images}):
        cam = load_cameras(dataset_dir, split, s)
        cams[s], scales[s] = cam["K"], cam["depth_scale"]
    for s, im in images:
        if im not in cams[s]:
            raise BopRunError(f"image {_key(s, im)} is not in scene_camera.json")
        if depth and not os.path.exists(depth_path(dataset_dir, split, s, im)):
            raise BopRunError(f"{depth_path(dataset_dir, split, s, im)} not found: depth refinement needs the depth "
                              f"image of every test image")
    return dict(name=name, split=split, images=images, test_list=test_list, detections=selected, cameras=cams,
                depth_scale=scales, dataset_dir=dataset_dir)


class _Prefetch:
    """Decodes image i + 1 on a background thread into one of two pinned buffers while image i runs; with `depths`
    ((dataset_dir, split, scene, im, depth_scale) per image, the arguments of `bop_eval.load_depth`), its depth image
    too, as f32 in the model unit.  `get(i)` -> (rgb, depth or None)."""

    def __init__(self, paths, depths=None):
        self.paths, self.depths = paths, depths
        self.pool, self.bufs = concurrent.futures.ThreadPoolExecutor(1), {}
        self.next = self.pool.submit(self._load, 0) if paths else None

    def _pinned(self, i, a, dtype):
        key = (i % 2, a.shape, dtype)
        buf = self.bufs.get(key)
        if buf is None:
            buf = self.bufs[key] = torch.empty(a.shape, dtype=dtype, pin_memory=True)
        buf.numpy()[...] = a
        return buf

    def _load(self, i):
        rgb = self._pinned(i, read_image(self.paths[i]), torch.uint8)
        return rgb, None if self.depths is None else self._pinned(i, load_depth(*self.depths[i]), torch.float32)

    def get(self, i):
        bufs = self.next.result()
        self.next = self.pool.submit(self._load, i + 1) if i + 1 < len(self.paths) else None
        return bufs

    def close(self):
        self.pool.shutdown(wait=True)


def image_batch(p, i, rgb, device):
    """Step i's batch for `eval_retrieval`: the RLE crop of the image's detections on the device plus the infos and
    test list the reference's collate builds (dataloader/test.py:167-205, 283-293)."""
    import pandas as pd
    import src.megapose.utils.tensor_collection as tc
    from .preprocess import crop_detections_rle
    s, im = p["images"][i]
    key = _key(s, im)
    x = image_inputs(p["detections"][key], p["test_list"][key], p["name"], tuple(rgb.shape[:2]), key)
    n = len(x["labels"])
    crop = crop_detections_rle(rgb.to(device, non_blocking=True)[None], x["counts"], x["offsets"], x["boxes"],
                               np.zeros(n, np.int64))
    K = torch.as_tensor(p["cameras"][s][im], dtype=torch.float64).float().to(device).expand(n, 3, 3).contiguous()
    infos = pd.DataFrame(dict(label=[str(v) for v in x["labels"]], scene_id=[s] * n, view_id=[im] * n,
                              batch_im_id=np.zeros(n, np.int64)))
    batch = tc.PandasTensorCollection(infos=infos, tar_img=crop["tar_img"], tar_mask=crop["tar_mask"], tar_K=K,
                                      tar_M=crop["tar_M"])
    batch.test_list = tc.PandasTensorCollection(infos=pd.DataFrame(dict(
        im_id=[im] * len(x["obj_id"]), scene_id=[s] * len(x["obj_id"]), obj_id=x["obj_id"],
        inst_count=x["inst_count"], detection_time=[x["detection_time"]] * len(x["obj_id"]))))
    batch.rle = (x["counts"], x["offsets"])
    return batch


def select_rle(rle, selected):
    """The (counts, offsets) of the detections `selected` (indices into the image's detections), in that order."""
    counts, off = rle
    parts = [counts[off[i]:off[i + 1]] for i in selected]
    return (np.concatenate(parts) if parts else np.zeros(0, np.int32),
            np.concatenate([[0], np.cumsum([len(c) for c in parts])]).astype(np.int64))


@torch.no_grad()
def refine_image(model, p, i, kept, depth, hypotheses, out_dir, masks=None, refiner="icp"):
    """Row f10 for image i of the plan: the first `hypotheses` poses of each of the `kept` instances (the collection
    `eval_retrieval` returns after its filter, with `time` and `detection_time`) go through
    `GigaPose.refine_depth(rank=True)` against `depth` (f32 [H,W] in the model unit, host or device), and
    out_dir/refined_predictions/{i}.npz takes, per instance, the pose of its best hypothesis, that hypothesis' coarse
    score, the dataset's object id, `time` = the image's coarse time (detection + retrieval) and `refinement_time`,
    measured with CUDA events from the depth upload to the end of the scoring, plus `hypothesis` (the index chosen) and
    its `icp_status`, which the csv writer does not read.  With `masks` = (counts, offsets), the run-length masks of
    the kept instances in their order, they refine with `mask_normals=True`; `refinement_time` then covers the mask
    decode.  With `refiner="teaserpp"` the hypotheses go through the TEASER++ refiner (row f13) and the npz holds
    `teaser_status` in place of `icp_status`.  -> the refined collection."""
    s, im = p["images"][i]
    device = kept.pred_poses.device
    n = len(kept)
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    depth = torch.as_tensor(depth).to(device, non_blocking=True)
    K = torch.as_tensor(p["cameras"][s][im], dtype=torch.float64).float()
    extra = {} if masks is None else dict(masks=dict(counts=masks[0], offsets=masks[1]), mask_normals=True)
    refined = model.refine_depth(p["name"], kept, depth[None], frame_idx=np.zeros(n, np.int64), hypotheses=hypotheses,
                                 K=K, rank=True, refiner=refiner, **extra)
    rows = torch.arange(n, device=device)
    poses = refined.pred_poses[rows, refined.best_hypothesis]
    scores = kept.scores[rows, refined.best_hypothesis]
    status_key = REFINERS[refiner].outputs[0]
    status = getattr(refined, status_key)[rows, refined.best_hypothesis]
    stop.record()
    stop.synchronize()
    labels = np.asarray(kept.infos.label).astype(np.int32)
    if "lmo" in p["name"]:
        labels = np.asarray(LMO_INDEX_TO_ID, np.int32)[labels - 1]
    coarse_time = (kept.time + kept.detection_time).cpu().numpy()
    os.makedirs(os.path.join(out_dir, "refined_predictions"), exist_ok=True)
    np.savez(os.path.join(out_dir, "refined_predictions", f"{i}.npz"),
             scene_id=np.asarray(kept.infos.scene_id).astype(np.int32),
             im_id=np.asarray(kept.infos.view_id).astype(np.int32), object_id=labels, time=coarse_time,
             refinement_time=np.full(n, start.elapsed_time(stop) / 1e3), poses=poses.cpu().numpy(),
             scores=scores.cpu().numpy(), hypothesis=refined.best_hypothesis.cpu().numpy(),
             **{status_key: status.cpu().numpy()})
    return refined


def check_refine(model, refine_hypotheses, refine_masks, depth_refiner):
    """-> H after checking the refinement options against the model's k."""
    H = int(refine_hypotheses)
    if not 0 <= H <= model.testing_metric.k:
        raise BopRunError(f"refine_hypotheses {H} outside [0, {model.testing_metric.k}]")
    if refine_masks and not H:
        raise BopRunError("refine_masks needs refine_hypotheses >= 1")
    if depth_refiner not in REFINERS:
        raise BopRunError(f"depth_refiner must be {' or '.join(map(repr, REFINERS))}, got {depth_refiner!r}")
    if refine_masks and not REFINERS[depth_refiner].masks:
        raise BopRunError(f"the {depth_refiner} depth refiner takes no masks (refine_masks)")
    return H


def check_out(out_dir):
    """Creates out_dir/predictions and refuses an out_dir whose prediction directories already hold .npz files."""
    pred_dir, ref_dir = os.path.join(out_dir, "predictions"), os.path.join(out_dir, "refined_predictions")
    os.makedirs(pred_dir, exist_ok=True)
    for d in (pred_dir, ref_dir):
        if glob.glob(os.path.join(glob.escape(d), "*.npz")):
            raise BopRunError(f"{d} already holds prediction files; use an empty --out")


def check_onboarding(onboarding, H, reconstruct=False):
    if onboarding not in ("models", "static"):
        raise BopRunError(f"onboarding must be 'models' or 'static', got {onboarding!r}")
    if reconstruct and onboarding != "static":
        raise BopRunError(RECONSTRUCT_NEEDS_STATIC)
    if reconstruct and not H:
        raise BopRunError(RECONSTRUCT_NEEDS_DEPTH)
    if onboarding == "static" and H and not reconstruct:
        raise BopRunError(STATIC_NO_DEPTH)


STATIC_NO_DEPTH = ("--onboarding static takes no --refine-depth: the depth refiners render the CAD model, which "
                   "model-free onboarding does not read")
RECONSTRUCT_NEEDS_STATIC = "--reconstruct needs --onboarding static: it builds the meshes of model-free objects"
RECONSTRUCT_NEEDS_DEPTH = "--reconstruct needs --refine-depth H: only the depth refiners use the reconstructed meshes"


def reconstruct_meshes(frames, out_dir=None):
    """Row f17: `reconstruct.reconstruct` of every object of {obj_id: Frames} (with depth), in object order; with
    `out_dir`, each mesh is also written to out_dir/reconstructed/obj_{id:06d}.ply."""
    from .reconstruct import reconstruct
    from .render import write_ply
    meshes = []
    for o in sorted(frames):
        try:
            meshes.append(reconstruct(frames[o]))
        except Exception as e:
            e.add_note(f"while reconstructing object {o}")
            raise
        if out_dir is not None:
            os.makedirs(os.path.join(out_dir, "reconstructed"), exist_ok=True)
            write_ply(os.path.join(out_dir, "reconstructed", f"obj_{o:06d}.ply"), meshes[-1])
    return meshes


def prepare(model, dataset_dir, p, template_poses=None, template_level=1, pose_distribution="all", attach=False,
            onboarding="models", mesh_dir=None):
    """Onboards the plan's dataset unless the model already holds it, from `template_poses` or, when that is None,
    from the generated `template_poses.template_poses(template_level, pose_distribution)`; from the CAD models, or
    with onboarding="static" from the onboarding_static/ frames (`onboard_static`).  With `attach` (depth
    refinement), attaches its meshes too: the CAD models, or with onboarding="static" the meshes reconstructed from
    the onboarding depth (`reconstruct_meshes`, written under `mesh_dir` when it is given)."""
    name = p["name"]
    if onboarding == "static":
        attach = attach and name not in getattr(model, "meshes", {})
        frames = None
        if attach or name not in model.engines:
            from .onboarding import read_onboarding_static
            frames = read_onboarding_static(dataset_dir, depth=attach)
        if name not in model.engines:
            if template_poses is None:
                from .template_poses import template_poses as generate
                template_poses = generate(template_level, pose_distribution)
            onboard_static(model, dataset_dir, template_poses, name, frames)
        if attach:
            model.attach_meshes(name, reconstruct_meshes(frames, mesh_dir))
        return
    attach = attach and name not in getattr(model, "meshes", {})
    meshes = read_meshes(dataset_dir, name) if attach or name not in model.engines else None
    if name not in model.engines:
        if template_poses is None:
            from .template_poses import template_poses as generate
            template_poses = generate(template_level, pose_distribution)
        onboard(model, dataset_dir, template_poses, name, meshes)
    if attach:
        model.attach_meshes(name, meshes)


def run_images(model, p, indices, out_dir, H=0, refine_masks=False, depth_refiner="icp", vis_every=0):
    """`eval_retrieval` (and, with H, `refine_image`) on the plan's images `indices`, each written under its index in
    the plan, so that runs over disjoint shares of the images fill one out_dir.  An exception names its image in a
    note."""
    name = p["name"]
    model.log_dir = out_dir
    device = model.engines[name].device
    images = [p["images"][i] for i in indices]
    pre = _Prefetch([image_path(p["dataset_dir"], p["split"], s, im) for s, im in images],
                    [(p["dataset_dir"], p["split"], s, im, p["depth_scale"][s][im]) for s, im in images] if H else None)
    try:
        for n, i in enumerate(indices):
            try:
                rgb, depth = pre.get(n)
                batch = image_batch(p, i, rgb, device)
                selected, kept = model.eval_retrieval(batch, idx_batch=i, dataset_name=name)
                if vis_every and i % vis_every == 0 and len(selected):
                    from torchvision.utils import save_image
                    save_image(model.vis_retrieval(name, batch, kept, selected),
                               os.path.join(out_dir, f"retrieved_sample_{i}.png"), nrow=len(selected))
                if H:
                    refine_image(model, p, i, kept, depth, H, out_dir,
                                 select_rle(batch.rle, selected) if refine_masks else None, depth_refiner)
            except Exception as e:
                e.add_note(f"while running image {i} (scene {images[n][0]}, image {images[n][1]})")
                raise
    finally:
        pre.close()


def write_csvs(model, name, out_dir, run_id="bop_run", H=0, refine_masks=False, depth_refiner="icp"):
    """The csv(s) of the predictions under out_dir (see `run`)."""
    from src.utils.inout import save_predictions_from_batched_predictions
    pred_dir, ref_dir = os.path.join(out_dir, "predictions"), os.path.join(out_dir, "refined_predictions")
    stem = f"{model.model_name}-pbrreal-rgb-mmodel_{name}-test_{run_id}"
    save_predictions_from_batched_predictions(pred_dir, dataset_name=name, model_name=model.model_name,
                                              run_id=run_id, is_refined=False)
    coarse = os.path.join(pred_dir, f"{stem}.csv")
    if not H:
        return coarse
    suffix = f"_{depth_refiner}_masked" if refine_masks else f"_{depth_refiner}"
    save_predictions_from_batched_predictions(ref_dir, dataset_name=name, model_name=model.model_name,
                                              run_id=f"{run_id}{suffix}", is_refined=True)
    return coarse, os.path.join(ref_dir, f"{stem}{suffix}.csv")


def default_run_id(onboarding="models"):
    return "bop_run_static" if onboarding == "static" else "bop_run"


@torch.no_grad()
def run(model, dataset_dir, out_dir, setting="localization", detections=None, template_poses=None, run_id=None,
        dataset_name=None, refine_hypotheses=0, refine_masks=False, depth_refiner="icp", vis_every=0,
        template_level=1, pose_distribution="all", onboarding="models", reconstruct=False):
    """Runs the test split: onboards the dataset unless the model already holds it, from `template_poses` ([T,4,4]
    array or .npy path) or, when that is None, from the generated icosphere poses of `template_level` and
    `pose_distribution` (`template_poses.template_poses`, the reference's test templates by default), then one
    `eval_retrieval` per image (predictions under out_dir/predictions, which must hold no .npz yet) and the csv.
    -> path of the csv (`{model}-pbrreal-rgb-mmodel_{dataset}-test_{run_id}.csv` in out_dir/predictions).
    With `refine_hypotheses` = H in 1 .. k, each image's kept instances also go through `refine_image` with the image's
    depth PNG, and a second csv (`..._{run_id}_icp.csv` in out_dir/refined_predictions) is written
    -> (coarse csv, refined csv).  With `refine_masks` they refine with their own CNOS masks (`refine_image`'s masks)
    and the second csv is `..._{run_id}_icp_masked.csv`.  With `depth_refiner="teaserpp"` (row f13) they go through
    the TEASER++ refiner instead and the second csv is `..._{run_id}_teaserpp.csv`; it takes no masks.
    With `vis_every` = N > 0 (row f14) every N-th image's retrieval panels (`GigaPose.vis_retrieval`) are written to
    out_dir/retrieved_sample_{i}.png, one row per rank and one column per kept detection, as the reference does.
    With onboarding="static" (row f16) the templates come from the onboarding_static/ frames instead of the CAD
    models (`onboard_static`), refinement is refused, and the default run_id is "bop_run_static" ("bop_run"
    otherwise).  With onboarding="static" and `reconstruct` (row f17), refinement is allowed: each object's mesh is
    reconstructed from its onboarding depth images, written to out_dir/reconstructed/obj_{id:06d}.ply and attached."""
    H = check_refine(model, refine_hypotheses, refine_masks, depth_refiner)
    check_onboarding(onboarding, H, reconstruct)
    run_id = run_id or default_run_id(onboarding)
    p = plan(dataset_dir, setting, detections, dataset_name, depth=H > 0)
    check_out(out_dir)
    prepare(model, dataset_dir, p, template_poses, template_level, pose_distribution, attach=H > 0,
            onboarding=onboarding, mesh_dir=out_dir)
    run_images(model, p, range(len(p["images"])), out_dir, H, refine_masks, depth_refiner, vis_every)
    return write_csvs(model, p["name"], out_dir, run_id, H, refine_masks, depth_refiner)


# ---------------------------------------------------------------------------------------------------- several ranks
def shard_images(counts, world_size):
    """Image indices per rank: greedy longest-first on the images' detection `counts` (the largest first, ties by image
    index, each to the rank with the fewest detections so far, ties by rank), each share in image order.  No rank
    ends more than the largest single count above the mean per rank."""
    loads, shares = [0] * world_size, [[] for _ in range(world_size)]
    for i in sorted(range(len(counts)), key=lambda i: (-counts[i], i)):
        r = min(range(world_size), key=lambda r: (loads[r], r))
        shares[r].append(i)
        loads[r] += counts[i]
    return [sorted(s) for s in shares]


class RankFailed(RuntimeError):
    pass


class Ranks:
    """The ranks of a `torchrun` launch on a gloo process group (env://).  `step(fn)` runs fn on this rank, then every
    rank learns whether any rank raised: if one did, each raises `RankFailed` naming every failing rank and its error,
    so no rank waits for one that has given up.  Each rank calls the same steps in the same order."""

    def __init__(self):
        import torch.distributed as dist
        self.dist = dist
        dist.init_process_group("gloo")
        self.rank, self.world_size = dist.get_rank(), dist.get_world_size()

    def step(self, fn, *args):
        out, err = None, None
        try:
            out = fn(*args)
        except Exception as e:
            err = "".join([f"rank {self.rank}: {type(e).__name__}: {e}"] +
                          [f"\n  {note}" for note in getattr(e, "__notes__", ())])
        errors = [None] * self.world_size
        self.dist.all_gather_object(errors, err)
        failed = [e for e in errors if e is not None]
        if failed:
            raise RankFailed("\n".join(failed))
        return out

    def close(self):
        self.dist.destroy_process_group()


def _evaluate(csv, dataset_dir, setting, out_dir, device):
    from . import bop_eval
    split, _ = split_name(os.path.basename(os.path.normpath(dataset_dir)))
    if setting == "localization":
        res = bop_eval.evaluate(csv, dataset_dir, split, out_dir=out_dir, device=device)
        print(json.dumps({k: res[k] for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd", "n_targets")}))
    else:
        res = bop_eval.evaluate_detection(csv, dataset_dir, split, out_dir=out_dir, device=device)
        print(json.dumps({k: res[k] for k in ("map", "map_mssd", "map_mspd")}))


def parser():
    ap = argparse.ArgumentParser(description="GigaPose on a BOP test split with its CNOS detections -> BOP results csv")
    ap.add_argument("--dataset-dir", required=True, help="BOP dataset directory, e.g. <root>/lmo")
    ap.add_argument("--checkpoint", required=True, help="Lightning checkpoint (gigaPose_v1.ckpt)")
    ap.add_argument("--template-poses", default=None,
                    help="[T,4,4] .npy of template poses (see INTEGRATION.md); default: generated from --template-level "
                         "and --pose-distribution")
    ap.add_argument("--template-level", type=int, choices=(0, 1, 2), default=None,
                    help="icosphere level of the generated template poses: 42, 162 or 642 views (default 1)")
    ap.add_argument("--pose-distribution", choices=("all", "upper"), default=None,
                    help="generated template poses: every view, or those whose camera has z >= 0 (default all)")
    ap.add_argument("--setting", choices=("localization", "detection"), default="localization")
    ap.add_argument("--detections", default=None, help="CNOS detections json (default: <root>/default_detections/...)")
    ap.add_argument("--out", default="bop_run_out")
    ap.add_argument("--refine-depth", type=int, default=0, choices=range(TOP_K + 1), metavar="H",
                    help=f"refine the first H (1..{TOP_K}) hypotheses of every kept instance against the depth images "
                         f"and write a second csv with the best one (0: no refinement)")
    ap.add_argument("--refine-masks", action="store_true",
                    help="with --refine-depth: refine each instance with its own CNOS mask, target normals smoothed "
                         "within it (writes ..._icp_masked.csv)")
    ap.add_argument("--depth-refiner", choices=tuple(REFINERS), default="icp",
                    help="with --refine-depth: the point-to-plane ICP (..._icp.csv) or MegaPose's TEASER++ refiner "
                         "(..._teaserpp.csv, no masks)")
    ap.add_argument("--vis-every", type=int, default=0, metavar="N",
                    help="write the retrieval panels of every N-th image to <out>/retrieved_sample_<i>.png (0: none)")
    ap.add_argument("--onboarding", choices=("models", "static"), default="models",
                    help="build the templates from the CAD models (models/) or, for objects without them, from the "
                         "onboarding_static/ frames (model-free; --refine-depth only with --reconstruct; run id "
                         "bop_run_static)")
    ap.add_argument("--reconstruct", action="store_true",
                    help="with --onboarding static and --refine-depth: reconstruct each object from its onboarding "
                         "depth images (<out>/reconstructed/obj_<id>.ply) and refine against that mesh")
    ap.add_argument("--evaluate", action="store_true", help="score the csv (both, coarse first, when refining) with bop_eval")
    ap.add_argument("--device", default="cuda")
    return ap


def main(argv=None):
    a = parser().parse_args(argv)
    if a.refine_masks and not a.refine_depth:
        parser().error("--refine-masks needs --refine-depth H")
    if a.refine_masks and not REFINERS[a.depth_refiner].masks:
        parser().error(f"--depth-refiner {a.depth_refiner} takes no --refine-masks")
    if a.template_poses is not None and (a.template_level is not None or a.pose_distribution is not None):
        parser().error("--template-level and --pose-distribution choose generated template poses; "
                       "they do not go with --template-poses")
    if a.reconstruct and a.onboarding != "static":
        parser().error(RECONSTRUCT_NEEDS_STATIC)
    if a.reconstruct and not a.refine_depth:
        parser().error(RECONSTRUCT_NEEDS_DEPTH)
    if a.onboarding == "static" and a.refine_depth and not a.reconstruct:
        parser().error(STATIC_NO_DEPTH)
    a.template_level = 1 if a.template_level is None else a.template_level
    a.pose_distribution = a.pose_distribution or "all"
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        return main_ranks(a)
    model = build_model(a.device, a.out, checkpoint=a.checkpoint)
    csvs = run(model, a.dataset_dir, a.out, a.setting, a.detections, a.template_poses, refine_hypotheses=a.refine_depth,
               refine_masks=a.refine_masks, depth_refiner=a.depth_refiner, vis_every=a.vis_every,
               template_level=a.template_level, pose_distribution=a.pose_distribution, onboarding=a.onboarding,
               reconstruct=a.reconstruct)
    report(a, csvs, a.device)


def report(a, csvs, device):
    csvs = (csvs,) if isinstance(csvs, str) else csvs
    for csv, out in zip(csvs, (a.out, os.path.join(a.out, "refined"))):
        print(csv)
        if a.evaluate:
            _evaluate(csv, a.dataset_dir, a.setting, out, device)


@torch.no_grad()
def main_ranks(a):
    """`main` under torchrun: every rank builds the model on cuda:LOCAL_RANK (or on --device when it names a device
    index, so that several ranks can share one GPU), onboards the dataset itself and runs its `shard_images` share of
    the plan's images into the same --out; rank 0 checks --out first and writes the csv(s) and scores last (and, with
    --reconstruct, the meshes, which every rank reconstructs alike: the kernels are deterministic).  A rank that
    fails makes every rank exit with its error (`Ranks.step`)."""
    ranks = Ranks()
    try:
        device = torch.device(f"cuda:{os.environ.get('LOCAL_RANK', '0')}" if a.device == "cuda" else a.device)
        if device.type == "cuda":
            torch.cuda.set_device(device)
        ranks.step(lambda: ranks.rank == 0 and check_out(a.out))

        def work():
            model = build_model(device, a.out, checkpoint=a.checkpoint)
            H = check_refine(model, a.refine_depth, a.refine_masks, a.depth_refiner)
            p = plan(a.dataset_dir, a.setting, a.detections, depth=H > 0)
            prepare(model, a.dataset_dir, p, a.template_poses, a.template_level, a.pose_distribution, attach=H > 0,
                    onboarding=a.onboarding, mesh_dir=a.out if ranks.rank == 0 else None)
            counts = [len(p["detections"][_key(s, im)]) for s, im in p["images"]]
            share = shard_images(counts, ranks.world_size)[ranks.rank]
            run_images(model, p, share, a.out, H, a.refine_masks, a.depth_refiner, a.vis_every)
            return model, p["name"], H

        model, name, H = ranks.step(work)
        ranks.step(lambda: ranks.rank == 0 and report(
            a, write_csvs(model, name, a.out, default_run_id(a.onboarding), H, a.refine_masks, a.depth_refiner), device))
    finally:
        ranks.close()


if __name__ == "__main__":
    main()
