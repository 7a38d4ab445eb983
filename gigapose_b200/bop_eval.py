"""BOP 2019 pose-error evaluation on the GPU (row f7): VSD, MSSD, MSPD and the average recalls, in place of the external
BOP toolkit's eval_bop19_pose.py that the reference shells out to (src/scripts/eval_bop.py:16-38).

Estimates and ground truths are rendered with `gp_render_depth` (one depth sample at each pixel centre), the per-pixel
VSD counts and the symmetry-aware vertex distances run in csrc/bop_eval.cu (whose header comment states the fp32
contract), and the matching into recalls runs here in numpy.

Row f8 scores the BOP 2024 6D-detection task (`evaluate_detection`): MSSD and MSPD of every kept estimate against every
ground truth of its object in its image, then the greedy matching with ignored ground truths and the COCO average
precision, all on the device (gp_bop_mssd_mspd, gp_bop_match, gp_bop_average_precision).  No depth images are read.

Row f12 scores the BOP 2019 targets with ADD, ADD-S and the 2D-projection error (`evaluate_add`): the errors on the
device (gp_bop_add), then minimum-error matching, the recalls at 0.1 d and 5 px and PoseCNN's AUC here in numpy.
Usage:

    python -m gigapose_b200.bop_eval --results X.csv --dataset-dir D [--split test] [--out DIR]
    python -m gigapose_b200.bop_eval --task detection --results X.csv --dataset-dir D [--split test] [--out DIR]
    python -m gigapose_b200.bop_eval --task add --results X.csv --dataset-dir D [--split test] [--out DIR]
"""
from __future__ import annotations

import argparse
import contextlib
import ctypes as C
import json
import os

import numpy as np
import torch

from . import _lib
from ._lib import check
from .render import read_ply

# Defaults of the BOP 2019/2020 methodology: VSD from Hodan et al., "BOP: Benchmark for 6D Object Pose Estimation"
# (ECCV 2018); MSSD, MSPD and the AR from Hodan et al., "BOP Challenge 2020 on 6D Object Localization" (ECCV 2020
# workshops).  They are taken from those papers; they could not be checked against the toolkit's own configuration.
DELTA = 15.0                    # VSD visibility tolerance, model unit (mm)
DELTA_ITODD = 5.0
TAUS = tuple(round(0.05 * i, 2) for i in range(1, 11))          # VSD misalignment tolerance, x diameter
THETA_VSD = TAUS                                                 # VSD correctness thresholds
THETA_MSSD = TAUS                                                # x diameter
THETA_MSPD = tuple(5.0 * i for i in range(1, 11))                # x r, r = image width / 640
MAX_SYM_DISC_STEP = 0.01        # continuous symmetries: the farthest vertex moves <= 1 % of the diameter per step
VISIB_GT_MIN = 0.1              # ground truths less visible than this are neither targets nor matchable
Z_NEAR = 10.0                   # renders: near plane, model unit
WORKSPACE_BYTES = 1 << 30       # device memory per chunk of images: measured depth, renders and the render keys
MAX_PAIRS_PER_CALL = 1 << 18    # pairs per gp_bop_mssd_mspd / gp_bop_add call: ~140 B of poses, indices and errors each


class BopEvalError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------- readers
def _json(path):
    if not os.path.exists(path):
        raise BopEvalError(f"{path} not found")
    with open(path) as f:
        return json.load(f)


def load_scene(dataset_dir, split, scene_id):
    """-> dict(gt={im: [dict(R [3,3], t [3], obj_id)]}, visib={im: [visib_fract]}, K={im: [3,3]},
    depth_scale={im: float}) from scene_gt.json, scene_gt_info.json and scene_camera.json."""
    d = os.path.join(dataset_dir, split, f"{scene_id:06d}")
    gt = _json(os.path.join(d, "scene_gt.json"))
    info = _json(os.path.join(d, "scene_gt_info.json"))
    out = dict(gt={}, visib={}, **load_cameras(dataset_dir, split, scene_id))
    for im, insts in gt.items():
        out["gt"][int(im)] = [dict(R=np.asarray(g["cam_R_m2c"], np.float64).reshape(3, 3),
                                   t=np.asarray(g["cam_t_m2c"], np.float64).reshape(3), obj_id=int(g["obj_id"]))
                              for g in insts]
        out["visib"][int(im)] = [float(i["visib_fract"]) for i in info[im]]
    return out


def load_cameras(dataset_dir, split, scene_id):
    """-> dict(K={im: [3,3]}, depth_scale={im: float}) from a scene's scene_camera.json (test splits without ground
    truth, such as those of hb and itodd, have this file only)."""
    cam = _json(os.path.join(dataset_dir, split, f"{scene_id:06d}", "scene_camera.json"))
    out = dict(K={}, depth_scale={})
    for im, c in cam.items():
        out["K"][int(im)] = np.asarray(c["cam_K"], np.float64).reshape(3, 3)
        out["depth_scale"][int(im)] = float(c.get("depth_scale", 1.0))
    return out


def load_depth(dataset_dir, split, scene_id, im_id, depth_scale):
    """16-bit PNG depth x depth_scale -> f32 [H,W] in the model unit (0 = missing)."""
    from PIL import Image
    path = os.path.join(dataset_dir, split, f"{scene_id:06d}", "depth", f"{im_id:06d}.png")
    if not os.path.exists(path):
        raise BopEvalError(f"{path} not found: VSD needs the depth images, and this dataset or split has none")
    with Image.open(path) as im:
        raw = np.asarray(im)
    return (raw.astype(np.float64) * depth_scale).astype(np.float32)


def models_dir(dataset_dir):
    """models_eval/ (the evaluation models of a BOP dataset) when present, else models/."""
    d = os.path.join(dataset_dir, "models_eval")
    return d if os.path.isdir(d) else os.path.join(dataset_dir, "models")


def load_models_info(mdir):
    """-> {obj_id: dict(diameter, symmetries_discrete [k,4,4], symmetries_continuous [(axis [3], offset [3])])}."""
    info = _json(os.path.join(mdir, "models_info.json"))
    out = {}
    for k, v in info.items():
        out[int(k)] = dict(diameter=float(v["diameter"]),
                           symmetries_discrete=[np.asarray(s, np.float64).reshape(4, 4)
                                                for s in v.get("symmetries_discrete", [])],
                           symmetries_continuous=[(np.asarray(s["axis"], np.float64), np.asarray(s["offset"], np.float64))
                                                  for s in v.get("symmetries_continuous", [])])
    return out


def load_targets(dataset_dir, name="test_targets_bop19.json"):
    """-> list of dict(scene_id, im_id, obj_id, inst_count)."""
    return [dict(scene_id=int(t["scene_id"]), im_id=int(t["im_id"]), obj_id=int(t["obj_id"]),
                 inst_count=int(t["inst_count"])) for t in _json(os.path.join(dataset_dir, name))]


def load_results(results):
    """A csv path (`src.utils.inout.load_bop_results`) or a list of dicts in that format."""
    if isinstance(results, (str, os.PathLike)):
        from src.utils.inout import load_bop_results
        return load_bop_results(results)
    return list(results)


# ---------------------------------------------------------------------------------------------------- symmetries
def _axis_rotation(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * k + (1 - np.cos(angle)) * (k @ k)


def symmetry_transforms(info, max_sym_disc_step=MAX_SYM_DISC_STEP):
    """Symmetry transforms [S,4,4] (fp64) of an object.  Discrete: the identity, then each declared discrete symmetry D.
    Continuous: each (axis a, offset o) becomes n = ceil(pi / max_sym_disc_step) rotations C_k by k * 2 pi / n,
    k = 0 .. n - 1, about the line through o along a (x -> R_k (x - o) + o), so that the vertex farthest from the axis
    (at most half a diameter away) moves at most max_sym_disc_step x diameter between two steps.  With continuous
    symmetries the transforms are the compositions C_k D (D applied first), discrete-major: for each D in the order
    above, every C_k of the first continuous symmetry, then of the next."""
    disc = [np.eye(4)] + [np.asarray(s, np.float64).reshape(4, 4) for s in info.get("symmetries_discrete", [])]
    cont = []
    for axis, offset in info.get("symmetries_continuous", []):
        n = int(np.ceil(np.pi / max_sym_disc_step))
        o = np.asarray(offset, np.float64).reshape(3)
        for k in range(n):
            T = np.eye(4)
            T[:3, :3] = _axis_rotation(axis, k * 2.0 * np.pi / n)
            T[:3, 3] = o - T[:3, :3] @ o
            cont.append(T)
    if not cont:
        return np.stack(disc)
    return np.stack([c @ d for d in disc for c in cont])


# ---------------------------------------------------------------------------------------------------- matching
def match_group(err, valid, thresholds):
    """Greedy matching of one (image, object): err [n_est, n_gt] with the estimates in descending score order, valid
    [n_gt] (matchable ground truths), thresholds [T] -> matched ground truths per threshold [T].  Each estimate in turn
    takes the unmatched valid ground truth with the smallest error strictly below the threshold (the lowest index on a
    tie)."""
    err = np.asarray(err, np.float64).reshape(-1, len(valid))
    th = np.asarray(thresholds, np.float64)
    taken = np.zeros((len(th), err.shape[1]), bool)
    for row in err:
        cand = valid[None] & ~taken & (row[None] < th[:, None])
        j = np.argmin(np.where(cand, row[None], np.inf), axis=1)
        has = cand.any(1)
        taken[np.nonzero(has)[0], j[has]] = True
    return taken.sum(1)


def recalls(groups, n_targets, taus=TAUS, theta_vsd=THETA_VSD, theta_mssd=THETA_MSSD, theta_mspd=THETA_MSPD, r=1.0):
    """groups: list of dict(vsd [n_est,n_gt,n_tau], mssd / mspd [n_est,n_gt], valid [n_gt], diameter) -> recall
    arrays: vsd [n_tau, n_theta], mssd [n_theta], mspd [n_theta] (matched targets / n_targets)."""
    m_vsd = np.zeros((len(taus), len(theta_vsd)))
    m_mssd, m_mspd = np.zeros(len(theta_mssd)), np.zeros(len(theta_mspd))
    for g in groups:
        if g["mssd"].shape[0] == 0:
            continue
        for t in range(len(taus)):
            m_vsd[t] += match_group(g["vsd"][:, :, t], g["valid"], theta_vsd)
        m_mssd += match_group(g["mssd"], g["valid"], np.asarray(theta_mssd) * g["diameter"])
        m_mspd += match_group(g["mspd"], g["valid"], np.asarray(theta_mspd) * r)
    n = max(n_targets, 1)
    return dict(vsd=m_vsd / n, mssd=m_mssd / n, mspd=m_mspd / n)


# ---------------------------------------------------------------------------------------------------- set-up
def _scene(scenes, dataset_dir, split, scene_id, im_id):
    """scenes[scene_id] (a `load_scene` dict), loaded on first use; refuses a target image that the scene's
    scene_gt.json or scene_camera.json lacks."""
    if scene_id not in scenes:
        scenes[scene_id] = load_scene(dataset_dir, split, scene_id)
    sc = scenes[scene_id]
    if im_id not in sc["gt"] or im_id not in sc["K"]:
        raise BopEvalError(f"target image {scene_id}/{im_id} is not in scene_gt.json / scene_camera.json")
    return sc


def prepare(results, dataset_dir, split="test", targets_name="test_targets_bop19.json"):
    """Host side: reads the dataset, keeps the top inst_count estimates per target by score and lists every
    (estimate, ground truth) pair of the same object in an image.  -> dict with `images` [(scene, im)], `targets`,
    per-image estimates / ground truths and `pairs`."""
    results = load_results(results)
    targets = load_targets(dataset_dir, targets_name)
    mdir = models_dir(dataset_dir)
    info = load_models_info(mdir)
    if not targets:
        raise BopEvalError(f"{os.path.join(dataset_dir, targets_name)} lists no targets")
    by_key = {}
    for i, res in enumerate(results):
        by_key.setdefault((res["scene_id"], res["im_id"], res["obj_id"]), []).append(i)
    scenes, images = {}, []
    groups = []                      # one per target: (scene, im, obj), kept estimate ids, gt instance ids, valid
    for t in targets:
        s, im, o = t["scene_id"], t["im_id"], t["obj_id"]
        if o not in info:
            raise BopEvalError(f"object {o} of a target is not in {mdir}/models_info.json")
        sc = _scene(scenes, dataset_dir, split, s, im)
        if (s, im) not in images:
            images.append((s, im))
        ests = by_key.get((s, im, o), [])
        ests = sorted(ests, key=lambda i: -results[i]["score"])[:t["inst_count"]]      # stable: csv order on ties
        gts = [k for k, g in enumerate(sc["gt"][im]) if g["obj_id"] == o]
        valid = np.array([sc["visib"][im][k] >= VISIB_GT_MIN for k in gts], bool)
        groups.append(dict(scene_id=s, im_id=im, obj_id=o, est=ests, gt=gts, valid=valid))
    return dict(results=results, targets=targets, groups=groups, images=images, scenes=scenes, info=info, mdir=mdir,
                dataset_dir=dataset_dir, split=split)


# ---------------------------------------------------------------------------------------------------- device stages
def _pose(R, t):
    T = np.eye(4)
    T[:3, :3] = np.asarray(R, np.float64).reshape(3, 3)
    T[:3, 3] = np.asarray(t, np.float64).reshape(3)
    return T


class _Stages:
    """CUDA events around each stage of each chunk (`with stages(name): ...`); milliseconds summed per stage after a
    synchronise.  Disabled, it records nothing."""

    def __init__(self, enabled):
        self.enabled, self.marks = enabled, []

    @contextlib.contextmanager
    def __call__(self, name):
        if not self.enabled:
            yield
            return
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
        self.marks.append((name, ev))
        yield
        ev[1].record()

    def totals(self):
        torch.cuda.synchronize()
        out = {}
        for name, (a, b) in self.marks:
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        return out


def render_depth(dm, poses, K, H, W, z_near, workspace, depth, boxes):
    """One gp_render_depth call on device tensors (dm from icp.device_meshes); enqueued on the current stream."""
    check(_lib.load().gp_render_depth(poses.shape[0], H, W, dm["vertices"].shape[0], dm["vertices"].data_ptr(),
                                      dm["faces"].shape[0], dm["faces"].data_ptr(), poses.data_ptr(), K.data_ptr(),
                                      float(z_near), workspace.data_ptr(), depth.data_ptr(), boxes.data_ptr(),
                                      torch.cuda.current_stream(poses.device).cuda_stream))


def vsd(depth_test, K, frame_idx, est_depth, est_boxes, est_idx, gt_depth, gt_boxes, gt_idx, diameter, delta, taus):
    """gp_bop_vsd on device tensors -> counts i32 [n, 2 + n_tau], errors f32 [n, n_tau]."""
    n, F, H, W = frame_idx.shape[0], depth_test.shape[0], depth_test.shape[1], depth_test.shape[2]
    counts = torch.empty(n, 2 + len(taus), dtype=torch.int32, device=depth_test.device)
    errors = torch.empty(n, len(taus), device=depth_test.device)
    tau = (C.c_float * len(taus))(*taus)
    check(_lib.load().gp_bop_vsd(n, F, H, W, depth_test.data_ptr(), K.data_ptr(), frame_idx.data_ptr(),
                                 est_depth.shape[0], est_depth.data_ptr(), est_boxes.data_ptr(), est_idx.data_ptr(),
                                 gt_depth.shape[0], gt_depth.data_ptr(), gt_boxes.data_ptr(), gt_idx.data_ptr(),
                                 diameter.data_ptr(), float(delta), len(taus), tau, counts.data_ptr(), errors.data_ptr(),
                                 torch.cuda.current_stream(depth_test.device).cuda_stream))
    return counts, errors


def mssd_mspd(obj_idx, vertex_offsets, vertices, sym_offsets, syms, K, frame_idx, pose_est, pose_gt):
    """gp_bop_mssd_mspd on device tensors (offsets are host int sequences), at most MAX_PAIRS_PER_CALL pairs per call
    and no call for no pairs -> mssd, mspd f32 [n]."""
    n = obj_idx.shape[0]
    mssd = torch.empty(n, device=vertices.device)
    mspd = torch.empty(n, device=vertices.device)
    vo = (C.c_int32 * len(vertex_offsets))(*vertex_offsets)
    so = (C.c_int32 * len(sym_offsets))(*sym_offsets)
    lib, stream = _lib.load(), torch.cuda.current_stream(vertices.device).cuda_stream
    # per-pair arrays as (address, bytes per pair): six slices per call would cost more host time than the launch
    rows = [(t.data_ptr(), t.stride(0) * t.element_size()) for t in (obj_idx, frame_idx, pose_est, pose_gt, mssd, mspd)]
    for p0 in range(0, n, MAX_PAIRS_PER_CALL):
        o, f, pe, pg, a, b = (ptr + p0 * step for ptr, step in rows)
        check(lib.gp_bop_mssd_mspd(min(MAX_PAIRS_PER_CALL, n - p0), len(vertex_offsets) - 1, o, vo, vertices.data_ptr(),
                                   so, syms.data_ptr(), K.shape[0], K.data_ptr(), f, pe, pg, a, b, stream))
    return mssd, mspd


def _object_tables(setup, obj_ids, device):
    """Reads each object's PLY once.  -> (host meshes (`read_ply` dicts), the objects' vertices f32 [sum V, 3] and
    symmetry transforms f32 [sum S, 4, 4] concatenated on `device`, vertex offsets and symmetry offsets [n_obj + 1]
    as host ints), in the order of obj_ids: the object tables of gp_bop_mssd_mspd."""
    meshes = [read_ply(os.path.join(setup["mdir"], f"obj_{o:06d}.ply")) for o in obj_ids]
    sym = [symmetry_transforms(setup["info"][o]) for o in obj_ids]
    vertices = torch.as_tensor(np.concatenate([m["vertices"] for m in meshes]), device=device).contiguous()
    syms = torch.as_tensor(np.concatenate(sym), dtype=torch.float32, device=device).contiguous()
    vertex_offsets = np.cumsum([0] + [len(m["vertices"]) for m in meshes]).tolist()
    sym_offsets = np.cumsum([0] + [len(s) for s in sym]).tolist()
    return meshes, vertices, syms, vertex_offsets, sym_offsets


def _pair_rows(groups, group_ids, images):
    """Every (kept estimate, ground truth) pair of groups[gi] for gi in group_ids, group after group, each group a
    row-major [n_est, n_gt] block (the layout gp_bop_match reads).  -> dict of int64 arrays over the pairs: group, est
    (result index), gt (instance index), frame (index of the group's image in `images`)."""
    frame = {key: f for f, key in enumerate(images)}
    cols = dict(group=[], est=[], gt=[], frame=[])
    for gi in group_ids:
        g = groups[gi]
        ne, ng = len(g["est"]), len(g["gt"])
        if ne and ng:
            cols["group"].append(np.full(ne * ng, gi))
            cols["est"].append(np.repeat(np.asarray(g["est"], np.int64), ng))
            cols["gt"].append(np.tile(np.asarray(g["gt"], np.int64), ne))
            cols["frame"].append(np.full(ne * ng, frame[(g["scene_id"], g["im_id"])]))
    return {k: np.concatenate(v).astype(np.int64) if v else np.zeros(0, np.int64) for k, v in cols.items()}


def compute_errors(setup, device="cuda", delta=None, taus=TAUS, z_near=Z_NEAR, stage_ms=None):
    """Per-pair errors of every (kept estimate, ground truth of its object) pair on the device, one chunk of images at a
    time within WORKSPACE_BYTES.  -> dict of numpy arrays over the pairs: group (target index), est (result index),
    gt (instance index in scene_gt), vsd [n, n_tau], vsd_counts [n, 2 + n_tau], mssd, mspd.  `stage_ms` (a dict)
    receives the summed milliseconds of the stages renders / vsd / mssd_mspd, from CUDA events."""
    from .icp import device_meshes
    device = _lib.cuda_device(device, "BOP evaluation")
    if not 1 <= len(taus) <= _lib.BOP_MAX_TAU:
        raise BopEvalError(f"between 1 and {_lib.BOP_MAX_TAU} VSD tolerances, got {len(taus)}")
    if delta is None:
        itodd = os.path.basename(os.path.normpath(setup["dataset_dir"])) == "itodd"
        delta = DELTA_ITODD if itodd else DELTA
    results, groups, scenes, info = setup["results"], setup["groups"], setup["scenes"], setup["info"]
    obj_ids = sorted({g["obj_id"] for g in groups})
    if len(obj_ids) > _lib.BOP_MAX_OBJECTS:
        raise BopEvalError(f"at most {_lib.BOP_MAX_OBJECTS} objects per evaluation")
    oidx = {o: i for i, o in enumerate(obj_ids)}
    out = dict(group=[], est=[], gt=[], vsd=[], vsd_counts=[], mssd=[], mspd=[])
    stages = _Stages(stage_ms is not None)
    with torch.cuda.device(device):
        meshes, vertices, syms, vo, so = _object_tables(setup, obj_ids, device)
        dms = device_meshes(meshes, device)
        diam = {o: info[o]["diameter"] for o in obj_ids}
        by_image = {}
        for gi, g in enumerate(groups):
            by_image.setdefault((g["scene_id"], g["im_id"]), []).append(gi)
        # chunks of images: measured depth plus every render of the chunk within half of the budget
        first = setup["images"][0]
        H, W = load_depth(setup["dataset_dir"], setup["split"], first[0], first[1],
                          scenes[first[0]]["depth_scale"][first[1]]).shape
        plane = 4 * H * W
        chunks, cur, cur_bytes = [], [], 0
        for key in setup["images"]:
            b = plane * (1 + sum(len(groups[gi]["est"]) + len(groups[gi]["gt"]) for gi in by_image[key]))
            if cur and cur_bytes + b > WORKSPACE_BYTES // 2:
                chunks.append(cur)
                cur, cur_bytes = [], 0
            cur.append(key)
            cur_bytes += b
        chunks.append(cur)
        key_views = max(1, WORKSPACE_BYTES // 2 // (8 * H * W))
        keys_ws = torch.empty(key_views * 8 * H * W, dtype=torch.uint8, device=device)
        for chunk in chunks:
            depth_np, K_np, group_ids = [], [], []
            renders = []               # (object, pose [4,4], frame) of every estimate, then every ground truth
            er, gr = {}, {}            # render of each (group, est id) / (group, gt id)
            for f, (s, im) in enumerate(chunk):
                sc = scenes[s]
                d = load_depth(setup["dataset_dir"], setup["split"], s, im, sc["depth_scale"][im])
                if d.shape != (H, W):
                    raise BopEvalError(f"depth of {s}/{im} is {d.shape}, the first image's is {(H, W)}")
                depth_np.append(d)
                K_np.append(sc["K"][im])
                for gi in by_image[(s, im)]:
                    g = groups[gi]
                    for e in g["est"]:
                        er[gi, e] = len(renders)
                        renders.append((g["obj_id"], _pose(results[e]["R"], results[e]["t"]), f))
                    for k in g["gt"]:
                        gr[gi, k] = len(renders)
                        renders.append((g["obj_id"], _pose(sc["gt"][im][k]["R"], sc["gt"][im][k]["t"]), f))
                    group_ids.append(gi)
            rows = _pair_rows(groups, group_ids, chunk)
            if not len(rows["group"]):
                continue
            with stages("renders"):
                depth_test = torch.as_tensor(np.stack(depth_np), device=device)
                K = torch.as_tensor(np.stack(K_np), dtype=torch.float32, device=device).contiguous()
                n_r = len(renders)
                rdepth = torch.empty(n_r, H, W, device=device)
                rboxes = torch.empty(n_r, 4, dtype=torch.int64, device=device)
                poses = torch.as_tensor(np.stack([r[1] for r in renders]), dtype=torch.float32, device=device)
                batches = {}
                for i, (o, _, f) in enumerate(renders):          # one call per (object, K) shares the mesh and K
                    batches.setdefault((o, K_np[f].astype(np.float32).tobytes()), []).append(i)
                for (o, _), idx in batches.items():
                    Kf = K[renders[idx[0]][2]].contiguous()
                    for s0 in range(0, len(idx), key_views):
                        sel = torch.as_tensor(idx[s0:s0 + key_views], device=device)
                        d = torch.empty(len(sel), H, W, device=device)
                        b = torch.empty(len(sel), 4, dtype=torch.int64, device=device)
                        render_depth(dms[oidx[o]], poses[sel].contiguous(), Kf, H, W, z_near, keys_ws, d, b)
                        rdepth[sel], rboxes[sel] = d, b
            group, est, gt = rows["group"].tolist(), rows["est"].tolist(), rows["gt"].tolist()
            col = lambda a: torch.as_tensor(np.asarray(a, np.int32), device=device)
            fi, ei, gi_ = col(rows["frame"]), col([er[p] for p in zip(group, est)]), col([gr[p] for p in zip(group, gt)])
            pair_obj = np.array([oidx[groups[gi]["obj_id"]] for gi in group], np.int32)
            pair_diam = torch.as_tensor(np.array([diam[groups[gi]["obj_id"]] for gi in group], np.float32), device=device)
            with stages("vsd"):
                counts, errs = vsd(depth_test, K, fi, rdepth, rboxes, ei, rdepth, rboxes, gi_, pair_diam, delta, taus)
            with stages("mssd_mspd"):
                mssd, mspd = mssd_mspd(torch.as_tensor(pair_obj, device=device), vo, vertices, so, syms, K, fi,
                                       poses[ei.long()].contiguous(), poses[gi_.long()].contiguous())
            out["group"].append(rows["group"])
            out["est"].append(rows["est"])
            out["gt"].append(rows["gt"])
            out["vsd"].append(errs.cpu().numpy())
            out["vsd_counts"].append(counts.cpu().numpy())
            out["mssd"].append(mssd.cpu().numpy())
            out["mspd"].append(mspd.cpu().numpy())
    if stage_ms is not None:
        stage_ms.update(stages.totals())
    if not out["group"]:
        return dict(group=np.zeros(0, np.int64), est=np.zeros(0, np.int64), gt=np.zeros(0, np.int64),
                    vsd=np.zeros((0, len(taus)), np.float32), vsd_counts=np.zeros((0, 2 + len(taus)), np.int32),
                    mssd=np.zeros(0, np.float32), mspd=np.zeros(0, np.float32))
    return {k: np.concatenate(v) for k, v in out.items()}


def error_groups(setup, errors):
    """Per target: the pairs' errors as [n_est, n_gt] tables in descending score order (the input of `recalls`)."""
    groups = setup["groups"]
    n_tau = errors["vsd"].shape[1]
    out = []
    for g in groups:
        ne, ng = len(g["est"]), len(g["gt"])
        out.append(dict(vsd=np.full((ne, ng, n_tau), np.inf), mssd=np.full((ne, ng), np.inf),
                        mspd=np.full((ne, ng), np.inf), valid=g["valid"],
                        diameter=setup["info"][g["obj_id"]]["diameter"]))
    pos = [({e: i for i, e in enumerate(g["est"])}, {k: i for i, k in enumerate(g["gt"])}) for g in groups]
    for p in range(len(errors["group"])):
        gi = int(errors["group"][p])
        a, b = pos[gi][0][int(errors["est"][p])], pos[gi][1][int(errors["gt"][p])]
        out[gi]["vsd"][a, b] = errors["vsd"][p]
        out[gi]["mssd"][a, b] = errors["mssd"][p]
        out[gi]["mspd"][a, b] = errors["mspd"][p]
    return out


def average_time_per_image(results):
    """Mean over the images with estimates of their csv `time` (the mean of the image's estimates), or -1 when an image
    has none (time < 0) or there are no estimates."""
    per = {}
    for r in results:
        per.setdefault((r["scene_id"], r["im_id"]), []).append(float(r.get("time", -1)))
    if not per or any(min(t) < 0 for t in per.values()):
        return -1.0
    return float(np.mean([np.mean(t) for t in per.values()]))


def _write_scores(out_dir, name, scores):
    """out_dir/name as indented JSON; nothing when out_dir is None."""
    if out_dir is None:
        return
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, name), "w") as f:
        json.dump(scores, f, indent=2)


@torch.no_grad()
def evaluate(results, dataset_dir, split="test", out_dir=None, device="cuda", delta=None, taus=TAUS,
             theta_vsd=THETA_VSD, theta_mssd=THETA_MSSD, theta_mspd=THETA_MSPD,
             targets_name="test_targets_bop19.json", stage_ms=None):
    """BOP 2019 evaluation of `results` (a csv path or a list of `load_bop_results` dicts) on a BOP dataset directory.
    -> dict(ar, ar_vsd, ar_mssd, ar_mspd, recall_vsd [n_tau, n_theta], recall_mssd, recall_mspd, n_targets,
    average_time_per_image, errors (per pair, see `compute_errors`)); with `out_dir`, also writes
    out_dir/scores_bop19.json with the keys the reference's eval_bop.py reads."""
    setup = prepare(results, dataset_dir, split, targets_name)
    errors = compute_errors(setup, device, delta, taus, stage_ms=stage_ms)
    r = image_width(dataset_dir, split, *setup["images"][0]) / 640.0
    n_targets = int(sum(g["valid"].sum() for g in setup["groups"]))
    rec = recalls(error_groups(setup, errors), n_targets, taus, theta_vsd, theta_mssd, theta_mspd, r)
    ar_vsd, ar_mssd, ar_mspd = float(rec["vsd"].mean()), float(rec["mssd"].mean()), float(rec["mspd"].mean())
    out = dict(ar=(ar_vsd + ar_mssd + ar_mspd) / 3.0, ar_vsd=ar_vsd, ar_mssd=ar_mssd, ar_mspd=ar_mspd,
               recall_vsd=rec["vsd"], recall_mssd=rec["mssd"], recall_mspd=rec["mspd"], n_targets=n_targets,
               average_time_per_image=average_time_per_image(setup["results"]), errors=errors)
    _write_scores(out_dir, "scores_bop19.json", {
        "bop19_average_recall": out["ar"], "bop19_average_recall_vsd": ar_vsd, "bop19_average_recall_mssd": ar_mssd,
        "bop19_average_recall_mspd": ar_mspd, "bop19_average_time_per_image": out["average_time_per_image"]})
    return out


# ---------------------------------------------------------------------------------------------------- BOP 2024 detection
# Row f8: the 6D-detection task of BOP 2024 (the reference's `test_setting: detection`, scored with the toolkit's
# eval_bop24_pose.py): every estimate competes, ground truths below VISIB_GT_MIN are ignored rather than missed, and the
# score is COCO-style average precision over MSSD and MSPD.  The statement, with its operation order, is the header
# comment of csrc/bop_eval.cu; the constants below are taken from it and are unverified against eval_bop24_pose.py.
TARGETS_BOP24 = "test_targets_bop24.json"
MAX_ESTIMATES_PER_IMAGE = 100   # highest scores kept per image (stable: csv order on ties)
RECALL_THRESHOLDS = np.linspace(0.0, 1.0, 101)                   # COCO's 101 recall points


def load_target_images(dataset_dir, name=TARGETS_BOP24):
    """-> [(scene_id, im_id)] of a targets file, once each in order of first appearance.  Other keys (obj_id,
    inst_count) are ignored, so both the BOP 2019 and the BOP 2024 target formats load."""
    out = {}
    for t in _json(os.path.join(dataset_dir, name)):
        out.setdefault((int(t["scene_id"]), int(t["im_id"])), None)
    return list(out)


def image_width(dataset_dir, split, scene_id, im_id):
    """Width in pixels, from the header of the image's file under depth/, rgb/ or gray/ (the first that has it)."""
    import glob
    from PIL import Image
    d = os.path.join(dataset_dir, split, f"{scene_id:06d}")
    for sub in ("depth", "rgb", "gray"):
        found = sorted(glob.glob(os.path.join(glob.escape(os.path.join(d, sub)), f"{im_id:06d}.*")))
        if found:
            with Image.open(found[0]) as im:
                return int(im.size[0])
    raise BopEvalError(f"no image {im_id:06d} under {d}/depth, rgb or gray: the image width sets the MSPD threshold")


def prepare_detection(results, dataset_dir, split="test", targets_name=TARGETS_BOP24,
                      max_estimates_per_image=MAX_ESTIMATES_PER_IMAGE):
    """Host side of the detection score: the target images, every ground truth in them (valid when visib_fract >=
    VISIB_GT_MIN, ignored otherwise), the evaluated objects (those with a valid ground truth), and per image the
    max_estimates_per_image highest-scoring estimates (stable sort: csv order on ties) of which those of evaluated
    objects are kept.  -> dict with `images`, `objects`, `n_valid` {obj: valid ground truths}, and `groups`: one per
    (image, evaluated object) with a kept estimate or a ground truth, dict(scene_id, im_id, obj_id, est (result indices
    in descending score order), gt (instance indices in scene_gt), valid [n_gt] bool)."""
    results = load_results(results)
    images = load_target_images(dataset_dir, targets_name)
    mdir = models_dir(dataset_dir)
    info = load_models_info(mdir)
    scenes = {}
    n_valid = {}
    for s, im in images:
        sc = _scene(scenes, dataset_dir, split, s, im)
        for g, v in zip(sc["gt"][im], sc["visib"][im]):
            if v >= VISIB_GT_MIN:
                n_valid[g["obj_id"]] = n_valid.get(g["obj_id"], 0) + 1
    objects = sorted(n_valid)
    for o in objects:
        if o not in info:
            raise BopEvalError(f"object {o} of a ground truth is not in {mdir}/models_info.json")
    by_image = {}
    for i, res in enumerate(results):
        by_image.setdefault((res["scene_id"], res["im_id"]), []).append(i)
    groups = []
    for s, im in images:
        ests = sorted(by_image.get((s, im), []), key=lambda i: -results[i]["score"])[:max_estimates_per_image]
        insts, visib = scenes[s]["gt"][im], scenes[s]["visib"][im]
        for o in objects:
            est = [i for i in ests if results[i]["obj_id"] == o]
            gt = [k for k, g in enumerate(insts) if g["obj_id"] == o]
            if est or gt:
                groups.append(dict(scene_id=s, im_id=im, obj_id=o, est=est, gt=gt,
                                   valid=np.array([visib[k] >= VISIB_GT_MIN for k in gt], bool)))
    return dict(results=results, images=images, scenes=scenes, info=info, mdir=mdir, dataset_dir=dataset_dir,
                split=split, objects=objects, n_valid=n_valid, groups=groups)


def detection_pairs(setup):
    """Every (kept estimate, ground truth) pair of every group, laid out as `_pair_rows` says.  -> dict of int64 arrays
    over the pairs: group, est (result index), gt (instance index), frame (index in setup["images"])."""
    return _pair_rows(setup["groups"], range(len(setup["groups"])), setup["images"])


def _int32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


@torch.no_grad()
def evaluate_detection(results, dataset_dir, split="test", out_dir=None, device="cuda", theta_mssd=THETA_MSSD,
                       theta_mspd=THETA_MSPD, targets_name=TARGETS_BOP24,
                       max_estimates_per_image=MAX_ESTIMATES_PER_IMAGE, stage_ms=None):
    """BOP 2024 6D-detection score of `results` (a csv path or a list of `load_bop_results` dicts) on a BOP dataset
    directory; needs no depth images.  MSSD / MSPD of every pair (gp_bop_mssd_mspd, at most MAX_PAIRS_PER_CALL pairs
    per call), the matching (gp_bop_match) and the AP (gp_bop_average_precision) run on the device in stream order.
    -> dict(map, map_mssd, map_mspd, ap_mssd / ap_mspd [n_objects, n_theta], objects, average_time_per_image,
    errors (per pair: group, est, gt, mssd, mspd), labels i8 [n_rows, 2, n_theta] (GP_BOP_LABEL_*), rows (result index
    of each label row)); with `out_dir`, also writes out_dir/scores_bop24.json.  `stage_ms` (a dict) receives the
    CUDA-event milliseconds of the stages mssd_mspd / match / ap."""
    device = _lib.cuda_device(device, "BOP evaluation")
    T = len(theta_mssd)
    if len(theta_mspd) != T or not 1 <= T <= _lib.BOP_MAX_TAU:
        raise BopEvalError(f"MSSD and MSPD need the same number of thresholds, between 1 and {_lib.BOP_MAX_TAU}")
    setup = prepare_detection(results, dataset_dir, split, targets_name, max_estimates_per_image)
    objects, groups, res, scenes, info = (setup[k] for k in ("objects", "groups", "results", "scenes", "info"))
    if not objects:
        raise BopEvalError(f"no target image has a ground truth with visib_fract >= {VISIB_GT_MIN}")
    if len(objects) > _lib.BOP_MAX_OBJECTS:
        raise BopEvalError(f"at most {_lib.BOP_MAX_OBJECTS} objects per evaluation, got {len(objects)}")
    for g in groups:
        if len(g["gt"]) > _lib.BOP_MAX_GT_PER_GROUP:
            raise BopEvalError(f"image {g['scene_id']}/{g['im_id']} has {len(g['gt'])} instances of object "
                               f"{g['obj_id']}, more than {_lib.BOP_MAX_GT_PER_GROUP}")
    oidx = {o: i for i, o in enumerate(objects)}
    r = image_width(dataset_dir, split, *setup["images"][0]) / 640.0
    pairs = detection_pairs(setup)
    n_pairs, n_obj = len(pairs["group"]), len(objects)
    est_off = np.concatenate([[0], np.cumsum([len(g["est"]) for g in groups])]).astype(np.int32)
    gt_off = np.concatenate([[0], np.cumsum([len(g["gt"]) for g in groups])]).astype(np.int32)
    n_rows = int(est_off[-1])
    rows = np.array([e for g in groups for e in g["est"]], np.int64)
    stages = _Stages(stage_ms is not None)
    lib = _lib.load()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        # one element even for no pairs: gp_bop_match refuses a null pointer, and an empty tensor's data_ptr() is 0
        mssd = mspd = torch.empty(1, device=device)
        if n_pairs:
            _, vertices, syms, vo, so = _object_tables(setup, objects, device)
            K = torch.as_tensor(np.stack([scenes[s]["K"][im] for s, im in setup["images"]]), dtype=torch.float32,
                                device=device).contiguous()
            pose_of_est = {e: _pose(res[e]["R"], res[e]["t"]) for e in set(rows.tolist())}
            pose_est = np.stack([pose_of_est[e] for e in pairs["est"].tolist()]).astype(np.float32)
            pose_gt = np.stack([_pose(scenes[groups[gi]["scene_id"]]["gt"][groups[gi]["im_id"]][k]["R"],
                                      scenes[groups[gi]["scene_id"]]["gt"][groups[gi]["im_id"]][k]["t"])
                                for gi, k in zip(pairs["group"].tolist(), pairs["gt"].tolist())]).astype(np.float32)
            pair_obj = np.array([oidx[groups[gi]["obj_id"]] for gi in pairs["group"].tolist()], np.int32)
            t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=device)
            obj_d, frame_d = t(pair_obj), t(pairs["frame"].astype(np.int32))
            pe_d, pg_d = t(pose_est), t(pose_gt)
            with stages("mssd_mspd"):
                mssd, mspd = mssd_mspd(obj_d, vo, vertices, so, syms, K, frame_d, pe_d, pg_d)
        ap = np.zeros((n_obj, 2, T))
        labels = np.zeros((0, 2, T), np.int8)
        if n_rows:
            thr = np.zeros((n_obj, 2, T))
            for k, o in enumerate(objects):
                thr[k, 0] = np.asarray(theta_mssd) * info[o]["diameter"]
                thr[k, 1] = np.asarray(theta_mspd) * r
            group_obj = np.array([oidx[g["obj_id"]] for g in groups], np.int32)
            valid = torch.as_tensor(np.concatenate([g["valid"] for g in groups]).astype(np.uint8).reshape(-1),
                                    device=device)
            if valid.numel() == 0:
                valid = torch.zeros(1, dtype=torch.uint8, device=device)
            ws = torch.empty(8 * thr.size + _lib.BOP_MATCH_GROUP_BYTES * len(groups), dtype=torch.uint8, device=device)
            lab_d = torch.empty(n_rows, 2, T, dtype=torch.int8, device=device)
            thr = np.ascontiguousarray(thr)
            with stages("match"):
                check(lib.gp_bop_match(len(groups), n_obj, T, _int32p(est_off), _int32p(gt_off), _int32p(group_obj),
                                       thr.ctypes.data_as(C.POINTER(C.c_double)), mssd.data_ptr(), mspd.data_ptr(),
                                       valid.data_ptr(), ws.data_ptr(), lab_d.data_ptr(), stream))
            # every kept estimate of an object over all images, by descending score, csv order on ties (stable)
            row_obj = np.array([oidx[g["obj_id"]] for g in groups for _ in g["est"]], np.int64)
            score = np.array([res[e]["score"] for e in rows.tolist()], np.float64)
            order = np.lexsort((rows, -score, row_obj)).astype(np.int32)
            rank_off = np.concatenate([[0], np.cumsum(np.bincount(row_obj, minlength=n_obj))]).astype(np.int32)
            nv = np.array([setup["n_valid"][o] for o in objects], np.int32)
            rec = np.ascontiguousarray(RECALL_THRESHOLDS, np.float64)
            rank_d = torch.as_tensor(order, device=device)
            ap_d = torch.empty(n_obj, 2, T, dtype=torch.float64, device=device)
            with stages("ap"):
                check(lib.gp_bop_average_precision(n_obj, T, n_rows, lab_d.data_ptr(), _int32p(rank_off),
                                                   rank_d.data_ptr(), _int32p(nv), len(rec),
                                                   rec.ctypes.data_as(C.POINTER(C.c_double)), ap_d.data_ptr(), stream))
            ap, labels = ap_d.cpu().numpy(), lab_d.cpu().numpy()
        errors = dict(group=pairs["group"], est=pairs["est"], gt=pairs["gt"], mssd=mssd[:n_pairs].cpu().numpy(),
                      mspd=mspd[:n_pairs].cpu().numpy())
    if stage_ms is not None:
        stage_ms.update(stages.totals())
    ap_mssd, ap_mspd = np.ascontiguousarray(ap[:, 0]), np.ascontiguousarray(ap[:, 1])
    map_mssd, map_mspd = float(np.mean(ap_mssd)), float(np.mean(ap_mspd))
    out = dict(map=(map_mssd + map_mspd) / 2.0, map_mssd=map_mssd, map_mspd=map_mspd, ap_mssd=ap_mssd, ap_mspd=ap_mspd,
               objects=list(objects), average_time_per_image=average_time_per_image(res), errors=errors,
               labels=labels, rows=rows)
    _write_scores(out_dir, "scores_bop24.json", {"bop24_mAP": out["map"], "bop24_mAP_mssd": map_mssd,
                                                 "bop24_mAP_mspd": map_mspd,
                                                 "bop24_average_time_per_image": out["average_time_per_image"]})
    return out


# ---------------------------------------------------------------------------------------------------- ADD, ADD-S, proj
# Row f12: the metrics of the LM / LM-O (ADD(-S) recall at 0.1 d), YCB-V (AUC of ADD-S and ADD(-S) up to 10 cm) and
# 2D-projection (5 px) tables, on the BOP 2019 targets of `prepare`.  The per-pair errors are gp_bop_add's (definitions
# in csrc/bop_eval.cu, above add_kernel); the matching, recalls and AUCs run here on the host.  This is this
# repository's restatement of MegaPose's vendored pieces (dists_add / dists_add_symmetric, get_top_n_ids, add_valid_gt,
# match_poses, compute_auc_posecnn); the meter that combined them is not part of the reference.
ADD_THRESHOLD = 0.1             # x diameter, ADD-S and ADD(-S)
PROJ_THRESHOLD = 5.0            # px, unscaled
AUC_MAX_M = 0.1                 # PoseCNN's AUC cap, metres
ADD_METRICS = ("add(-s)", "add-s", "proj")


def is_symmetric(info):
    """An object that declares a discrete or a continuous symmetry in models_info.json: ADD(-S) takes its ADD-S."""
    return bool(info.get("symmetries_discrete")) or bool(info.get("symmetries_continuous"))


def add_errors(obj_idx, vertex_offsets, vertices, K, frame_idx, pose_est, pose_gt):
    """gp_bop_add on device tensors (offsets are host int sequences), at most MAX_PAIRS_PER_CALL pairs per call and no
    call for no pairs -> f64 [n, 3] = (ADD, ADD-S, proj)."""
    n = obj_idx.shape[0]
    out = torch.empty(n, 3, dtype=torch.float64, device=vertices.device)
    if n == 0:
        return out
    vo = (C.c_int32 * len(vertex_offsets))(*vertex_offsets)
    max_v = max(b - a for a, b in zip(vertex_offsets[:-1], vertex_offsets[1:]))
    n_chunks = -(-max_v // _lib.BOP_ADD_CHUNK)
    ws = torch.empty(min(n, MAX_PAIRS_PER_CALL) * n_chunks * 3, dtype=torch.float64, device=vertices.device)
    lib, stream = _lib.load(), torch.cuda.current_stream(vertices.device).cuda_stream
    rows = [(t.data_ptr(), t.stride(0) * t.element_size()) for t in (obj_idx, frame_idx, pose_est, pose_gt, out)]
    for p0 in range(0, n, MAX_PAIRS_PER_CALL):
        o, f, pe, pg, d = (ptr + p0 * step for ptr, step in rows)
        check(lib.gp_bop_add(min(MAX_PAIRS_PER_CALL, n - p0), len(vertex_offsets) - 1, o, vo, vertices.data_ptr(),
                             K.shape[0], K.data_ptr(), f, pe, pg, ws.data_ptr(), d, stream))
    return out


def compute_add_errors(setup, device="cuda", stage_ms=None):
    """ADD, ADD-S and proj of every (kept estimate, ground truth of its object) pair of the targets of `prepare`, on
    the device.  -> dict of numpy arrays over the pairs (the layout of `_pair_rows`): group (target index), est (result
    index), gt (instance index in scene_gt), add, adds, proj (f64, model unit and px).  `stage_ms` (a dict) receives
    the CUDA-event milliseconds of the stage `add`."""
    device = _lib.cuda_device(device, "BOP evaluation")
    results, groups, scenes = setup["results"], setup["groups"], setup["scenes"]
    pairs = _pair_rows(groups, range(len(groups)), setup["images"])
    n = len(pairs["group"])
    out = dict(pairs, add=np.zeros(0), adds=np.zeros(0), proj=np.zeros(0))
    del out["frame"]
    if n == 0:
        return out
    obj_ids = sorted({groups[gi]["obj_id"] for gi in set(pairs["group"].tolist())})
    if len(obj_ids) > _lib.BOP_MAX_OBJECTS:
        raise BopEvalError(f"at most {_lib.BOP_MAX_OBJECTS} objects per evaluation")
    oidx = {o: i for i, o in enumerate(obj_ids)}
    stages = _Stages(stage_ms is not None)
    with torch.cuda.device(device):
        _, vertices, _, vo, _ = _object_tables(setup, obj_ids, device)
        K = torch.as_tensor(np.stack([scenes[s]["K"][im] for s, im in setup["images"]]), dtype=torch.float32,
                            device=device).contiguous()
        gl, el, kl = pairs["group"].tolist(), pairs["est"].tolist(), pairs["gt"].tolist()
        pose_est = np.stack([_pose(results[e]["R"], results[e]["t"]) for e in el]).astype(np.float32)
        gts = [scenes[groups[gi]["scene_id"]]["gt"][groups[gi]["im_id"]][k] for gi, k in zip(gl, kl)]
        pose_gt = np.stack([_pose(g["R"], g["t"]) for g in gts]).astype(np.float32)
        t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=device)
        obj_d = t(np.array([oidx[groups[gi]["obj_id"]] for gi in gl], np.int32))
        frame_d = t(pairs["frame"].astype(np.int32))
        with stages("add"):
            err = add_errors(obj_d, vo, vertices, K, frame_d, t(pose_est), t(pose_gt))
        err = err.cpu().numpy()
    if stage_ms is not None:
        stage_ms.update(stages.totals())
    out.update(add=err[:, 0].copy(), adds=err[:, 1].copy(), proj=err[:, 2].copy())
    return out


def match_min_error(err, valid):
    """Minimum-error matching of one target (MegaPose's match_poses rule): err [n_est, n_gt] with the estimates in
    descending score order, valid [n_gt].  Each estimate in turn takes the unmatched valid ground truth with the
    smallest error (strict `<` against a running best that starts at +inf, so the lowest index wins a tie and an inf or
    NaN error never matches); there is no threshold.  -> (matched error per ground truth [n_gt], inf when unmatched;
    the matching estimate's row [n_gt], -1 when unmatched)."""
    err = np.asarray(err, np.float64).reshape(-1, len(valid))
    out = np.full(len(valid), np.inf)
    row_of = np.full(len(valid), -1, np.int64)
    for a, row in enumerate(err):
        best, best_j = np.inf, -1
        for j in range(len(valid)):
            if valid[j] and row_of[j] < 0 and row[j] < best:
                best, best_j = row[j], j
        if best_j >= 0:
            row_of[best_j] = a
            out[best_j] = best
    return out, row_of


def auc_posecnn(errors_m):
    """PoseCNN's area under the accuracy-threshold curve, as MegaPose's compute_auc_posecnn computes it: the errors
    (metres, inf for a missed target) sorted; accuracy (k + 1) / n at the k-th; errors above AUC_MAX_M (and inf or NaN)
    dropped, so an error of exactly AUC_MAX_M counts; the precision envelope made non-decreasing; the step area over
    the recall points [0, kept errors..., AUC_MAX_M], times 10 (= 1 / AUC_MAX_M, applied as a multiplication the way
    MegaPose does).  NaN when no error is within AUC_MAX_M."""
    d = np.sort(np.asarray(errors_m, np.float64))
    acc = np.cumsum(np.ones(len(d))) / len(d)
    keep = d <= AUC_MAX_M
    if not keep.any():
        return float("nan")
    rec = np.concatenate(([0.0], d[keep], [AUC_MAX_M]))
    pre = np.maximum.accumulate(np.concatenate(([0.0], acc[keep], [acc[keep][-1]])))
    i = np.nonzero(rec[1:] != rec[:-1])[0] + 1
    return float(((rec[i] - rec[i - 1]) * pre[i]).sum() * 10.0)


def add_scores(setup, errors):
    """Host half of `evaluate_add`: per target, each metric matched on its own error (`match_min_error`), then the
    recalls (matched valid ground truths with error < threshold over n_targets; 0.1 x diameter for ADD-S and ADD(-S),
    5 px for proj) and the AUCs of ADD-S and ADD(-S) (`auc_posecnn` on mm / 1000, inf for an unmatched target), over
    all targets and per object.  The targets are the valid ground truths, target group after target group.
    -> dict(n_targets, matched {metric: matched error f64 [n_targets], inf if missed}, matched_est {metric: result
    index of the matching estimate [n_targets], -1 if missed}, target_obj [n_targets], target_gt [(target group,
    instance index)], recall {metric}, auc {metric}, objects {obj_id: dict(n_targets, recall, auc)})."""
    groups, info = setup["groups"], setup["info"]
    pos = [({e: i for i, e in enumerate(g["est"])}, {k: i for i, k in enumerate(g["gt"])}) for g in groups]
    tables = [{m: np.full((len(g["est"]), len(g["gt"])), np.inf) for m in ADD_METRICS} for g in groups]
    for p in range(len(errors["group"])):
        gi = int(errors["group"][p])
        a, b = pos[gi][0][int(errors["est"][p])], pos[gi][1][int(errors["gt"][p])]
        sym = is_symmetric(info[groups[gi]["obj_id"]])
        tables[gi]["add(-s)"][a, b] = errors["adds"][p] if sym else errors["add"][p]
        tables[gi]["add-s"][a, b] = errors["adds"][p]
        tables[gi]["proj"][a, b] = errors["proj"][p]
    matched, matched_est = {m: [] for m in ADD_METRICS}, {m: [] for m in ADD_METRICS}
    target_obj, target_gt, thr = [], [], {m: [] for m in ADD_METRICS}
    for gi, (g, tab) in enumerate(zip(groups, tables)):
        v = np.asarray(g["valid"], bool)
        for m in ADD_METRICS:
            e, a = match_min_error(tab[m], v)
            matched[m].append(e[v])
            matched_est[m].append(np.array([g["est"][i] if i >= 0 else -1 for i in a[v]], np.int64))
        target_gt += [(gi, k) for k, ok in zip(g["gt"], v) if ok]
        n = int(v.sum())
        target_obj += [g["obj_id"]] * n
        d = info[g["obj_id"]]["diameter"]
        thr["add(-s)"] += [ADD_THRESHOLD * d] * n
        thr["add-s"] += [ADD_THRESHOLD * d] * n
        thr["proj"] += [PROJ_THRESHOLD] * n
    matched = {m: np.concatenate(v) if v else np.zeros(0) for m, v in matched.items()}
    matched_est = {m: np.concatenate(v) if v else np.zeros(0, np.int64) for m, v in matched_est.items()}
    target_obj = np.asarray(target_obj, np.int64)
    thr = {m: np.asarray(v, np.float64) for m, v in thr.items()}

    def scores(sel):
        n = int(sel.sum())
        rec = {m: float(np.count_nonzero(matched[m][sel] < thr[m][sel]) / max(n, 1)) for m in ADD_METRICS}
        auc = {m: auc_posecnn(matched[m][sel] / 1000.0) if n else float("nan") for m in ("add(-s)", "add-s")}
        return n, rec, auc

    n_targets, recall, auc = scores(np.ones(len(target_obj), bool))
    objects = {}
    for o in sorted(set(target_obj.tolist())):
        n, rec, a = scores(target_obj == o)
        objects[o] = dict(n_targets=n, recall=rec, auc=a)
    return dict(n_targets=n_targets, matched=matched, matched_est=matched_est, target_obj=target_obj,
                target_gt=target_gt, recall=recall, auc=auc, objects=objects)


def _add_json(n_targets, recall, auc):
    return {"add(-s)_0.1d": recall["add(-s)"], "add-s_0.1d": recall["add-s"], "proj_5px": recall["proj"],
            "auc_add(-s)": auc["add(-s)"], "auc_add-s": auc["add-s"], "n_targets": n_targets}


@torch.no_grad()
def evaluate_add(results, dataset_dir, split="test", out_dir=None, device="cuda",
                 targets_name="test_targets_bop19.json", stage_ms=None):
    """ADD, ADD-S and 2D-projection scores of `results` (a csv path or a list of `load_bop_results` dicts) on the BOP
    2019 targets of a dataset directory; needs no depth images.  -> dict(errors (per pair: group, est, gt, add, adds,
    proj), matched / matched_est / target_obj / target_gt (per target, see `add_scores`), recall / auc {metric}, n_targets,
    objects {obj_id: dict(n_targets, recall, auc)}, scores (the JSON below)).  Metrics: "add(-s)" (ADD-S for an object
    with declared symmetries, else ADD), "add-s", "proj".  With `out_dir`, writes out_dir/scores_add.json:
    add(-s)_0.1d, add-s_0.1d, proj_5px (recalls), auc_add(-s), auc_add-s (NaN when no target is within 0.1 m),
    n_targets, and the same keys per object under "objects" {obj_id}.  `stage_ms` (a dict) receives the CUDA-event
    milliseconds of the stage `add`."""
    setup = prepare(results, dataset_dir, split, targets_name)
    errors = compute_add_errors(setup, device, stage_ms=stage_ms)
    s = add_scores(setup, errors)
    scores = dict(_add_json(s["n_targets"], s["recall"], s["auc"]),
                  objects={str(o): _add_json(v["n_targets"], v["recall"], v["auc"]) for o, v in s["objects"].items()})
    _write_scores(out_dir, "scores_add.json", scores)
    return dict(s, errors=errors, scores=scores)


def main(argv=None):
    ap = argparse.ArgumentParser(description="BOP pose-error evaluation on the GPU: the BOP 2019 localization task "
                                             "(VSD, MSSD, MSPD, AR), the BOP 2024 6D-detection task (MSSD, MSPD, mAP) "
                                             "or ADD / ADD-S / 2D-projection scores on the BOP 2019 targets")
    ap.add_argument("--results", required=True, help="BOP results csv")
    ap.add_argument("--dataset-dir", required=True)
    ap.add_argument("--split", default="test")
    ap.add_argument("--task", choices=("localization", "detection", "add"), default="localization")
    ap.add_argument("--out", default=None, help="directory for scores_bop19.json / scores_bop24.json / scores_add.json "
                                                "(default: next to the csv)")
    a = ap.parse_args(argv)
    out_dir = a.out if a.out is not None else os.path.dirname(os.path.abspath(a.results))
    if a.task == "add":
        res = evaluate_add(a.results, a.dataset_dir, a.split, out_dir=out_dir)
        print(json.dumps({k: v for k, v in res["scores"].items() if k != "objects"}))
        return
    if a.task == "detection":
        res = evaluate_detection(a.results, a.dataset_dir, a.split, out_dir=out_dir)
        print(json.dumps({k: res[k] for k in ("map", "map_mssd", "map_mspd", "objects", "average_time_per_image")}))
        return
    res = evaluate(a.results, a.dataset_dir, a.split, out_dir=out_dir)
    print(json.dumps({k: res[k] for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd", "n_targets",
                                          "average_time_per_image")}))


if __name__ == "__main__":
    main()
