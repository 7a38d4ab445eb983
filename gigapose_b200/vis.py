"""The reference's diagnostic images on the GPU (row f14): result overlays, per-vertex error heat maps and retrieval
panels.  The kernels are csrc/vis.cu (whose header comment states every rounding); this module holds their ctypes
wrappers, `render_results` and its command line:

    python -m gigapose_b200.vis --results A.csv [B.csv ...] --dataset-dir D [--split test] [--out DIR]
                                [--max-images N] [--max-distance-mm 100]

For each image of test_targets_bop19.json it writes `<scene>_<im>.png` in the layout of the reference's
src/scripts/vis_bop_results.py: the top row is the RGB image followed by one error heat map per csv, the bottom row the
ground truths drawn over a grey copy of the image (green contours) followed by each csv's estimates (red contours).
Give a coarse and a refined csv together (for example `..._icp.csv`) to compare them.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._lib import GigaPoseNativeError, check

MAX_PAIRS_PER_CALL = 1 << 16
MAX_DISTANCE_MM = 100.0          # the reference's max_distance = 10 in its scene unit (the mesh scaled by 0.1 from mm)
GT_COLOR = (0, 255, 0)
EST_COLOR = (255, 0, 0)
Z_NEAR = 10.0                    # model unit (mm)


def _need(cond, msg):
    if not cond:
        raise GigaPoseNativeError(msg)


def _cuda(t, name, dtype, shape=None):
    _need(torch.is_tensor(t) and t.is_cuda, f"{name} must be a CUDA tensor")
    _need(t.dtype == dtype, f"{name} must be {dtype}, got {t.dtype}")
    _need(t.is_contiguous(), f"{name} must be contiguous")
    if shape is not None:
        _need(tuple(t.shape) == tuple(shape), f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
    return t


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


# ---------------------------------------------------------------------------------------------------- wrappers
def vertex_errors(obj_idx, vertex_offsets, vertices, pose_est, pose_gt, symmetric):
    """gp_vis_vertex_errors.  obj_idx: host int sequence [n] (0-based); vertex_offsets: host ints [n_obj + 1];
    vertices f32 [sum V, 3], pose_est / pose_gt f32 [n,4,4] on the device; symmetric: host bools [n].
    -> (values f32 [sum of the pairs' V] on the device, offsets i64 [n + 1] on the host).  ADD distances per vertex, ADD-S
    distances for the symmetric pairs."""
    obj_idx = np.asarray(obj_idx, np.int64).reshape(-1)
    sym = np.asarray(symmetric, bool).reshape(-1)
    n, n_obj = len(obj_idx), len(vertex_offsets) - 1
    _need(len(sym) == n, f"symmetric has {len(sym)} entries for {n} pairs")
    _need(1 <= n_obj <= _lib.BOP_MAX_OBJECTS, f"{n_obj} objects outside [1, {_lib.BOP_MAX_OBJECTS}]")
    _need(n == 0 or (obj_idx.min() >= 0 and obj_idx.max() < n_obj), f"obj_idx outside [0, {n_obj})")
    _cuda(vertices, "vertices", torch.float32)
    _need(vertices.dim() == 2 and vertices.shape[1] == 3 and vertices.shape[0] == vertex_offsets[-1],
          "vertices must be [vertex_offsets[-1], 3]")
    dev = vertices.device
    _cuda(pose_est, "pose_est", torch.float32, (n, 4, 4))
    _cuda(pose_gt, "pose_gt", torch.float32, (n, 4, 4))
    counts = np.diff(np.asarray(vertex_offsets, np.int64))[obj_idx] if n else np.zeros(0, np.int64)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    values = torch.empty(int(offsets[-1]), dtype=torch.float32, device=dev)
    if n == 0:
        return values, offsets
    vo = (C.c_int32 * len(vertex_offsets))(*vertex_offsets)
    lib, stream = _lib.load(), _stream(vertices)
    o_d = torch.as_tensor(obj_idx.astype(np.int32), device=dev)
    s_d = torch.as_tensor(sym.astype(np.uint8), device=dev)
    for p0 in range(0, n, MAX_PAIRS_PER_CALL):
        p1 = min(n, p0 + MAX_PAIRS_PER_CALL)
        off_d = torch.as_tensor(offsets[p0:p1 + 1] - offsets[p0], device=dev)
        check(lib.gp_vis_vertex_errors(p1 - p0, n_obj, o_d[p0:].data_ptr(), vo, vertices.data_ptr(),
                                       pose_est[p0:].data_ptr(), pose_gt[p0:].data_ptr(), s_d[p0:].data_ptr(),
                                       off_d.data_ptr(), values[int(offsets[p0]):].data_ptr(), stream))
    return values, offsets


def heat_colors(values, offsets, symmetric, max_distance=MAX_DISTANCE_MM):
    """gp_vis_heat_colors.  values f32 [N] on the device and host offsets i64 [n + 1] as vertex_errors returns them,
    symmetric host bools [n], max_distance > 0 in the unit of the values -> colours f32 [N, 3] in [0, 1]."""
    offsets = np.asarray(offsets, np.int64).reshape(-1)
    sym = np.asarray(symmetric, bool).reshape(-1)
    n = len(offsets) - 1
    _need(n >= 0 and len(sym) == n, f"symmetric has {len(sym)} entries for {n} pairs")
    _need(np.isfinite(max_distance) and max_distance > 0, "max_distance must be positive and finite")
    _cuda(values, "values", torch.float32)
    _need(values.dim() == 1 and values.shape[0] == (offsets[-1] if n >= 0 and len(offsets) else 0),
          "values must be [offsets[-1]]")
    _need(len(offsets) >= 1 and offsets[0] == 0 and np.all(np.diff(offsets) >= 0), "offsets must start at 0 and not decrease")
    colors = torch.empty(values.shape[0], 3, dtype=torch.float32, device=values.device)
    if n == 0:
        return colors
    lib, stream = _lib.load(), _stream(values)
    s_d = torch.as_tensor(sym.astype(np.uint8), device=values.device)
    for p0 in range(0, n, MAX_PAIRS_PER_CALL):
        p1 = min(n, p0 + MAX_PAIRS_PER_CALL)
        off_d = torch.as_tensor(offsets[p0:p1 + 1] - offsets[p0], device=values.device)
        check(lib.gp_vis_heat_colors(p1 - p0, off_d.data_ptr(), s_d[p0:].data_ptr(),
                                     values[int(offsets[p0]):].data_ptr(), float(max_distance),
                                     colors[int(offsets[p0]):].data_ptr(), stream))
    return colors


def overlay(image, renders, boxes, colors=None, size=None):
    """gp_vis_overlay.  image u8 [H,W,3] on the device, or None for a black background (then `size` = (H, W) or the
    renders' size); renders f32 [n,4,H,W] and boxes i64 [n,4] as render_templates returns them; colors: outline colour
    per layer, u8 [n,3] (any sequence), or None for no contours.  -> u8 [H,W,3] on the device."""
    if image is not None:
        _cuda(image, "image", torch.uint8)
        _need(image.dim() == 3 and image.shape[2] == 3, "image must be [H,W,3]")
        H, W = image.shape[:2]
        dev = image.device
    else:
        _need(size is not None or (renders is not None and len(renders)), "a black background needs `size`")
        H, W = size if size is not None else renders.shape[-2:]
        dev = renders.device if renders is not None else torch.device("cuda", torch.cuda.current_device())
    _need(1 <= H <= _lib.VIS_MAX_SIDE and 1 <= W <= _lib.VIS_MAX_SIDE, f"image size {H} x {W} outside [1, {_lib.VIS_MAX_SIDE}]")
    n = 0 if renders is None else renders.shape[0]
    if n:
        _cuda(renders, "renders", torch.float32, (n, 4, H, W))
        _cuda(boxes, "boxes", torch.int64, (n, 4))
        _need(renders.device == dev and boxes.device == dev, "image, renders and boxes must be on one device")
    col = None
    if colors is not None and n:
        col = torch.as_tensor(np.asarray(colors, np.uint8).reshape(-1, 3), device=dev)
        _need(col.shape[0] == n, f"{col.shape[0]} colours for {n} layers")
    out = torch.empty(H, W, 3, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().gp_vis_overlay(H, W, n, _lib.ptr(image), renders.data_ptr() if n else None,
                                         boxes.data_ptr() if n else None, _lib.ptr(col), out.data_ptr(), _stream(out)))
    return out


def kabsch(query, query_mask, tmpl, tmpl_mask, M):
    """gp_vis_kabsch.  query / tmpl f32 [b,3,224,224] normalised crops, query_mask / tmpl_mask f32 [b,224,224], M f32
    [b,3,3] (template crop -> query crop), all on one device -> u8 [b,224,224,3] (plot_Kabsch's panel)."""
    S = _lib.VIS_CROP
    _cuda(query, "query", torch.float32)
    b = query.shape[0]
    _cuda(query, "query", torch.float32, (b, 3, S, S))
    _cuda(tmpl, "tmpl", torch.float32, (b, 3, S, S))
    _cuda(query_mask, "query_mask", torch.float32, (b, S, S))
    _cuda(tmpl_mask, "tmpl_mask", torch.float32, (b, S, S))
    _cuda(M, "M", torch.float32, (b, 3, 3))
    _need(len({t.device for t in (query, tmpl, query_mask, tmpl_mask, M)}) == 1, "all inputs must be on one device")
    out = torch.empty(b, S, S, 3, dtype=torch.uint8, device=query.device)
    lib, stream = _lib.load(), _stream(query)
    for b0 in range(0, b, 65535):
        b1 = min(b, b0 + 65535)
        check(lib.gp_vis_kabsch(b1 - b0, query[b0:].data_ptr(), query_mask[b0:].data_ptr(), tmpl[b0:].data_ptr(),
                                tmpl_mask[b0:].data_ptr(), M[b0:].data_ptr(), out[b0:].data_ptr(), stream))
    return out


# ---------------------------------------------------------------------------------------------------- result figures
def result_lists(results):
    """The results argument of `plan` / `render_results` as a list of result lists: one csv path, one result list (a
    list of result dicts), or a sequence of csv paths and result lists, one per method."""
    from . import bop_eval
    if isinstance(results, (str, os.PathLike)):
        results = [results]
    results = list(results)
    if results and all(isinstance(r, dict) for r in results):
        results = [results]                     # one result list, not one csv per result
    if not results:
        raise ValueError("no results to draw")
    return [bop_eval.load_results(r) for r in results]


def display_models_dir(dataset_dir):
    """The models the overlays draw, the reference's Panda3D models: models_reconst/ where a dataset has it (T-LESS),
    else the textured models/; the evaluation models (bop_eval.models_dir) when neither exists.  The errors, the
    pairing and the heat maps use the evaluation models."""
    from . import bop_eval
    for name in ("models_reconst", "models"):
        d = os.path.join(dataset_dir, name)
        if os.path.isdir(d):
            return d
    return bop_eval.models_dir(dataset_dir)


def plan(results, dataset_dir, split="test", max_images=None, targets_name="test_targets_bop19.json"):
    """Host side of `render_results`: the target images in the order of the targets file (at most `max_images`), each
    with its ground truths of the target objects sorted far to near by |t| (the reference's order), and per results
    list the `inst_count` highest-scoring estimates of each target object (stable: csv order on ties).  `results` as
    `result_lists` takes it.
    -> dict(images=[dict(scene_id, im_id, K, gt=[dict(R, t, obj_id)], est=[[result index...] per results list],
    targets={obj_id: inst_count})], results=[list of result dicts per csv], info, mdir)."""
    from . import bop_eval
    results = result_lists(results)
    targets = bop_eval.load_targets(dataset_dir, targets_name)
    mdir = bop_eval.models_dir(dataset_dir)
    info = bop_eval.load_models_info(mdir)
    order, per_image = [], {}
    for t in targets:
        key = (t["scene_id"], t["im_id"])
        if key not in per_image:
            order.append(key)
            per_image[key] = {}
        per_image[key][t["obj_id"]] = t["inst_count"]
    if max_images is not None:
        order = order[:max_images]
    by_key = []
    for res in results:
        d = {}
        for i, r in enumerate(res):
            d.setdefault((r["scene_id"], r["im_id"], r["obj_id"]), []).append(i)
        by_key.append(d)
    scenes, images = {}, []
    for s, im in order:
        sc = bop_eval._scene(scenes, dataset_dir, split, s, im)
        objs = per_image[(s, im)]
        gts = [g for g in sc["gt"][im] if g["obj_id"] in objs]
        gts = [gts[k] for k in sorted(range(len(gts)), key=lambda k: -np.linalg.norm(gts[k]["t"]))]
        est = []
        for res, d in zip(results, by_key):
            kept = []
            for o, n in objs.items():
                kept += sorted(d.get((s, im, o), []), key=lambda i: -res[i]["score"])[:n]
            est.append(kept)
        images.append(dict(scene_id=s, im_id=im, K=sc["K"][im], gt=gts, est=est, targets=objs))
    return dict(images=images, results=results, info=info, mdir=mdir)


def pair_estimates(image, results, ests, err):
    """Pairs the kept estimates `ests` (indices into `results`) of an image with its ground truths, per target object, by f12's
    minimum-error matching (bop_eval.match_min_error) on `err[(est, gt)]`, the ADD(-S) error of result `est` against
    ground truth `gt` (an index into image["gt"]).  -> {result index: gt index or None}."""
    from .bop_eval import match_min_error
    out = {}
    for o in image["targets"]:
        mine = [e for e in ests if results[e]["obj_id"] == o]
        gts = [k for k, g in enumerate(image["gt"]) if g["obj_id"] == o]
        for e in mine:
            out[e] = None
        if not mine or not gts:
            continue
        E = np.array([[err[(e, k)] for k in gts] for e in mine], np.float64)
        _, row_of = match_min_error(E, np.ones(len(gts), bool))
        for j, a in enumerate(row_of):
            if a >= 0:
                out[mine[a]] = gts[j]
    return out


def _pose(R, t):
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = np.asarray(R, np.float64).reshape(3, 3)
    T[:3, 3] = np.asarray(t, np.float64).reshape(3)
    return T


def _far_to_near(poses):
    return sorted(range(len(poses)), key=lambda i: -float(np.linalg.norm(poses[i][:3, 3].astype(np.float64))))


@torch.no_grad()
def render_results(results, dataset_dir, out_dir, split="test", max_images=None, max_distance_mm=MAX_DISTANCE_MM,
                   device="cuda", stage_ms=None):
    """Writes `<scene>_<im>.png` (the reference's two-row figure) for the target images of `dataset_dir` into `out_dir`
    for `results`: one csv path or result list, or a sequence of them, one per method (`result_lists`).
    The overlays draw the models of `display_models_dir`; the ADD(-S) pairing, the per-vertex errors and the heat maps
    use the evaluation models (`bop_eval.models_dir`).  A heat map draws each matched estimate's errors on its ground
    truth's model at the ground truth's pose, as the reference paints them on its ground-truth entity.
    -> list of the written paths.  `stage_ms` (a dict)
    receives the CUDA-event milliseconds of the stages render, vertex_errors, overlay, and the wall-clock
    milliseconds of png."""
    import time
    from PIL import Image

    from . import bop_eval
    from .bop_run import image_path, read_image
    from .render import _device_mesh, read_ply, render_templates
    device = _lib.cuda_device(device, "render_results")
    p = plan(results, dataset_dir, split, max_images)
    os.makedirs(out_dir, exist_ok=True)
    stages = bop_eval._Stages(stage_ms is not None)
    png_ms = 0.0
    shown_dir, meshes = display_models_dir(dataset_dir), {}

    def load(mdir, o):
        """an object's mesh, uploaded once: render_templates takes the device tensors as they are"""
        if (mdir, o) not in meshes:
            meshes[(mdir, o)] = _device_mesh(read_ply(os.path.join(mdir, f"obj_{o:06d}.ply")), device)
        return meshes[(mdir, o)]

    mesh = lambda o: load(p["mdir"], o)                      # evaluation model: errors, pairing, heat maps
    shown = lambda o: load(shown_dir, o)                     # overlays

    written = []
    with torch.cuda.device(device):
        for image in p["images"]:
            s, im = image["scene_id"], image["im_id"]
            rgb = read_image(image_path(dataset_dir, split, s, im))
            H, W = rgb.shape[:2]
            K = np.asarray(image["K"], np.float32)
            img_d = torch.as_tensor(np.array(rgb), device=device)        # read_image's array is read-only

            def draw(layers, colors, background):
                """layers: [(mesh dict, pose [4,4])] -> u8 [H,W,3] on the device, far to near."""
                if not layers:
                    return overlay(background, None, None, size=(H, W))
                order = _far_to_near([T for _, T in layers])
                rgba, boxes = [], []
                with stages("render"):
                    for i in order:
                        r = render_templates(layers[i][0], torch.as_tensor(layers[i][1][None], device=device), K,
                                             size=(H, W), z_near=Z_NEAR, device=device)
                        rgba.append(r["rgba"])
                        boxes.append(r["boxes"])
                with stages("overlay"):
                    return overlay(background, torch.cat(rgba), torch.cat(boxes),
                                   None if colors is None else [colors[i] for i in order], size=(H, W))

            gt_poses = [_pose(g["R"], g["t"]) for g in image["gt"]]
            top, bottom = [img_d], [draw([(shown(g["obj_id"]), T) for g, T in zip(image["gt"], gt_poses)],
                                         [GT_COLOR] * len(gt_poses), img_d)]
            for res, ests in zip(p["results"], image["est"]):
                est_poses = {e: _pose(res[e]["R"], res[e]["t"]) for e in ests}
                # ADD(-S) of every (estimate, ground truth of its object) pair, then the minimum-error matching
                cand = [(e, k) for e in ests for k, g in enumerate(image["gt"]) if g["obj_id"] == res[e]["obj_id"]]
                err = {}
                if cand:
                    objs = sorted({res[e]["obj_id"] for e, _ in cand})
                    oi = {o: i for i, o in enumerate(objs)}
                    V = torch.cat([mesh(o)["vertices"] for o in objs]).contiguous()
                    vo = np.cumsum([0] + [len(mesh(o)["vertices"]) for o in objs]).tolist()
                    pe = torch.as_tensor(np.stack([est_poses[e] for e, _ in cand]), device=device)
                    pg = torch.as_tensor(np.stack([gt_poses[k] for _, k in cand]), device=device)
                    Kd = torch.as_tensor(K[None], device=device)
                    o_d = torch.as_tensor(np.array([oi[res[e]["obj_id"]] for e, _ in cand], np.int32), device=device)
                    f_d = torch.zeros(len(cand), dtype=torch.int32, device=device)
                    with stages("vertex_errors"):
                        a = bop_eval.add_errors(o_d, vo, V, Kd, f_d, pe, pg).cpu().numpy()
                    for (e, k), row in zip(cand, a):
                        err[(e, k)] = row[1] if bop_eval.is_symmetric(p["info"][res[e]["obj_id"]]) else row[0]
                match = pair_estimates(image, res, ests, err)
                bottom.append(draw([(shown(res[e]["obj_id"]), est_poses[e]) for e in ests], [EST_COLOR] * len(ests),
                                   img_d))
                # heat map: each matched estimate's per-vertex error colours on its ground truth's model at the ground
                # truth's pose (ADD-S value j belongs to ground-truth point j), over black, no contour
                pairs = [(e, k) for e, k in match.items() if k is not None]
                layers = []
                if pairs:
                    objs = sorted({res[e]["obj_id"] for e, _ in pairs})
                    oi = {o: i for i, o in enumerate(objs)}
                    V = torch.cat([mesh(o)["vertices"] for o in objs]).contiguous()
                    vo = np.cumsum([0] + [len(mesh(o)["vertices"]) for o in objs]).tolist()
                    sym = [bop_eval.is_symmetric(p["info"][res[e]["obj_id"]]) for e, _ in pairs]
                    pe = torch.as_tensor(np.stack([est_poses[e] for e, _ in pairs]), device=device)
                    pg = torch.as_tensor(np.stack([gt_poses[k] for _, k in pairs]), device=device)
                    with stages("vertex_errors"):
                        vals, offs = vertex_errors([oi[res[e]["obj_id"]] for e, _ in pairs], vo, V, pe, pg, sym)
                        cols = heat_colors(vals, offs, sym, max_distance_mm)
                    for j, (e, k) in enumerate(pairs):
                        m = mesh(res[e]["obj_id"])
                        layers.append((dict(vertices=m["vertices"], faces=m["faces"],
                                            vertex_color=cols[int(offs[j]):int(offs[j + 1])]), gt_poses[k]))
                top.append(draw(layers, None, None))
            fig = torch.cat([torch.cat(top, 1), torch.cat(bottom, 1)], 0).cpu().numpy()
            t0 = time.perf_counter()
            path = os.path.join(out_dir, f"{s:06d}_{im:06d}.png")
            Image.fromarray(fig).save(path)
            png_ms += (time.perf_counter() - t0) * 1e3
            written.append(path)
    if stage_ms is not None:
        stage_ms.update(stages.totals())
        stage_ms["png"] = png_ms
    return written


def parser():
    ap = argparse.ArgumentParser(description="Draw BOP results: overlays and per-vertex error heat maps per image")
    ap.add_argument("--results", nargs="+", required=True, help="one or more BOP results csvs (e.g. coarse and _icp)")
    ap.add_argument("--dataset-dir", required=True)
    ap.add_argument("--split", default="test")
    ap.add_argument("--out", default="vis_out")
    ap.add_argument("--max-images", type=int, default=None)
    ap.add_argument("--max-distance-mm", type=float, default=MAX_DISTANCE_MM,
                    help="error at the top of the heat-map colour scale (the reference's 10 cm)")
    ap.add_argument("--device", default="cuda")
    return ap


def main(argv=None):
    a = parser().parse_args(argv)
    for path in render_results(a.results, a.dataset_dir, a.out, a.split, a.max_images, a.max_distance_mm, a.device):
        print(path)


if __name__ == "__main__":
    main()
