"""Depth refinement of coarse poses on the GPU (row f6): every hypothesis is rendered at its pose with the frame's K
(`gp_render_templates`), the measured depth of each frame becomes an organised target map with normals
(`gp_icp_prepare_scene`), and one CTA per hypothesis runs the centroid shift and a point-to-plane ICP
(`gp_icp_refine`).  csrc/depth_icp.cu's header comment states the contract; it restates MegaPose's ICPRefiner
(src/megapose/inference/icp_refiner.py:134-287) with the deviations listed in INTEGRATION.md.  Row f10:
`score_hypotheses` renders final poses the same way and scores them against the measured depth (`gp_depth_score`,
csrc/depth_score.cu), so that the best hypothesis of a detection can be kept.  Row f11: `refine_icp_masked` smooths the
target normals within each detection's own mask (dense or COCO run-length), over the mask's box only."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import GpIcpDebug, GpIcpMaskSet, GpIcpParams, check, ptr
from .render import _device_mesh, render_chunk

STATUS_NAMES = {_lib.ICP_OK: "ok", _lib.ICP_TOO_FEW_POINTS: "too few points", _lib.ICP_DEGENERATE: "degenerate",
                _lib.ICP_RESIDUAL: "residual above max_residual", _lib.ICP_INVALID: "invalid frame index",
                _lib.ICP_LOST: "lost: no pairs, or fewer than 6 kept"}
DEFAULTS = dict(unit_per_m=1000.0, min_points=1000, num_levels=4, max_iters=100, rejection_scale=2.5,
                max_residual=0.01, min_step_rad=1e-6, min_step_m=1e-6)
WORKSPACE_BYTES = 1 << 30          # renders + refiner scratch per chunk of hypotheses: ~20 MB per 640 x 480 hypothesis


def _params(struct, debug_struct, defaults, what, debug, params):
    """A refiner's params `struct` from `defaults` updated with `params`, and its debug member from `debug` (ints as
    they are, tensors as device addresses); unknown names raise TypeError."""
    unknown = set(params) - set(defaults)
    if unknown:
        raise TypeError(f"unknown {what} parameters {sorted(unknown)}")
    out = struct(**dict(defaults, **params))
    if debug:
        out.debug = debug_struct(**{k: v if isinstance(v, int) else ptr(v) for k, v in debug.items()})
    return out


def make_params(debug=None, **params) -> GpIcpParams:
    return _params(GpIcpParams, GpIcpDebug, DEFAULTS, "ICP", debug, params)


def _outputs(n, device, dtype):
    """A refiner's four per-hypothesis outputs: poses f32 [n,4,4], status i32 [n] and two [n] of `dtype`."""
    return (torch.empty(n, 4, 4, device=device), torch.empty(n, dtype=torch.int32, device=device),
            torch.empty(n, dtype=dtype, device=device), torch.empty(n, dtype=dtype, device=device))


def _refine_call(entry, args, n, device, dtype, *workspaces):
    """A refiner's entry point on n hypotheses: `args` (everything before its outputs), its `_outputs`, `workspaces`
    and the current stream.  -> the outputs."""
    out = _outputs(n, device, dtype)
    check(entry(*args, *(t.data_ptr() for t in out), *(w.data_ptr() for w in workspaces),
                torch.cuda.current_stream(device).cuda_stream))
    return out


def device_meshes(meshes, device):
    """`read_ply` dicts (or paths) -> the device tensors the renderer takes, uploaded once."""
    from .render import read_ply
    return [_device_mesh(read_ply(m) if isinstance(m, str) else m, device) for m in meshes]


def render_hypotheses(meshes_dev, labels, poses, K, frame_idx, H, W, unit_per_m=1000.0):
    """Depth [n,H,W] and boxes [n,4] of mesh labels[i] at poses[i] with K[frame_idx[i]], rendered in groups of equal
    (object, frame); z_near = 0.1 m, Panda3D's."""
    device = poses.device
    n = poses.shape[0]
    per_view = C.c_size_t()
    check(_lib.load().gp_render_query_sizes(1, H, W, C.byref(per_view)))
    depth = torch.empty(n, H, W, device=device)
    boxes = torch.empty(n, 4, dtype=torch.int64, device=device)
    lab, fr = labels.tolist(), frame_idx.tolist()
    groups = {}
    for i, key in enumerate(zip(lab, fr)):
        groups.setdefault(key, []).append(i)
    chunk = max(1, min(n, WORKSPACE_BYTES // 2 // (per_view.value + 16 * H * W)))
    ws = torch.empty(chunk * per_view.value, dtype=torch.uint8, device=device)
    rgba = torch.empty(chunk, 4, H, W, device=device)
    for (o, f), idx in groups.items():
        for s in range(0, len(idx), chunk):
            sel = torch.tensor(idx[s:s + chunk], device=device)
            m = len(sel)
            d, b = torch.empty(m, H, W, device=device), torch.empty(m, 4, dtype=torch.int64, device=device)
            render_chunk(meshes_dev[o], poses[sel].contiguous(), K[f].contiguous(), H, W, 0.1 * unit_per_m, ws,
                         rgba[:m], d, b)
            depth[sel], boxes[sel] = d, b
    return depth, boxes


def prepare_scene(depth, K, workspace, unit_per_m=1000.0):
    F, H, W = depth.shape
    check(_lib.load().gp_icp_prepare_scene(F, H, W, depth.data_ptr(), K.data_ptr(), float(unit_per_m),
                                           workspace.data_ptr(), torch.cuda.current_stream(depth.device).cuda_stream))


def workspace_bytes(n_frames, n_hyp, H, W):
    b = C.c_size_t()
    check(_lib.load().gp_icp_query_sizes(n_frames, n_hyp, H, W, C.byref(b)))
    return b.value


def refine_rendered(depth, K, frame_idx, rendered, boxes, poses, masks, workspace, debug=None, **params):
    """gp_icp_refine over n hypotheses whose scene is already in `workspace` -> poses, status, residual, fitness."""
    F, H, W = depth.shape
    n = poses.shape[0]
    p = make_params(debug, **params)
    return _refine_call(_lib.load().gp_icp_refine, (F, n, H, W, frame_idx.data_ptr(), ptr(masks), rendered.data_ptr(),
                                                    boxes.data_ptr(), poses.data_ptr(), K.data_ptr(), C.byref(p)),
                        n, poses.device, torch.float32, workspace)


def _inputs(what, meshes_dev, labels, poses, depth, K, frame_idx):
    """The checked inputs `refine_icp` and `score_hypotheses` share: poses f32 [n,4,4], depth f32 [F,H,W] and K f32
    [F,3,3] on the poses' device, labels and frame_idx i64 [n] on the host."""
    device = poses.device
    if device.type != "cuda":
        raise _lib.GigaPoseNativeError(f"{what} runs on CUDA devices only (no CPU fallback)")
    poses = poses.to(device, torch.float32).reshape(-1, 4, 4).contiguous()
    depth = torch.as_tensor(depth).to(device, torch.float32).contiguous()
    if depth.dim() == 2:
        depth = depth[None]
    F, H, W = depth.shape
    K = torch.as_tensor(K).to(device, torch.float32)
    if tuple(K.shape) not in ((3, 3), (1, 3, 3), (F, 3, 3)):
        raise ValueError(f"K must be [3,3] or one full-image K per frame [{F},3,3], got {tuple(K.shape)}")
    K = K.reshape(-1, 3, 3).expand(F, 3, 3).contiguous()
    n = poses.shape[0]
    labels = torch.as_tensor(labels).reshape(-1).to("cpu", torch.int64)
    frame_idx = torch.as_tensor(frame_idx).reshape(-1).to("cpu", torch.int64)
    if labels.shape[0] != n or frame_idx.shape[0] != n:
        raise ValueError("labels and frame_idx need one entry per pose")
    if n and (int(labels.min()) < 0 or int(labels.max()) >= len(meshes_dev)):
        raise ValueError(f"labels outside [0, {len(meshes_dev)})")
    if n and (int(frame_idx.min()) < 0 or int(frame_idx.max()) >= F):
        raise ValueError(f"frame_idx outside [0, {F})")
    return poses, depth, K, labels, frame_idx


def _chunk(n, per_hyp_bytes, H, W, group=1):
    """Hypotheses per chunk: whole groups of `group` whose renders (52 B per pixel) and `per_hyp_bytes` of scratch
    each fit WORKSPACE_BYTES, at least one group."""
    return group * max(1, min(n // group, WORKSPACE_BYTES // (group * (per_hyp_bytes + 52 * H * W))))


def _render_and_run(meshes_dev, labels, poses, K, frame_idx, H, W, upm, per_hyp_bytes, run, outputs, group=1):
    """Renders the n hypotheses (`_inputs`' layout) chunk by chunk (`_chunk`), calls run(slice, rendered, boxes) on
    each chunk and copies the per-hypothesis tensors it returns into the chunk's rows of `outputs`.  Every result
    depends on its own hypothesis (or group) only, so the chunking changes no output.  -> `outputs`."""
    n = poses.shape[0]
    chunk = _chunk(n, per_hyp_bytes, H, W, group)
    for s in range(0, n, chunk):
        sl = slice(s, min(n, s + chunk))
        rendered, boxes = render_hypotheses(meshes_dev, labels[sl], poses[sl], K, frame_idx[sl], H, W, upm)
        for o, r in zip(outputs, run(sl, rendered, boxes)):
            o[sl] = r
    return outputs


@torch.no_grad()
def refine_icp(meshes_dev, labels, poses, depth, K, frame_idx, masks=None, **params):
    """Refines n hypotheses against the measured depth.

    meshes_dev  list of device meshes (`device_meshes`), indexed by labels [n] (0-based);
    poses       [n,4,4] coarse object -> camera poses, in the depth unit;
    depth       [F,H,W] measured depth (0 = missing), K [F,3,3] full-image intrinsics, frame_idx [n] frame of each;
    masks       None (the reference's threshold rule) or [n,H,W] full-frame detection masks;
    params      see DEFAULTS (unit_per_m = 1000 for mm).
    -> (poses [n,4,4], status [n] i32 (STATUS_NAMES), residual [n], fitness [n]) on the device; a pose whose status is
    not 0 is its input pose bit for bit."""
    upm = float(params.get("unit_per_m", DEFAULTS["unit_per_m"]))
    poses, depth, K, labels, frame_idx = _inputs("refine_icp", meshes_dev, labels, poses, depth, K, frame_idx)
    device = poses.device
    F, H, W = depth.shape
    n = poses.shape[0]
    if masks is not None:
        masks = torch.as_tensor(masks).to(device).reshape(n, H, W).to(torch.uint8).contiguous()
    out = _outputs(n, device, torch.float32)
    if n == 0:
        return out
    scene = workspace_bytes(F, 0, H, W)
    per_hyp = workspace_bytes(F, 1, H, W) - scene
    ws = torch.empty(scene + _chunk(n, per_hyp, H, W) * per_hyp, dtype=torch.uint8, device=device)
    prepare_scene(depth, K, ws, upm)
    fi = frame_idx.to(device, torch.int32)
    return _render_and_run(meshes_dev, labels, poses, K, frame_idx, H, W, upm, per_hyp,
                           lambda sl, rendered, boxes: refine_rendered(depth, K, fi[sl].contiguous(), rendered, boxes,
                                                                       poses[sl], None if masks is None else masks[sl],
                                                                       ws, **params), out)


@torch.no_grad()
def score_hypotheses(meshes_dev, labels, poses, depth, K, frame_idx, n_hyp, tolerance_m=0.015, unit_per_m=1000.0):
    """Depth-consistency score of n = n_det * n_hyp poses (row d * n_hyp + j is hypothesis j of detection d; labels,
    poses, depth, K and frame_idx as `refine_icp` takes them, the hypotheses of a detection sharing one frame): every
    pose is rendered with `render_hypotheses`, the renderer call the ICP's sources come from, and gp_depth_score counts
    the rendered pixels whose measured depth is within `tolerance_m` (VSD's visibility tolerance, 15 mm), behind it, in
    front of it or missing (csrc/depth_score.cu's header comment states the contract).
    -> (counts [n,4] i32 = consistent, behind, front, missing; score [n] = consistent / (consistent + behind + front);
    best [n_det] i32, the hypothesis with the largest score, the lowest index on a tie) on the device."""
    n_hyp = int(n_hyp)
    if n_hyp < 1:
        raise ValueError(f"n_hyp {n_hyp} must be >= 1")
    poses, depth, K, labels, frame_idx = _inputs("score_hypotheses", meshes_dev, labels, poses, depth, K, frame_idx)
    device = poses.device
    F, H, W = depth.shape
    n = poses.shape[0]
    if n % n_hyp:
        raise ValueError(f"{n} poses are not a whole number of groups of {n_hyp} hypotheses")
    if not torch.equal(frame_idx, frame_idx[::n_hyp].repeat_interleave(n_hyp)):
        raise ValueError("the hypotheses of a detection must share one frame")
    counts = torch.empty(n, 4, dtype=torch.int32, device=device)
    score = torch.empty(n, device=device)
    best = torch.empty(n // n_hyp, dtype=torch.int32, device=device)
    fi = frame_idx[::n_hyp].to(device, torch.int32)

    def run(sl, rendered, boxes):                                      # writes the chunk's rows in place
        det = slice(sl.start // n_hyp, sl.stop // n_hyp)
        check(_lib.load().gp_depth_score(F, det.stop - det.start, n_hyp, H, W, fi[det].data_ptr(), depth.data_ptr(),
                                         rendered.data_ptr(), boxes.data_ptr(), float(tolerance_m) * float(unit_per_m),
                                         counts[sl].data_ptr(), score[sl].data_ptr(), best[det].data_ptr(),
                                         torch.cuda.current_stream(device).cuda_stream))
        return ()

    _render_and_run(meshes_dev, labels, poses, K, frame_idx, H, W, unit_per_m, 0, run, (), group=n_hyp)
    return counts, score, best


# ---------------------------------------------------------------------------------------------------- masked normals
def rle_boxes(counts, offsets, H, W):
    """Mask boxes i32 [n,4] (x0, y0, x1, y1, exclusive max; all 0 for an empty mask) of COCO run-length masks, from
    the runs on the host: detection d owns counts[offsets[d]:offsets[d+1]], column-major, the first run counting
    zeros; runs past H * W are cut off."""
    counts = np.asarray(counts, np.int64).reshape(-1)
    off = np.asarray(offsets, np.int64).reshape(-1)
    out = np.zeros((len(off) - 1, 4), np.int32)
    for d in range(len(off) - 1):
        c = counts[off[d]:off[d + 1]]
        ends = np.minimum(np.cumsum(c), H * W)
        starts = np.minimum(ends - c, H * W)
        ones = (np.arange(len(c)) % 2 == 1) & (ends > starts)
        if not ones.any():
            continue
        s, e = starts[ones], ends[ones] - 1                            # first and last pixel of each run of ones
        c0, c1 = s // H, e // H
        r0 = np.where(c1 > c0, 0, s % H)                               # a run over two columns covers rows 0 .. H-1
        r1 = np.where(c1 > c0, H - 1, e % H)
        out[d] = (c0.min(), r0.min(), c1.max() + 1, r1.max() + 1)
    return out


def dense_boxes(masks):
    """Mask boxes i32 [n,4] (as `rle_boxes`) of dense masks [n,H,W] (nonzero = in the mask), on the host."""
    m = torch.as_tensor(masks) != 0
    n, H, W = m.shape
    rows, cols = m.any(2), m.any(1)
    first = lambda a: a.to(torch.int8).argmax(1)                      # noqa: E731  (first True; 0 when none)
    box = torch.stack([first(cols), first(rows), W - first(cols.flip(1)), H - first(rows.flip(1))], 1)
    return torch.where(rows.any(1)[:, None], box, torch.zeros_like(box)).to("cpu", torch.int32).numpy()


class MaskSet:
    """The host description gp_icp_mask_set_t points to (frames, boxes, run offsets), kept alive with it."""

    def __init__(self, frame, boxes, run_offsets=None):
        self.frame = np.ascontiguousarray(np.asarray(frame).reshape(-1), np.int32)
        self.boxes = np.ascontiguousarray(np.asarray(boxes).reshape(-1, 4), np.int32)
        self.run_offsets = None if run_offsets is None else np.ascontiguousarray(np.asarray(run_offsets).reshape(-1),
                                                                                 np.int64)
        if self.boxes.shape[0] != self.frame.shape[0]:
            raise ValueError("one box per detection")
        if self.run_offsets is not None and self.run_offsets.shape[0] != self.frame.shape[0] + 1:
            raise ValueError(f"run offsets need n_det + 1 = {self.frame.shape[0] + 1} entries")
        i32 = C.POINTER(C.c_int32)
        self.c = GpIcpMaskSet(len(self.frame), self.frame.ctypes.data_as(i32), self.boxes.ctypes.data_as(i32),
                              None if self.run_offsets is None else self.run_offsets.ctypes.data_as(C.POINTER(C.c_int64)))

    def __len__(self):
        return len(self.frame)

    def query(self, F, H, W, offsets=False):
        """-> (scene workspace bytes, box_pixels), and with `offsets` the byte offsets of the tiles and the maps."""
        b, px, t0, m0 = C.c_size_t(), C.c_int64(), C.c_size_t(), C.c_size_t()
        check(_lib.load().gp_icp_masked_query_sizes(F, H, W, C.byref(self.c), C.byref(b), C.byref(px), C.byref(t0),
                                                    C.byref(m0)))
        return (b.value, px.value, t0.value, m0.value) if offsets else (b.value, px.value)

    def tiles(self, workspace, F, H, W):
        """Per detection, views (mask u8 [h,w], map f32 [h,w,6]) of its box in a decoded and prepared workspace."""
        area = (self.boxes[:, 2] - self.boxes[:, 0]).astype(np.int64) * (self.boxes[:, 3] - self.boxes[:, 1])
        start = np.concatenate([[0], np.cumsum(area)])
        _, _, t0, m0 = self.query(F, H, W, offsets=True)
        maps = workspace[m0:m0 + int(start[-1]) * 24].view(torch.float32)
        out = []
        for d, (x0, y0, x1, y1) in enumerate(self.boxes.tolist()):
            h, w = max(y1 - y0, 0), max(x1 - x0, 0)
            a, b = int(start[d]), int(start[d + 1])
            out.append((workspace[t0 + a:t0 + b].reshape(h, w), maps[6 * a:6 * b].reshape(h, w, 6)))
        return out


def masked_scene(depth, K, det_frame, masks=None, rle=None, unit_per_m=1000.0):
    """Decodes the detections' masks into box tiles and prepares their masked target maps (gp_icp_masked_decode +
    gp_icp_prepare_masked_scene).  depth f32 [F,H,W] and K f32 [F,3,3] on the device, det_frame [n_det] frame of each
    detection; masks dense [n_det,H,W] (device) or rle = (counts i32, offsets [n_det+1]) (host or device counts, host
    offsets).  -> (workspace u8, MaskSet, box_pixels)."""
    F, H, W = depth.shape
    dev = depth.device
    if (masks is None) == (rle is None):
        raise ValueError("give either dense masks or rle = (counts, offsets)")
    stream = torch.cuda.current_stream(dev).cuda_stream
    n = len(np.asarray(det_frame).reshape(-1))
    if masks is not None:
        masks = torch.as_tensor(masks).to(dev)
        if tuple(masks.shape) != (n, H, W):
            raise ValueError(f"dense masks must be [{n},{H},{W}], got {tuple(masks.shape)}")
        masks = (masks != 0).to(torch.uint8).contiguous()
        ms, counts = MaskSet(det_frame, dense_boxes(masks)), None
    else:
        counts, off = rle
        off = np.asarray(off, np.int64).reshape(-1)
        counts = torch.as_tensor(np.asarray(counts) if not torch.is_tensor(counts) else counts,
                                 dtype=torch.int32).reshape(-1)
        if off.shape != (n + 1,) or counts.numel() < off[-1]:
            raise ValueError(f"rle offsets must have n_det + 1 = {n + 1} entries within the {counts.numel()} counts")
        ms = MaskSet(det_frame, rle_boxes(counts.cpu().numpy(), off, H, W), off)
        counts = counts.to(dev, non_blocking=True).contiguous()
    nbytes, box_pixels = ms.query(F, H, W)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    lib = _lib.load()
    check(lib.gp_icp_masked_decode(F, H, W, C.byref(ms.c), ptr(masks), ptr(counts), ws.data_ptr(), stream))
    check(lib.gp_icp_prepare_masked_scene(F, H, W, C.byref(ms.c), depth.data_ptr(), K.data_ptr(), float(unit_per_m),
                                          ws.data_ptr(), stream))
    return ws, ms, box_pixels


def refine_rendered_masked(ms, scene_ws, box_pixels, depth, K, det_idx, rendered, boxes, poses, debug=None, **params):
    """gp_icp_refine_masked over n hypotheses against a prepared masked scene -> poses, status, residual, fitness."""
    F, H, W = depth.shape
    n = poses.shape[0]
    scratch = torch.empty(max(n * box_pixels * 12, 1), dtype=torch.uint8, device=poses.device)
    p = make_params(debug, **params)
    return _refine_call(_lib.load().gp_icp_refine_masked,
                        (F, H, W, C.byref(ms.c), n, det_idx.data_ptr(), rendered.data_ptr(), boxes.data_ptr(),
                         poses.data_ptr(), K.data_ptr(), C.byref(p)), n, poses.device, torch.float32, scene_ws, scratch)


@torch.no_grad()
def refine_icp_masked(meshes_dev, labels, poses, depth, K, det_frame, det_idx, masks=None, rle=None, **params):
    """`refine_icp` with target normals smoothed within each detection's mask (row f11, csrc/depth_icp.cu 1'-2').

    det_frame [n_det] frame of each detection; det_idx [n] detection of each hypothesis (the hypotheses of a detection
    share its map: no mask is copied per hypothesis); masks dense [n_det,H,W] or rle = (counts, offsets [n_det+1]) of
    COCO run-length masks (bop_run's layout).  The rest as `refine_icp` -> (poses, status, residual, fitness)."""
    upm = float(params.get("unit_per_m", DEFAULTS["unit_per_m"]))
    det_frame = np.asarray(torch.as_tensor(det_frame).cpu(), np.int64).reshape(-1)
    det_idx = np.asarray(torch.as_tensor(det_idx).cpu(), np.int64).reshape(-1)
    if len(det_idx) and (det_idx.min() < 0 or det_idx.max() >= len(det_frame)):
        raise ValueError(f"det_idx outside [0, {len(det_frame)})")
    poses, depth, K, labels, frame_idx = _inputs("refine_icp_masked", meshes_dev, labels, poses, depth, K,
                                                 det_frame[det_idx])
    device = poses.device
    F, H, W = depth.shape
    n = poses.shape[0]
    out = _outputs(n, device, torch.float32)
    if n == 0:
        return out
    ws, ms, box_pixels = masked_scene(depth, K, det_frame, masks, rle, upm)
    di = torch.as_tensor(det_idx, dtype=torch.int32).to(device)
    return _render_and_run(meshes_dev, labels, poses, K, frame_idx, H, W, upm, box_pixels * 12,
                           lambda sl, rendered, boxes: refine_rendered_masked(
                               ms, ws, box_pixels, depth, K, di[sl].contiguous(), rendered, boxes, poses[sl], **params),
                           out)
