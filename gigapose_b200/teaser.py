"""Depth refinement with MegaPose's TeaserppRefiner on the GPU (row f13; src/megapose/inference/teaserpp_refiner.py):
every hypothesis is rendered at its pose with the frame's K (`icp.render_hypotheses`), the pixels where both the render
and the measured depth are positive become pixel-aligned correspondences, farthest-point sampled, and
gp_teaser_refine keeps an exact maximum clique of the pairwise-consistent ones and solves rotation (GNC-TLS) and
translation (adaptive voting) on them.  csrc/depth_teaser.cu's header comment states the contract; INTEGRATION.md
lists the deviations."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import GpTeaserDebug, GpTeaserParams, check, ptr
from .icp import _inputs, render_hypotheses

STATUS_NAMES = {_lib.TEASER_OK: "ok", _lib.TEASER_TOO_FEW_POINTS: "too few points",
                _lib.TEASER_CLIQUE_TOO_SMALL: "clique too small", _lib.TEASER_CLIQUE_BUDGET: "clique budget",
                _lib.TEASER_TOO_FEW_INLIERS: "too few inliers", _lib.TEASER_INVALID: "invalid frame index"}
DEFAULTS = dict(unit_per_m=1000.0, min_points=100, n_points=1000, noise_bound=0.01, cbar2=1.0, min_inliers=50,
                gnc_factor=1.4, gnc_max_iters=100, gnc_cost_threshold=1e-12, clique_budget=20000)
WORKSPACE_BYTES = 1 << 30          # renders + TEASER scratch per chunk of hypotheses


def make_params(debug=None, **params) -> GpTeaserParams:
    unknown = set(params) - set(DEFAULTS)
    if unknown:
        raise TypeError(f"unknown TEASER++ parameters {sorted(unknown)}")
    p = GpTeaserParams(**dict(DEFAULTS, **params))
    if debug:
        p.debug = GpTeaserDebug(**{k: v if isinstance(v, int) else ptr(v) for k, v in debug.items()})
    return p


def workspace_bytes(n_hyp, H, W):
    b = C.c_size_t()
    check(_lib.load().gp_teaser_query_sizes(n_hyp, H, W, C.byref(b)))
    return b.value


def refine_rendered(depth, K, frame_idx, rendered, boxes, poses, debug=None, **params):
    """gp_teaser_refine over n hypotheses already rendered -> poses, status, inliers, clique (device)."""
    F, H, W = depth.shape
    n = poses.shape[0]
    dev = poses.device
    out = torch.empty(n, 4, 4, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    inliers = torch.empty(n, dtype=torch.int32, device=dev)
    clique = torch.empty(n, dtype=torch.int32, device=dev)
    ws = torch.empty(workspace_bytes(n, H, W) + 1024, dtype=torch.uint8, device=dev)
    ws = ws[(-ws.data_ptr()) % 1024:]
    p = make_params(debug, **params)
    check(_lib.load().gp_teaser_refine(F, n, H, W, frame_idx.data_ptr(), depth.data_ptr(), rendered.data_ptr(),
                                       boxes.data_ptr(), poses.data_ptr(), K.data_ptr(), C.byref(p), out.data_ptr(),
                                       status.data_ptr(), inliers.data_ptr(), clique.data_ptr(), ws.data_ptr(),
                                       torch.cuda.current_stream(dev).cuda_stream))
    return out, status, inliers, clique


@torch.no_grad()
def refine_teaserpp(meshes_dev, labels, poses, depth, K, frame_idx, **params):
    """Refines n hypotheses against the measured depth with the TEASER++ refiner.

    meshes_dev, labels, poses, depth, K and frame_idx as `icp.refine_icp` takes them; params see DEFAULTS (metre
    parameters are scaled by unit_per_m = 1000 for mm; clique_budget bounds the clique search, which the reference
    does not).  -> (poses [n,4,4], status [n] i32 (STATUS_NAMES), inliers [n] i32, clique [n] i32) on the device; a
    pose whose status is not 0 is its input pose bit for bit."""
    upm = float(params.get("unit_per_m", DEFAULTS["unit_per_m"]))
    poses, depth, K, labels, frame_idx = _inputs("refine_teaserpp", meshes_dev, labels, poses, depth, K, frame_idx)
    device = poses.device
    F, H, W = depth.shape
    n = poses.shape[0]
    out = poses.clone()
    status = torch.empty(n, dtype=torch.int32, device=device)
    inliers = torch.empty(n, dtype=torch.int32, device=device)
    clique = torch.empty(n, dtype=torch.int32, device=device)
    if n == 0:
        return out, status, inliers, clique
    make_params(**params)                                              # unknown names fail before any GPU work
    per_hyp = workspace_bytes(2, H, W) - workspace_bytes(1, H, W)
    chunk = max(1, min(n, WORKSPACE_BYTES // (per_hyp + 52 * H * W)))
    fi = frame_idx.to(device, torch.int32)
    for s in range(0, n, chunk):
        sl = slice(s, min(n, s + chunk))
        rendered, boxes = render_hypotheses(meshes_dev, labels[sl], poses[sl], K, frame_idx[sl], H, W, upm)
        o = refine_rendered(depth, K, fi[sl].contiguous(), rendered, boxes, poses[sl], **params)
        out[sl], status[sl], inliers[sl], clique[sl] = o
    return out, status, inliers, clique
