"""Depth refinement with MegaPose's TeaserppRefiner on the GPU (row f13; src/megapose/inference/teaserpp_refiner.py):
every hypothesis is rendered at its pose with the frame's K (`icp.render_hypotheses`), the pixels where both the render
and the measured depth are positive become pixel-aligned correspondences, farthest-point sampled, and
gp_teaser_refine keeps an exact maximum clique of the pairwise-consistent ones and solves rotation (GNC-TLS) and
translation (adaptive voting) on them.  csrc/depth_teaser.cu's header comment states the contract; INTEGRATION.md
lists the deviations.  `REFINERS` names every depth refiner."""
from __future__ import annotations

import ctypes as C
from typing import Callable, NamedTuple

import torch

from . import _lib, icp
from ._lib import GpTeaserDebug, GpTeaserParams, check
from .icp import _inputs, _outputs, _params, _refine_call, _render_and_run

STATUS_NAMES = {_lib.TEASER_OK: "ok", _lib.TEASER_TOO_FEW_POINTS: "too few points",
                _lib.TEASER_CLIQUE_TOO_SMALL: "clique too small", _lib.TEASER_CLIQUE_BUDGET: "clique budget",
                _lib.TEASER_TOO_FEW_INLIERS: "too few inliers", _lib.TEASER_INVALID: "invalid frame index"}
DEFAULTS = dict(unit_per_m=1000.0, min_points=100, n_points=1000, noise_bound=0.01, cbar2=1.0, min_inliers=50,
                gnc_factor=1.4, gnc_max_iters=100, gnc_cost_threshold=1e-12, clique_budget=20000)


def make_params(debug=None, **params) -> GpTeaserParams:
    return _params(GpTeaserParams, GpTeaserDebug, DEFAULTS, "TEASER++", debug, params)


def workspace_bytes(n_hyp, H, W):
    b = C.c_size_t()
    check(_lib.load().gp_teaser_query_sizes(n_hyp, H, W, C.byref(b)))
    return b.value


def refine_rendered(depth, K, frame_idx, rendered, boxes, poses, debug=None, **params):
    """gp_teaser_refine over n hypotheses already rendered -> poses, status, inliers, clique (device)."""
    F, H, W = depth.shape
    n = poses.shape[0]
    _, ws = _lib.aligned_buffer(workspace_bytes(n, H, W), poses.device)
    p = make_params(debug, **params)
    return _refine_call(_lib.load().gp_teaser_refine, (F, n, H, W, frame_idx.data_ptr(), depth.data_ptr(),
                                                       rendered.data_ptr(), boxes.data_ptr(), poses.data_ptr(),
                                                       K.data_ptr(), C.byref(p)), n, poses.device, torch.int32, ws)


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
    out = _outputs(n, device, torch.int32)
    if n == 0:
        return out
    make_params(**params)                                              # unknown names fail before any GPU work
    fi = frame_idx.to(device, torch.int32)
    return _render_and_run(meshes_dev, labels, poses, K, frame_idx, H, W, upm,
                           workspace_bytes(2, H, W) - workspace_bytes(1, H, W),
                           lambda sl, rendered, boxes: refine_rendered(depth, K, fi[sl].contiguous(), rendered, boxes,
                                                                       poses[sl], **params), out)


class Refiner(NamedTuple):
    refine: Callable            # (meshes_dev, labels, poses, depth, K, frame_idx, **params) -> (poses, status, a, b)
    defaults: dict              # its params
    masks: bool                 # whether it takes detection masks
    outputs: tuple              # the names `GigaPose.refine_depth` gives status, a and b


# Every depth refiner of `GigaPose.refine_depth(refiner=)` and `bop_run --depth-refiner`.
REFINERS = {"icp": Refiner(icp.refine_icp, icp.DEFAULTS, True, ("icp_status", "icp_residual", "icp_fitness")),
            "teaserpp": Refiner(refine_teaserpp, DEFAULTS, False, ("teaser_status", "teaser_inliers", "teaser_clique"))}
