"""The rasteriser's kernels against an fp64 ray caster (tests/render_fp64.py): gp_render_templates through
render.render_chunk (per-sample keys from its workspace, RGBA, depth, boxes) and gp_render_depth through
bop_eval.render_depth, at 480 x 640 with the template camera, 1080 x 1920 (depth only, the HOPE frame) and 37 x 53.
The bars and their derivations are those of tests/test_render_fp64_cpu.py, which runs the same comparisons on the CPU
port; six mutated definitions of the renderer must each fail clearly against the same kernel output.  The measured
worst ratios, excluded fractions and mutation margins are printed (pytest -s) for DESIGN.md."""
import json

import numpy as np
import pytest
import torch

from gigapose_b200 import bop_eval, icp, render

import render_fp64 as rf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCENES = rf.scenes(full=True)
_OUT, _CASTS = {}, {}


def _kernel(name):
    """All views of a scene in one call, so that the per-view offsets are exercised."""
    if name in _OUT:
        return _OUT[name]
    s = SCENES[name]
    n, H, W = len(s["poses"]), s["H"], s["W"]
    poses = torch.as_tensor(s["poses"], dtype=torch.float32, device=DEV).contiguous()
    K = torch.as_tensor(s["K"], dtype=torch.float32, device=DEV).contiguous()
    depth = torch.full((n, H, W), float("nan"), device=DEV)
    boxes = torch.full((n, 4), -7, dtype=torch.int64, device=DEV)
    if s["mode"] == "templates":
        ws = torch.empty(n * H * W * 4, dtype=torch.int64, device=DEV)
        rgba = torch.full((n, 4, H, W), float("nan"), device=DEV)
        render.render_chunk(render._device_mesh(s["mesh"], DEV), poses, K, H, W, s["z_near"], ws, rgba, depth, boxes)
        keys = ws.cpu().numpy().view(np.uint64).reshape(n, H, W, 4)
        rgba = rgba.cpu().numpy()
    else:
        ws = torch.empty(n * H * W, dtype=torch.int64, device=DEV)
        bop_eval.render_depth(icp.device_meshes([s["mesh"]], DEV)[0], poses, K, H, W, s["z_near"], ws, depth, boxes)
        keys = ws.cpu().numpy().view(np.uint64).reshape(n, H, W, 1)
    torch.cuda.synchronize()
    depth, boxes = depth.cpu().numpy(), boxes.cpu().numpy()
    _OUT[name] = [dict(keys=keys[v], depth=depth[v], box=boxes[v], **({"rgba": rgba[v]} if s["mode"] == "templates" else {}))
                  for v in range(n)]
    return _OUT[name]


@pytest.mark.parametrize("name", list(SCENES))
def test_kernel_matches_the_fp64_ray_caster_within_the_bars(name):
    rep, casts = rf.check_scene(SCENES[name], _kernel(name), cache=_CASTS)
    print("fp64-gpu", name, json.dumps(rep))
    rf.assert_within_bars(name, rep)
    if name.startswith("clipped"):
        rf.clipped_scene_is_exercised(SCENES[name], casts)


@pytest.mark.parametrize("mutation,name,which", rf.MUTATION_CASES)
def test_a_mutated_definition_fails_clearly_against_the_kernel(mutation, name, which):
    rep, _ = rf.check_scene(SCENES[name], _kernel(name), mutation, cache=_CASTS)
    n, worst = rf.assert_mutation_fails(name, mutation, rep, which)
    print("fp64-gpu-mutation", mutation, name, json.dumps(dict(fail=n, worst=worst)))
