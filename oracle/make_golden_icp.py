"""TEST INFRASTRUCTURE ONLY -- regenerates tests/golden/icp_scenes.npz by running the UNMODIFIED reference
`icp_refinement` (/root/reference/src/megapose/inference/icp_refiner.py:112-200; build container only) on seeded
hole-free scenes with an integer principal point, where its int16 truncation of u - cx and its cv2.inpaint are no-ops.
OpenCV's `ppf_match_3d_ICP` is replaced by a stub that records the two point sets it is given and returns the identity,
so the fixture pins stages 2-6 (target and source sets, points, target normals, counts, centroid shift) to the
reference itself.  Needs scipy and OpenCV (cv2.inpaint); the unused imports (panda3d, open3d, transforms3d, trimesh,
the megapose config) are stubbed.

    python -m oracle.make_golden_icp
"""
from __future__ import annotations

import os
import types

import numpy as np

from . import ref_import

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "icp_scenes.npz")
H, W = 96, 128
K = np.array([[300.0, 0.0, 64.0], [0.0, 310.0, 48.0], [0.0, 0.0, 1.0]], np.float32)


def _stubs():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m
    cls = lambda name: type(name, (), {})
    return {
        "src.megapose.config": mod("src.megapose.config", DEBUG_DATA_DIR="/nonexistent"),
        "src.megapose.inference.depth_refiner": mod("src.megapose.inference.depth_refiner", DepthRefiner=cls("DepthRefiner")),
        "src.megapose.inference.types": mod("src.megapose.inference.types", PoseEstimatesType=object),
        "src.megapose.lib3d.rigid_mesh_database": mod("src.megapose.lib3d.rigid_mesh_database",
                                                      BatchedMeshes=cls("BatchedMeshes")),
        "src.megapose.panda3d_renderer.panda3d_batch_renderer": mod(
            "src.megapose.panda3d_renderer.panda3d_batch_renderer", Panda3dBatchRenderer=cls("Panda3dBatchRenderer")),
        "src.megapose.panda3d_renderer.types": mod("src.megapose.panda3d_renderer.types",
                                                   Panda3dLightData=cls("Panda3dLightData")),
        "open3d": mod("open3d"), "transforms3d": mod("transforms3d"), "trimesh": mod("trimesh"),
        "panda3d": mod("panda3d"),
    }


class _RecordingICP:
    """Stands in for cv2.ppf_match_3d_ICP: records registerModelToScene's inputs, returns (0, 0.0, identity)."""
    calls = []

    def __init__(self, *args, **kwargs):
        pass

    def registerModelToScene(self, src, tgt):
        _RecordingICP.calls.append((np.array(src, np.float32), np.array(tgt, np.float32)))
        return 0, 0.0, np.eye(4)


def make_scene(seed):
    """Metres.  Measured depth: a tilted background plane with a smooth bump (the object) and a strip beyond 5 m;
    rendered depth: the object's region, offset and tilted against the measurement, with a patch more than 0.1 m off."""
    rng = np.random.default_rng(seed)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    cu, cv = rng.uniform(50, 78), rng.uniform(38, 58)
    ru, rv = rng.uniform(26, 34), rng.uniform(20, 26)
    r2 = ((u - cu) / ru) ** 2 + ((v - cv) / rv) ** 2
    plane = 1.1 + 0.002 * (u - 64) - 0.0015 * (v - 48)
    bump = 0.25 * np.exp(-1.5 * r2) + 0.02 * np.sin(u / 7.0) * np.cos(v / 9.0)
    D = np.where(r2 < 1, plane - bump, plane)
    D[:, -6:] = 5.5                                                     # out of (0.2, 5) m, still not a hole
    D = D.astype(np.float32)
    obj = r2 < rng.uniform(0.85, 1.1)
    R = np.where(obj, D + 0.01 + 0.0004 * (u - cu), 0).astype(np.float32)
    R[int(cv) - 4:int(cv) + 4, int(cu) - 12:int(cu) - 4] += np.float32(0.15)   # fails the threshold rule
    mask = r2 < 1
    T0 = np.eye(4, dtype=np.float32)
    Q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    T0[:3, :3] = Q * np.sign(np.linalg.det(Q))                         # a rotation (det +1)
    T0[:3, 3] = ((cu - 64) / 300 * 0.9, (cv - 48) / 310 * 0.9, 0.95)
    return D, R, mask, T0


def main():
    stubs = _stubs()
    with ref_import._ReferenceImports(extra_stubs=stubs) as ctx:
        icp_mod = ctx.import_reference("src.megapose.inference.icp_refiner")
        utils = ctx.import_reference("src.megapose.inference.refiner_utils")
    import cv2
    icp_mod.cv2 = types.SimpleNamespace(inpaint=cv2.inpaint, INPAINT_NS=cv2.INPAINT_NS,
                                        ppf_match_3d_ICP=_RecordingICP)
    # the reference hands its result back with torch.tensor(...).cuda(); keep it in numpy here
    icp_mod.torch = types.SimpleNamespace(float32=np.float32,
                                          tensor=lambda x, dtype=None: types.SimpleNamespace(cuda=lambda: np.asarray(x)))
    arrays = {"K": K}
    for case, (seed, rule) in {"mask": (11, "mask"), "threshold": (12, "threshold")}.items():
        D, R, mask, T0 = make_scene(seed)
        if rule == "threshold":                                       # ICPRefiner.refine_poses without masks
            _, mask = utils.compute_masks(mask_type="threshold", depth_rendered=R, depth_measured=D,
                                          depth_delta_thresh=0.1)
        _RecordingICP.calls.clear()
        pose, retval = icp_mod.icp_refinement(D, R, mask, K, T0, n_min_points=1000)
        assert retval == 0 and len(_RecordingICP.calls) == 1, (case, retval)
        src, tgt = _RecordingICP.calls[0]
        arrays.update({f"{case}_depth": D, f"{case}_rendered": R, f"{case}_mask": np.asarray(mask, bool),
                       f"{case}_T0": T0, f"{case}_src": src, f"{case}_tgt": tgt,
                       f"{case}_counts": np.array([len(tgt), len(src)], np.int64),
                       f"{case}_pose_shifted": np.asarray(pose, np.float32)})
        print(f"{case}: {len(tgt)} targets, {len(src)} sources")
    np.savez_compressed(GOLDEN, **arrays)
    print(f"wrote {GOLDEN}")


if __name__ == "__main__":
    main()
