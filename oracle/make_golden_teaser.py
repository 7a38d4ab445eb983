"""TEST INFRASTRUCTURE ONLY -- regenerates tests/golden/teaser_scenes.npz by running the UNMODIFIED reference
`TeaserppRefiner.refine_poses` and `compute_teaserpp_refinement` (src/megapose/inference/teaserpp_refiner.py:53-291;
build container only) on seeded scenes in metres.  The pieces that are not installed are replaced:
- the renderer returns the planted depth render of each prediction;
- `teaserpp_python` is a recorder: it keeps the [3,N] clouds `solve` receives and returns a planted R, t;
- `pytorch3d.ops.sample_farthest_points` returns planted indices, padded with -1 past the masked count as pytorch3d
  documents, so the reference's own indexing decides what the padding becomes;
- `open3d` (the inlier count's transform) is a numpy PointCloud, and meshcat, trimesh, transforms3d and panda3d are
  empty modules.
The fixture pins the mask counts, the masked clouds, the sampled clouds (with the reference's padding), the skip below
n_min_points, the inlier count and the accepted pose.

    python -m oracle.make_golden_teaser
"""
from __future__ import annotations

import os
import types

import numpy as np
import torch

from . import ref_import, teaser_port

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "teaser_scenes.npz")
H, W = 48, 64
K = np.array([[90.0, 0.0, 31.3], [0.0, 92.5, 23.7], [0.0, 0.0, 1.0]], np.float32)


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    return m


class _PointCloud:
    def __init__(self):
        self.points = None

    def transform(self, T):
        self.points = np.asarray(self.points, np.float64) @ np.asarray(T)[:3, :3].T + np.asarray(T)[:3, 3]
        return self


class _Solver:
    """Stands in for teaserpp_python.RobustRegistrationSolver: records solve's clouds, returns the planted R, t."""
    calls, planted = [], None

    class Params:
        pass

    class ROTATION_ESTIMATION_ALGORITHM:
        GNC_TLS = "GNC_TLS"

    def __init__(self, params):
        self.params = params

    def solve(self, src, tgt):
        _Solver.calls.append((np.array(src), np.array(tgt), dict(vars(self.params))))

    def getSolution(self):
        R, t = _Solver.planted
        return types.SimpleNamespace(rotation=R, translation=t)


class _Sampler:
    """pytorch3d.ops.sample_farthest_points stand-in: the planted indices of the current prediction, -1 past N."""
    planted = []

    @staticmethod
    def sample_farthest_points(x, lengths, K):
        idx = np.full(K, -1, np.int64)
        got = _Sampler.planted.pop(0)[:K]
        idx[:len(got)] = got
        return None, torch.as_tensor(idx)[None]


def _stubs():
    cls = lambda name: type(name, (), {})                              # noqa: E731
    p3d_ops = _mod("pytorch3d.ops", sample_farthest_points=_Sampler.sample_farthest_points)
    return {
        "teaserpp_python": _mod("teaserpp_python", RobustRegistrationSolver=_Solver),
        "pytorch3d": _mod("pytorch3d", ops=p3d_ops), "pytorch3d.ops": p3d_ops,
        "open3d": _mod("open3d", geometry=_mod("open3d.geometry", PointCloud=_PointCloud),
                       utility=_mod("open3d.utility", Vector3dVector=lambda a: np.asarray(a, np.float64))),
        "transforms3d": _mod("transforms3d"), "trimesh": _mod("trimesh"),
        "trimesh.transformations": _mod("trimesh.transformations"),
        "meshcat": _mod("meshcat"), "meshcat.geometry": _mod("meshcat.geometry"),
        "meshcat.transformations": _mod("meshcat.transformations"), "panda3d": _mod("panda3d"),
        "src.megapose.inference.depth_refiner": _mod("src.megapose.inference.depth_refiner",
                                                     DepthRefiner=cls("DepthRefiner")),
        "src.megapose.inference.types": _mod("src.megapose.inference.types", PoseEstimatesType=object),
        "src.megapose.lib3d.rigid_mesh_database": _mod("src.megapose.lib3d.rigid_mesh_database",
                                                       BatchedMeshes=cls("BatchedMeshes")),
        "src.megapose.panda3d_renderer.panda3d_batch_renderer": _mod(
            "src.megapose.panda3d_renderer.panda3d_batch_renderer", Panda3dBatchRenderer=cls("Panda3dBatchRenderer")),
        "src.megapose.panda3d_renderer.types": _mod("src.megapose.panda3d_renderer.types",
                                                    Panda3dLightData=lambda *a, **k: None),
    }


class _Renderer:
    def __init__(self, depths):
        self.depths = depths

    def render(self, labels, TCO, K, light_datas, resolution, render_depth):
        return types.SimpleNamespace(depths=torch.as_tensor(self.depths)[:, None])


class _Predictions:
    """The slice of PandasTensorCollection refine_poses touches: infos, poses, poses_input, len, clone."""

    def __init__(self, infos, poses):
        self.infos, self.poses, self.poses_input = infos, poses, poses.clone()

    def __len__(self):
        return len(self.poses)

    def clone(self):
        return _Predictions(self.infos.copy(), self.poses.clone())


def make_scene(seed, n_keep=None, far=False):
    """Metres.  Rendered: a bumped surface inside a box; measured: the same surface 4 mm deeper with 15 % outliers
    20-60 mm off and 5 % holes.  n_keep cuts the render to its first n_keep masked pixels in row-major order."""
    rng = np.random.default_rng(seed)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    z = 0.7 + 0.0004 * (u - 32) + 0.01 * np.sin(u / 6.0) * np.cos(v / 5.0)
    R = np.zeros((H, W), np.float32)
    x0, y0 = rng.integers(2, 12, 2)
    R[y0:y0 + 36, x0:x0 + 48] = z[y0:y0 + 36, x0:x0 + 48]
    D = (z + 0.004 + np.where(rng.random((H, W)) < 0.15, rng.uniform(0.02, 0.06, (H, W)), 0)).astype(np.float32)
    D[rng.random((H, W)) < 0.05] = 0
    if n_keep is not None:
        ys, xs = np.nonzero((R > 0) & (D > 0))
        cut = np.zeros_like(R)
        cut[ys[:n_keep], xs[:n_keep]] = R[ys[:n_keep], xs[:n_keep]]
        R = cut
    a = np.deg2rad(0.8 if not far else 25.0)
    Rp = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    tp_ = np.array([0.001, -0.002, 0.004]) if not far else np.array([0.05, 0.04, 0.03])
    T0 = np.eye(4, dtype=np.float32)
    Q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    T0[:3, :3] = Q * np.sign(np.linalg.det(Q))
    T0[:3, 3] = (0.02, -0.01, 0.7)
    return D, R, T0, Rp, tp_


CASES = {"full": dict(seed=1), "padded": dict(seed=2, n_keep=400), "skip": dict(seed=3, n_keep=99),
         "rejected": dict(seed=4, far=True)}


def main():
    with ref_import._ReferenceImports(extra_stubs=_stubs()) as ctx:
        mod = ctx.import_reference("src.megapose.inference.teaserpp_refiner")
    import sys
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self                      # the reference moves FPS inputs to the GPU
    lazy = {k: v for k, v in _stubs().items() if k.startswith("pytorch3d")}   # imported inside the function
    sys.modules.update(lazy)
    try:
        import pandas as pd
        arrays = {"K": K}
        for case, kw in CASES.items():
            D, R, T0, Rp, tp_ = make_scene(**kw)
            src, _ = teaser_port.points(D, R, (0, 0, W, H), K)
            order = teaser_port.fps(src, min(1000, len(src))) if len(src) else np.zeros(0, np.int64)
            _Solver.calls.clear()
            _Solver.planted = (Rp, tp_)
            # compute_teaserpp_refinement alone (the clouds, the sampled clouds, the inlier count)
            mask = (D > 0) & (R > 0)
            out = None
            if mask.sum() >= 100:
                _Sampler.planted = [order]
                out = mod.compute_teaserpp_refinement(depth_src=R, depth_tgt=D, mask=mask, cam_K=K,
                                                      max_num_points=1000, noise_bound=0.01)
            # refine_poses end to end
            _Sampler.planted = [order]
            ref = mod.TeaserppRefiner(None, _Renderer(R[None]))
            preds = _Predictions(pd.DataFrame(dict(label=["obj"], batch_im_id=[0])), torch.as_tensor(T0[None]))
            refined, _ = ref.refine_poses(preds, depth=torch.as_tensor(D[None]), K=torch.as_tensor(K[None]))
            arrays.update({f"{case}_depth": D, f"{case}_rendered": R, f"{case}_T0": T0, f"{case}_R": Rp,
                           f"{case}_t": tp_, f"{case}_fps": order, f"{case}_mask_count": np.int64(mask.sum()),
                           f"{case}_pose": refined.poses[0].numpy().astype(np.float32)})
            if out is not None:
                arrays.update({f"{case}_pc_src_mask": out["pc_src_mask"], f"{case}_pc_tgt_mask": out["pc_tgt_mask"],
                               f"{case}_pc_src": out["pc_src"], f"{case}_pc_tgt": out["pc_tgt"],
                               f"{case}_num_inliers": np.int64(out["num_inliers"]),
                               f"{case}_solver_src": _Solver.calls[0][0]})
            print(f"{case}: {int(mask.sum())} masked, inliers {None if out is None else out['num_inliers']}, "
                  f"accepted {not np.array_equal(arrays[f'{case}_pose'], T0)}")
    finally:
        torch.Tensor.cuda = cuda
        for k in lazy:
            sys.modules.pop(k, None)
    np.savez_compressed(GOLDEN, **arrays)
    print(f"wrote {GOLDEN}")


if __name__ == "__main__":
    main()
