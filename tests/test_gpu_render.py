"""Row f5 on the GPU: `gp_render_templates` (csrc/render.cu) against the numpy restatement oracle/render_port.py on
seeded procedural meshes, bit for bit: the per-sample keys (winning face id and depth), RGBA after the 8-bit
quantisation, depth and boxes.  Then onboarding from meshes against onboarding from the same renders, and retrieval
of a rendered query."""
import numpy as np
import pandas as pd
import pytest
import torch

from gigapose_b200 import render, synth
from oracle import render_port as rp
from render_fp64 import icosphere
from render_fp64 import uv_sphere as _uv_sphere

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K_FULL = np.array(render.TEMPLATE_K, np.float32)
K_QUARTER = np.array([[K_FULL[0, 0] / 4, 0, K_FULL[0, 2] / 4], [0, K_FULL[1, 1] / 4, K_FULL[1, 2] / 4], [0, 0, 1]],
                     np.float32)


def meshes():
    rng = np.random.default_rng(11)
    V, Fc = icosphere(3, 60.0, rng)
    colour = dict(vertices=V, faces=Fc, vertex_color=rng.uniform(0, 1, (len(V), 3)).astype(np.float32))
    textured = dict(vertices=V, faces=Fc, face_uv=_uv_sphere(V, Fc, 3.0),
                    texture=rng.uniform(0, 1, (37, 53, 3)).astype(np.float32))
    # two screen-filling triangles behind 20 000 sub-pixel ones (constant colour)
    big = np.array([[-3000, -3000, 300], [3000, -3000, 300], [0, 3000, 300]], np.float32)
    c = rng.uniform(-40, 40, (20000, 1, 3)) + rng.uniform(-0.08, 0.08, (20000, 3, 3))
    tiny = np.concatenate([big, np.array([[-3000, 3000, 310], [3000, 3000, 310], [0, -3000, 310]], np.float32),
                           c.reshape(-1, 3).astype(np.float32)])
    huge_tiny = dict(vertices=tiny, faces=np.arange(len(tiny), dtype=np.int32).reshape(-1, 3),
                     constant_color=np.float32([0.2, 0.7, 0.4]))
    # z-fighting: the same quad twice (separate vertices, identical coordinates), listed in other corner orders
    q = np.array([[-30, -30, 0], [30, -30, 0], [30, 30, 0], [-30, 30, 0]], np.float32)
    zf = dict(vertices=np.concatenate([q, q]), faces=np.array([[6, 5, 4], [0, 1, 2], [4, 6, 7], [3, 0, 2], [1, 2, 0]],
                                                              np.int32),
              vertex_color=np.concatenate([np.tile([1, 0, 0], (4, 1)), np.tile([0, 0, 1], (4, 1))]).astype(np.float32))
    # a triangle reaching behind the near plane (dropped whole) next to a valid one
    near = dict(vertices=np.array([[0, 0, 0], [50, 0, 0], [0, 50, 0], [0, 0, 350], [-50, 0, 0], [0, -50, 0]], np.float32),
                faces=np.array([[0, 1, 3], [0, 4, 5]], np.int32))
    return dict(colour=colour, textured=textured, huge_tiny=huge_tiny, zfight=zf, near=near)


def _poses(n, distance=400.0, miss=False):
    p = synth.fibonacci_view_poses(n, distance).numpy()
    if miss:
        p[-1, :3, 3] = [5000.0, 0.0, distance]                 # the object is far outside the frustum
    return p


def _gpu(mesh, poses, K, H, W, z_near=100.0):
    dm = render._device_mesh(mesh, DEV)
    n = len(poses)
    ws = torch.empty(n * H * W * 4, dtype=torch.int64, device=DEV)
    rgba = torch.full((n, 4, H, W), float("nan"), device=DEV)
    depth = torch.full((n, H, W), float("nan"), device=DEV)
    boxes = torch.full((n, 4), -7, dtype=torch.int64, device=DEV)
    render.render_chunk(dm, torch.as_tensor(poses, dtype=torch.float32, device=DEV).contiguous(),
                        torch.as_tensor(K, dtype=torch.float32, device=DEV).contiguous(), H, W, z_near, ws, rgba, depth,
                        boxes)
    torch.cuda.synchronize()
    return dict(keys=ws.cpu().numpy().view(np.uint64).reshape(n, H, W, 4), rgba=rgba.cpu().numpy(),
                depth=depth.cpu().numpy(), boxes=boxes.cpu().numpy())


CASES = [("colour", 3, 480, 640), ("colour", 12, 120, 160), ("textured", 2, 480, 640), ("textured", 12, 120, 160),
         ("huge_tiny", 2, 480, 640), ("zfight", 6, 120, 160), ("near", 6, 120, 160)]


@pytest.mark.parametrize("name,n,H,W", CASES)
def test_render_is_bit_identical_to_the_oracle(name, n, H, W):
    mesh = meshes()[name]
    K = K_FULL if H == 480 else K_QUARTER
    poses = _poses(n, distance=250.0 if name == "near" else 400.0, miss=True)
    if name == "huge_tiny":
        poses[0] = np.eye(4)
        poses[0, 2, 3] = 200.0
    got = _gpu(mesh, poses, K, H, W)
    again = _gpu(mesh, poses, K, H, W)
    for k in got:
        assert np.array_equal(got[k], again[k], equal_nan=True), f"{k} differs between two runs"
    for v in range(n):
        ref = rp.render(mesh["vertices"], mesh["faces"], poses[v], K, H, W, 100.0, vertex_color=mesh.get("vertex_color"),
                        face_uv=mesh.get("face_uv"), texture=mesh.get("texture"), constant_color=mesh.get("constant_color"))
        assert np.array_equal(got["keys"][v], ref["keys"]), f"view {v}: face id / depth keys differ"
        assert np.array_equal(got["rgba"][v, 3], ref["rgba"][3]), f"view {v}: alpha differs"
        assert np.array_equal(got["depth"][v], ref["depth"]), f"view {v}: depth differs"
        assert np.array_equal(got["boxes"][v], ref["box"]), f"view {v}: box differs"
        assert np.array_equal(got["rgba"][v, :3], ref["rgba"][:3]), f"view {v}: RGB differs"
    covered = (got["keys"] != rp.EMPTY).any(-1)
    assert covered[0].any() and not covered[-1].any()          # the last view misses the object
    assert got["boxes"][-1].tolist() == [0, 0, W, H]
    if name == "zfight":                                       # view 0 looks at the quads face on
        ids = got["keys"][0][covered[0]] & np.uint64(0xFFFFFFFF)
        assert set(ids.ravel().tolist()) - {rp.EMPTY & np.uint64(0xFFFFFFFF)} == {0, 2}   # lowest id of each half


def test_render_templates_chunks_views_and_validates(monkeypatch):
    mesh = meshes()["colour"]
    poses = _poses(7)
    whole = render.render_templates(mesh, poses, K_QUARTER, size=(120, 160))
    monkeypatch.setattr(render, "WORKSPACE_BYTES", 3 * 120 * 160 * 32)            # 3 views per chunk
    parts = render.render_templates(mesh, poses, K_QUARTER, size=(120, 160))
    for k in ("rgba", "depth", "boxes"):
        assert torch.equal(whole[k], parts[k]), k
    bad = dict(mesh, faces=np.array([[0, 1, len(mesh["vertices"])]]))
    with pytest.raises(ValueError, match="outside"):
        render.render_templates(bad, poses, K_QUARTER, size=(120, 160))


def _models():
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    return bench.build_models(torch.device(DEV))


def test_onboarding_from_meshes_equals_onboarding_from_their_renders():
    """`onboard_meshes` renders and onboards one object at a time; `onboard_templates` fed the same renderer's RGBA and
    boxes must write a byte-identical bank (crop, both encoders in 64-crop chunks across objects, set_poses)."""
    ms = meshes()
    objs = [ms["colour"], ms["textured"]]
    T = 40
    poses = torch.as_tensor(_poses(T))
    model = _models()
    eng_m = model.onboard_meshes("meshes", objs, poses)
    renders = [render.render_templates(m, poses, render.TEMPLATE_K) for m in objs]
    eng_t = model.onboard_templates("renders", [r["rgba"] for r in renders], torch.stack([r["boxes"] for r in renders]),
                                    render.TEMPLATE_K, poses.expand(2, T, 4, 4))
    torch.cuda.synchronize()
    assert torch.equal(model.template_datas["meshes"].M, model.template_datas["renders"].M)
    assert torch.equal(model.template_datas["meshes"].poses, model.template_datas["renders"].poses)
    assert torch.equal(eng_m._bank_view(), eng_t._bank_view()), "banks differ"
    assert model.onboarding_s_per_object > 0


def test_a_query_rendered_at_a_template_pose_retrieves_that_template():
    """End to end: the query is rendered at template tau's pose and cropped with its box, so its crop equals the
    template's.  tau must be among the top-k, and its correspondences must be the identity on the patches (the
    high-frequency texture leaves no exact feature ties between patches)."""
    import src.megapose.utils.tensor_collection as tc
    from gigapose_b200.preprocess import CLIP_MEAN, CLIP_STD, crop_resize_pad
    rng = np.random.default_rng(5)
    V, Fc = icosphere(3, 70.0, rng, bumps=0.1)
    mesh = dict(vertices=V, faces=Fc, face_uv=_uv_sphere(V, Fc, 1.0),
                texture=rng.uniform(0, 1, (256, 256, 3)).astype(np.float32))
    T, tau = 24, 9
    poses = torch.as_tensor(_poses(T))
    model = _models()
    model.onboard_meshes("e2e", [mesh], poses)
    q = render.render_templates(mesh, poses[tau:tau + 1], render.TEMPLATE_K)
    crop = crop_resize_pad(q["boxes"], q["rgba"], 224, mean=CLIP_MEAN + (0.0,), std=CLIP_STD + (1.0,))
    batch = tc.PandasTensorCollection(infos=pd.DataFrame(dict(label=["1"], scene_id=[0], view_id=[0])),
                                      tar_img=crop["images"][:, :3].contiguous(), tar_mask=crop["images"][:, 3].contiguous(),
                                      tar_K=torch.tensor(render.TEMPLATE_K).view(1, 3, 3), tar_M=crop["M"])
    pred = model.retrieve(batch, "e2e", sort_pred_by_inliers=False)
    ids = pred.id_src[0].cpu().tolist()
    assert tau in ids, ids
    j = ids.index(tau)
    tar, src = pred.tar_pts[0, j].cpu(), pred.src_pts[0, j].cpu()
    valid = tar[:, 0] >= 0
    assert int(valid.sum()) >= 40, int(valid.sum())
    assert torch.equal(tar[valid], src[valid])
