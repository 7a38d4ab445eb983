"""Row f14 on the GPU: csrc/vis.cu against oracle/vis_port.py and the cv2 / PIL / scipy fixture bit for bit, the per-vertex
errors against gp_bop_add, `python -m gigapose_b200.vis` end to end on a synthetic tree, and the retrieval panels."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

import add_fp64 as af
from gigapose_b200 import _lib, bop_eval, render, vis
from oracle import add_port
from oracle import vis_port as P

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vis_reference.npz")


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def _pose(rng, dist=500.0):
    a = rng.normal(size=3)
    a /= np.linalg.norm(a)
    R = render_rot(a, rng.uniform(0, 2 * np.pi))
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = R
    T[:3, 3] = rng.normal(0, 20, 3) + [0, 0, dist]
    return T


def render_rot(a, t):
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * k + (1 - np.cos(t)) * (k @ k)


def _near(T, rng, deg=3.0, mm=4.0):
    D = np.eye(4, dtype=np.float32)
    a = rng.normal(size=3)
    D[:3, :3] = render_rot(a / np.linalg.norm(a), np.deg2rad(deg))
    D[:3, 3] = rng.normal(0, mm, 3)
    return (D @ T).astype(np.float32)


# ---------------------------------------------------------------------------------------------- vertex errors
def test_vertex_errors_sum_to_gp_bop_add_and_equal_the_port():
    rng = np.random.default_rng(0)
    sizes = [1, 255, 1024, 1025, 100000]
    objs = [rng.normal(0, 40, (n, 3)).astype(np.float32) for n in sizes]
    vo = np.cumsum([0] + sizes).tolist()
    V = torch.as_tensor(np.concatenate(objs), device=DEV)
    obj, pe, pg, sym = [], [], [], []
    for o in range(len(sizes)):
        for s in (False, True):
            T = _pose(rng)
            obj.append(o)
            pg.append(T)
            pe.append(_near(T, rng))
            sym.append(s)
    pe_d, pg_d = torch.as_tensor(np.stack(pe), device=DEV), torch.as_tensor(np.stack(pg), device=DEV)
    vals, offs = vis.vertex_errors(obj, vo, V, pe_d, pg_d, sym)
    K = torch.as_tensor(np.array([[[600, 0, 320], [0, 600, 240], [0, 0, 1]]], np.float32), device=DEV)
    ref = bop_eval.add_errors(torch.as_tensor(np.array(obj, np.int32), device=DEV), vo, V, K,
                              torch.zeros(len(obj), dtype=torch.int32, device=DEV), pe_d, pg_d).cpu().numpy()
    vals = vals.cpu().numpy()
    for p, (o, s) in enumerate(zip(obj, sym)):
        v = vals[offs[p]:offs[p + 1]]
        assert len(v) == sizes[o]
        # fp64 sums in gp_bop_add's chunk order equal its ADD / ADD-S bit for bit
        assert add_port.chunked_mean(v) == ref[p, 1 if s else 0], (o, s)
        if sizes[o] <= 1025:
            assert np.array_equal(v.view(np.uint32), P.vertex_errors(objs[o], pe[p], pg[p], s).view(np.uint32))
    assert np.isfinite(vals).all()
    # per vertex against tests/add_fp64.py (fp64, cKDTree nearest neighbours) within f12's per-point bar
    worst = 0.0
    for p, (o, s) in enumerate(zip(obj, sym)):
        e, g = af._apply(pe[p], objs[o]), af._apply(pg[p], objs[o])
        want = af.nn_kdtree(g, e) if s else np.linalg.norm(e - g, axis=1)
        bar = af.bars(objs[o], pe[p], pg[p], K[0].cpu().numpy().astype(np.float64))[1 if s else 0]
        worst = max(worst, float((np.abs(vals[offs[p]:offs[p + 1]].astype(np.float64) - want) / bar).max()))
    print("f14 per-vertex ADD / ADD-S, worst |kernel - fp64| / bar:", worst)
    assert worst <= 1.0


def test_vertex_errors_invalid_pairs_are_nan():
    lib = _lib.load()
    import ctypes as C
    V = torch.zeros(10, 3, device=DEV)
    vo = (C.c_int32 * 3)(0, 4, 10)
    obj = torch.tensor([0, 5, 1], dtype=torch.int32, device=DEV)              # object 5 does not exist
    off = torch.tensor([0, 4, 7, 10], dtype=torch.int64, device=DEV)          # pair 2's slot is 3 long, not 6
    I = torch.eye(4, device=DEV).expand(3, 4, 4).contiguous()
    sym = torch.zeros(3, dtype=torch.uint8, device=DEV)
    out = torch.full((10,), 7.0, device=DEV)
    _lib.check(lib.gp_vis_vertex_errors(3, 2, obj.data_ptr(), vo, V.data_ptr(), I.data_ptr(), I.data_ptr(),
                                        sym.data_ptr(), off.data_ptr(), out.data_ptr(), None))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert (o[:4] == 0).all() and np.isnan(o[4:]).all()


def test_heat_colors_equal_the_port(z):
    rng = np.random.default_rng(1)
    values = [rng.uniform(0, 150, 3000).astype(np.float32), rng.uniform(5, 20, 999).astype(np.float32),
              np.zeros(17, np.float32), np.array([1.0, np.nan, 3.0], np.float32), rng.uniform(0, 90, 1).astype(np.float32)]
    sym = [False, True, True, False, False]
    offs = np.cumsum([0] + [len(v) for v in values])
    cols = vis.heat_colors(torch.as_tensor(np.concatenate(values), device=DEV), offs, sym, 100.0).cpu().numpy()
    for i, (v, s) in enumerate(zip(values, sym)):
        ref, _ = P.heat_colors(v, s, 100.0, z["turbo"])
        assert np.array_equal(cols[offs[i]:offs[i + 1]].view(np.uint32), ref.view(np.uint32)), i
    assert np.array_equal(cols[offs[2]:offs[3]], np.tile(z["turbo"][0] / np.float32(255), (17, 1)).astype(np.float32))


# ---------------------------------------------------------------------------------------------- overlay
def _box(alpha):
    ys, xs = np.nonzero(alpha > 0)
    if len(ys) == 0:
        return [0, 0, alpha.shape[1], alpha.shape[0]]
    return [xs.min(), ys.min(), xs.max() + 1, ys.max() + 1]


def _layers(H, W, rng, n):
    """n layers: blobs that touch each border in turn, an empty one, one covering the frame and one hidden behind a
    later, larger one."""
    yy, xx = np.mgrid[0:H, 0:W]
    rgba = np.zeros((n, 4, H, W), np.float32)
    for l in range(n):
        kind = l % 8
        if kind == 5:
            continue                                                     # empty render
        if kind == 6:
            a = np.ones((H, W), bool)                                    # the whole frame
        else:
            cy, cx = [(0, W / 2), (H - 1, W / 2), (H / 2, 0), (H / 2, W - 1), (H / 2, W / 2), None, None,
                      (H / 3, W / 3)][kind]
            r = max(2.0, min(H, W) * rng.uniform(0.1, 0.3))
            a = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
        rgba[l, :3] = rng.integers(0, 256, (3, H, W)) / np.float32(255)
        rgba[l, 3] = a
        rgba[l, :3] *= a
    if n > 1:                                   # layer 0, its contour included, fully hidden by the last layer
        rgba[-1, 3] = np.maximum(rgba[-1, 3], P.dilate2(rgba[0, 3] > 0))
    rgba[:, :3] = (np.rint(rgba[:, :3] * 255) / 255).astype(np.float32)
    boxes = np.array([_box(rgba[l, 3]) for l in range(n)], np.int64)
    return rgba, boxes


@pytest.mark.parametrize("H,W", [(17, 17), (480, 640), (1080, 1920)])
def test_overlay_equals_the_port(H, W):
    rng = np.random.default_rng(H)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    for n in ((8, 40) if H < 1000 else (9,)):
        rgba, boxes = _layers(H, W, rng, n)
        colors = rng.integers(0, 256, (n, 3), dtype=np.uint8)
        out = vis.overlay(torch.as_tensor(img, device=DEV), torch.as_tensor(rgba, device=DEV),
                          torch.as_tensor(boxes, device=DEV), colors).cpu().numpy()
        assert np.array_equal(out, P.overlay(img, rgba, boxes, colors)), n
        black = vis.overlay(None, torch.as_tensor(rgba, device=DEV), torch.as_tensor(boxes, device=DEV)).cpu().numpy()
        assert np.array_equal(black, P.overlay(None, rgba, boxes, None)), n


def test_overlay_background_equals_cvtcolor(z):
    for k in ("random", "extreme"):
        img = z[f"gray_in_{k}"]
        out = vis.overlay(torch.as_tensor(img, device=DEV), None, None).cpu().numpy()
        assert np.array_equal(out, np.repeat(z[f"gray_out_{k}"][..., None], 3, 2)), k


# ---------------------------------------------------------------------------------------------- Kabsch panels
def _crops(n, rng):
    return P.crop_from_u8(rng.integers(0, 256, (n, 3, 224, 224), dtype=np.uint8),
                          np.where(rng.random((n, 224, 224)) < 0.7, 255, rng.integers(0, 256, (n, 224, 224))).astype(np.uint8))


def test_kabsch_equals_the_fixture(z):
    q, qm = P.crop_from_u8(z["kabsch_query_u8"], z["kabsch_query_mask_u8"])
    t, tm = P.crop_from_u8(z["kabsch_tmpl_u8"], z["kabsch_tmpl_mask_u8"])
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    out = vis.kabsch(d(q), d(qm), d(t), d(tm), d(z["kabsch_M"])).cpu().numpy()
    assert np.array_equal(out, z["kabsch_out"])


def _exact_crop(u8):
    """f32 [3,H,W] crop that convert_tensor_to_image maps back to the u8 planes [3,H,W] exactly."""
    m = np.array((0.485, 0.456, 0.406))[:, None, None]
    sd = np.array((0.229, 0.224, 0.225))[:, None, None]
    x = (((u8.astype(np.float64) + 0.5) / 255 - m) / sd).astype(np.float32)
    assert np.array_equal(P.unnormalise(x), u8.transpose(1, 2, 0))
    return x


def _exact_mask(u8):
    x = ((u8.astype(np.float64) + 0.5) / 255).astype(np.float32)
    assert np.array_equal(P.mask_u8(x), u8)
    return x


def test_kabsch_warps_equal_cv2_on_every_fixture_matrix(z):
    """The template unnormalises exactly to the fixture's RGBA warp source, so the kernel warps what cv2 warped.  For
    each of the 20 matrices the expected panel is built from the port's warp after checking that it is cv2's output
    (its SHA-256 is the fixture's): the query's grey with cv2's warp pasted through its alpha and the red edge."""
    import hashlib
    src = z["warp_src"]
    tmpl, tmask = _exact_crop(src[..., :3].transpose(2, 0, 1)), _exact_mask(src[..., 3])
    q8 = np.random.default_rng(20).integers(0, 256, (3, 224, 224), dtype=np.uint8)
    q = _exact_crop(q8)
    Ms = z["warp_M"]
    n = len(Ms)
    assert n == 20
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    out = vis.kabsch(d(np.repeat(q[None], n, 0)), d(np.zeros((n, 224, 224), np.float32)), d(np.repeat(tmpl[None], n, 0)),
                     d(np.repeat(tmask[None], n, 0)), d(Ms)).cpu().numpy()
    grey = np.repeat(P.gray(q8.transpose(1, 2, 0))[..., None], 3, 2)
    for i in range(n):
        w = P.warp_affine(src, Ms[i][:2])
        assert hashlib.sha256(np.ascontiguousarray(w).tobytes()).hexdigest() == str(z["warp_sha256"][i]), i
        want = P.paste(grey, w[..., :3], w[..., 3])
        want[P.dilate3(P.boundary_edge(P.self_pasted(w[..., 3]) > 0))] = (255, 0, 0)
        assert np.array_equal(out[i], want), i


@pytest.mark.parametrize("b", [1, 257])
def test_kabsch_batches_equal_the_port(b):
    rng = np.random.default_rng(b)
    q, qm = _crops(b, rng)
    t, tm = _crops(b, rng)
    M = np.stack([np.array([[np.cos(a) * s, -np.sin(a) * s, tx], [np.sin(a) * s, np.cos(a) * s, ty], [0, 0, 1]])
                  for a, s, tx, ty in zip(rng.uniform(-3, 3, b), rng.uniform(0.3, 3, b), rng.uniform(-100, 200, b),
                                          rng.uniform(-100, 200, b))]).astype(np.float32)
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    out = vis.kabsch(d(q), d(qm), d(t), d(tm), d(M)).cpu().numpy()
    for i in ([0] if b == 1 else [0, 1, 128, 255, 256]):
        assert np.array_equal(out[i], P.kabsch_panel(q[i], qm[i], t[i], tm[i], M[i])), i


def test_kabsch_identity_on_its_own_query():
    rng = np.random.default_rng(9)
    q, qm = _crops(1, rng)
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    out = vis.kabsch(d(q), d(qm), d(q), d(qm), d(np.eye(3, dtype=np.float32)[None])).cpu().numpy()[0]
    img, a = P.unnormalise(q[0]), P.mask_u8(qm[0])
    expect = P.paste(np.repeat(P.gray(img)[..., None], 3, 2), img, a)
    edge = P.dilate3(P.boundary_edge(P.self_pasted(a) > 0))
    expect[edge] = (0, 255, 0)                        # both edges coincide: the query's green is drawn last
    assert np.array_equal(out, expect)
    assert edge.any() and (out == [0, 255, 0]).all(-1).sum() == edge.sum()


# ---------------------------------------------------------------------------------------------- end to end
def _write_csv(path, rows):
    with open(path, "w") as f:
        f.write("scene_id,im_id,obj_id,score,R,t,time\n")
        for r in rows:
            f.write(f"{r['scene_id']},{r['im_id']},{r['obj_id']},{r['score']},"
                    f"{' '.join(repr(float(v)) for v in np.asarray(r['R']).reshape(-1))},"
                    f"{' '.join(repr(float(v)) for v in np.asarray(r['t']).reshape(-1))},{r['time']}\n")


def test_cli_end_to_end(tmp_path, z):
    from test_vis_cpu import synthetic_results, synthetic_tree
    models, info, scenes = synthetic_tree(tmp_path / "ds")
    coarse = synthetic_results(scenes)
    refined = [dict(r) for r in coarse]
    refined[3]["R"], refined[3]["t"] = scenes[1][0]["gt"][1][1], np.asarray(scenes[1][0]["gt"][1][2], float)
    a, b = str(tmp_path / "coarse.csv"), str(tmp_path / "coarse_icp.csv")
    _write_csv(a, coarse)
    _write_csv(b, refined)
    out = str(tmp_path / "vis")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "gigapose_b200.vis", "--results", a, b, "--dataset-dir",
                        str(tmp_path / "ds"), "--out", out], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    from PIL import Image
    files = sorted(os.listdir(out))
    assert files == ["000001_000000.png", "000001_000003.png"]
    fig = np.asarray(Image.open(os.path.join(out, files[0])))
    H, W = 120, 160
    assert fig.shape == (2 * H, 3 * W, 3)
    rgb = np.asarray(Image.open(str(tmp_path / "ds" / "test" / "000001" / "rgb" / "000000.png")))
    assert np.array_equal(fig[:H, :W], rgb)
    # the ground-truth overlay is the port's overlay of the same renders, far to near, green contours
    gts = sorted(scenes[1][0]["gt"], key=lambda g: -np.linalg.norm(g[2]))
    K = np.asarray(scenes[1][0]["K"], np.float32)
    rgba, boxes = [], []
    for o, R, t in gts:
        T = vis._pose(R, t)
        rr = render.render_templates(dict(vertices=models[o][0], faces=models[o][1]), T[None], K, size=(H, W),
                                     z_near=vis.Z_NEAR, device=DEV)
        rgba.append(rr["rgba"].cpu().numpy())
        boxes.append(rr["boxes"].cpu().numpy())
    rgba, boxes = np.concatenate(rgba), np.concatenate(boxes)
    ref = P.overlay(rgb, rgba, boxes, np.tile(vis.GT_COLOR, (len(gts), 1)))
    assert np.array_equal(fig[H:, :W], ref)
    green = (fig[H:, :W] == [0, 255, 0]).all(-1)
    cont = np.zeros((H, W), bool)                    # the port's contours, each painted over by later layers' masks
    for l in range(len(gts)):
        cont[rgba[l, 3] > 0] = False
        cont |= P.contour(rgba[l, 3] > 0)
    assert np.array_equal(green, cont) and cont.any()
    # the refined csv's symmetric estimate equals its ground truth: turbo's first entry on its heat map
    heat = fig[:H, 2 * W:3 * W].reshape(-1, 3).astype(int)
    t0 = z["turbo"][0].astype(int)
    sph = render.render_templates(dict(vertices=models[2][0], faces=models[2][1]), vis._pose(*gts[0][1:])[None], K,
                                  size=(H, W), z_near=vis.Z_NEAR, device=DEV)["rgba"][0, 3].cpu().numpy() > 0
    inside = sph.reshape(-1)
    counts = {tuple(c): n for c, n in zip(*np.unique(heat[inside], axis=0, return_counts=True))}
    assert counts.get(tuple(t0), 0) > 0.5 * inside.sum(), counts
    assert (heat[inside] <= t0).all()
    assert fig.shape == np.asarray(Image.open(os.path.join(out, files[1]))).shape
    # heat maps are drawn at the ground-truth poses (every estimate here is matched): both csvs' heat maps cover
    # exactly the ground truths' silhouette, whatever the estimates' poses
    sil = (rgba[:, 3] > 0).any(0)
    for c in (1, 2):
        assert np.array_equal(fig[:H, c * W:(c + 1) * W].any(-1), sil), c


# ---------------------------------------------------------------------------------------------- retrieval panels
def test_template_crops_and_vis_retrieval():
    import src.megapose.utils.tensor_collection as tc
    from gigapose_b200.preprocess import CLIP_MEAN, CLIP_STD, crop_resize_pad
    from test_gpu_render import _models, _poses, meshes
    ms = meshes()
    objs = [ms["colour"], ms["textured"]]
    T = 24
    poses = torch.as_tensor(_poses(T))
    model = _models()
    seen = []                                        # the onboarding crops, recomputed the way _onboard makes them
    model.onboard_meshes("vis", objs, poses)
    for o, m in enumerate(objs):
        r = render.render_templates(m, poses, render.TEMPLATE_K)
        crop = crop_resize_pad(r["boxes"], r["rgba"], 224, mean=CLIP_MEAN + (0.0,), std=CLIP_STD + (1.0,))
        ids = [3, 0, 17, 3]
        rgb, mask = model.template_crops("vis", o, ids)
        assert torch.equal(rgb, crop["images"][ids, :3]) and torch.equal(mask, crop["images"][ids, 3])
        seen.append(crop)
    # a batch of two queries, one per object: template views 5 and 11 rendered and cropped
    q = [render.render_templates(objs[o], poses[v:v + 1], render.TEMPLATE_K) for o, v in ((0, 5), (1, 11))]
    crops = [crop_resize_pad(x["boxes"], x["rgba"], 224, mean=CLIP_MEAN + (0.0,), std=CLIP_STD + (1.0,)) for x in q]
    img = torch.cat([c["images"] for c in crops])
    batch = tc.PandasTensorCollection(infos=pd.DataFrame(dict(label=["1", "2"], scene_id=[0, 0], view_id=[0, 0])),
                                      tar_img=img[:, :3].contiguous(), tar_mask=img[:, 3].contiguous(),
                                      tar_K=torch.tensor(render.TEMPLATE_K).view(1, 3, 3).expand(2, 3, 3).contiguous(),
                                      tar_M=torch.cat([c["M"] for c in crops]))
    pred = model.retrieve(batch, "vis")
    panels = model.vis_retrieval("vis", batch, pred)
    k = pred.id_src.shape[1]
    assert tuple(panels.shape) == (k * 2, 3, 224, 224)
    ids, M = pred.id_src.cpu().numpy(), pred.M.float().cpu().numpy()
    for r in range(k):
        for b in range(2):
            src = seen[b]["images"][int(ids[b, r])].cpu().numpy()
            ref = P.kabsch_panel(img[b, :3].cpu().numpy(), img[b, 3].cpu().numpy(), src[:3], src[3], M[b, r])
            got = panels[r * 2 + b].permute(1, 2, 0).cpu().numpy()
            assert np.array_equal(np.rint(got * 255).astype(np.uint8), ref), (r, b)


def test_bop_run_vis_every_writes_retrieval_panels(tmp_path):
    from PIL import Image

    from gigapose_b200 import bop_run
    from gigapose_b200.synth import fibonacci_view_poses
    from test_gpu_bop_run_masked import _occluded_lmo_tree
    ds, _, _ = _occluded_lmo_tree(str(tmp_path))
    np.save(str(tmp_path / "poses.npy"), fibonacci_view_poses(24, 400.0).numpy())
    model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)
    out = str(tmp_path / "run")
    bop_run.run(model, ds, out, template_poses=str(tmp_path / "poses.npy"), vis_every=2)
    n_images = len(bop_run.plan(ds)["images"])
    written = sorted(f for f in os.listdir(out) if f.startswith("retrieved_sample_"))
    assert written == [f"retrieved_sample_{i}.png" for i in range(0, n_images, 2)]
    k = model.testing_metric.k
    w, h = Image.open(os.path.join(out, written[0])).size
    assert (h - 2) % (224 + 2) == 0 and (h - 2) // (224 + 2) == k          # save_image: one row per rank, padding 2
    plain = str(tmp_path / "plain")
    bop_run.run(model, ds, plain)
    assert not [f for f in os.listdir(plain) if f.startswith("retrieved_sample_")]


def test_onboard_templates_keeps_no_renders():
    """The model keeps no reference to the caller's template renders: they are freed with the caller's copy, and
    template_crops says why it cannot return them.  After onboard_meshes it re-renders instead."""
    import gc

    from test_gpu_render import _models, _poses, meshes
    ms = meshes()
    objs = [ms["colour"], ms["textured"]]
    T = 24
    poses = torch.as_tensor(_poses(T))
    model = _models()
    rgba = [render.render_templates(m, poses, render.TEMPLATE_K)["rgba"] for m in objs]
    boxes = torch.stack([render.render_templates(m, poses, render.TEMPLATE_K)["boxes"] for m in objs])
    nbytes = sum(r.numel() * r.element_size() for r in rgba)
    model.onboard_templates("renders", rgba, boxes, render.TEMPLATE_K, poses.expand(2, T, 4, 4))
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    del rgba
    gc.collect()
    torch.cuda.synchronize()
    assert before - torch.cuda.memory_allocated() >= nbytes
    with pytest.raises(ValueError, match="not kept"):
        model.template_crops("renders", 0, [0])
    model.onboard_meshes("renders", objs, poses)                  # the same name rebuilt from meshes re-renders
    assert tuple(model.template_crops("renders", 1, [2, 5])[0].shape) == (2, 3, 224, 224)
