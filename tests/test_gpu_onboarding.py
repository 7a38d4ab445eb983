"""Row f16 on the GPU: gp_recentre_boxes / gp_recentre_crop against the fp64 restatement (tests/onboarding_fp64.py),
the planted identity against gp_crop_resize_pad, the geometry of a re-centred off-axis render against a direct render
at the virtual pose (with the two plausible wrong maps shown to fail), and `bop_run --onboarding static` end to end on
a synthetic tree whose onboarding_static sequences are rendered by the rasteriser."""
import json
import os

import numpy as np
import pytest
import torch

import onboarding_fp64 as ref
from bop_tree import rot, spheroid, tetra, write_tree
from gigapose_b200 import _lib, bop_eval, bop_run, onboarding, render
from gigapose_b200.preprocess import CLIP_MEAN, CLIP_STD, crop_resize_pad
from oracle.bop_run_port import binary_mask_to_rle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K_HOPE = np.array([[1390.0, 0, 961.5], [0, 1390.0, 538.5], [0, 0, 1]])     # a 1920 x 1080 camera of HOPE's kind


def _off_axis_pose(rng, max_deg, dist):
    off, az = np.radians(rng.uniform(0.3 * max_deg, max_deg)), rng.uniform(0, 2 * np.pi)
    P = np.eye(4)
    P[:3, :3] = rot(rng.normal(size=3), rng.uniform(0, 360))
    P[:3, 3] = np.array([np.sin(off) * np.cos(az), np.sin(off) * np.sin(az), np.cos(off)]) * dist
    return P


def _ellipse(rng, H, W, K, P):
    """A filled ellipse around the projection of the object origin, radii 3-12 % of the width."""
    p = K @ P[:3, 3]
    cx, cy = p[0] / p[2], p[1] / p[2]
    yy, xx = np.mgrid[:H, :W]
    a, b, th = rng.uniform(0.03, 0.12) * W, rng.uniform(0.03, 0.12) * W, rng.uniform(0, np.pi)
    u, v = (xx - cx) * np.cos(th) + (yy - cy) * np.sin(th), -(xx - cx) * np.sin(th) + (yy - cy) * np.cos(th)
    return ((u / a) ** 2 + (v / b) ** 2 < 1).astype(np.uint8)


@pytest.mark.parametrize("H,W", [(480, 640), (1080, 1920)])
def test_boxes_and_crops_equal_the_fp64_evaluator(H, W):
    rng = np.random.default_rng(H)
    n = 6
    Ks, poses, masks = [], [], []
    for _ in range(n):
        K = np.array([[rng.uniform(0.8, 1.2) * W, 0, W / 2 + rng.uniform(-0.05, 0.05) * W],
                      [0, rng.uniform(0.8, 1.2) * W, H / 2 + rng.uniform(-0.05, 0.05) * H], [0, 0, 1]])
        P = _off_axis_pose(rng, 25.0, rng.uniform(400, 900))
        Ks.append(K)
        poses.append(P)
        masks.append(_ellipse(rng, H, W, K, P))
    rgb = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    hinv = np.stack([onboarding.recentre(K, P)[2] for K, P in zip(Ks, poses)])
    src = np.stack([onboarding.mask_box(m) for m in masks])
    m_dev = torch.as_tensor(np.stack(masks)).to(DEV)
    boxes = onboarding.recentre_boxes(m_dev, hinv, src)
    crop = onboarding.recentre_crop(torch.as_tensor(rgb).to(DEV), m_dev, hinv, boxes)
    boxes = boxes.cpu().numpy()
    ties = 0
    for i in range(n):
        want_box = ref.recentred_box(masks[i], hinv[i])
        assert boxes[i].tolist() == want_box.tolist(), (i, boxes[i], want_box)
        want = ref.recentred_crop(rgb[i], masks[i], hinv[i], want_box)
        got_m = crop["mask"][i].cpu().numpy()
        differ = got_m != want["mask"]
        assert not (differ & ~want["tie"]).any(), (i, int((differ & ~want["tie"]).sum()))
        ties += int(want["tie"].sum())
        same = ~differ
        got = crop["images"][i].cpu().numpy()
        err = np.abs(got - want["images"])[:, same]
        assert err.max() <= 1e-5, (i, float(err.max()))
        gm = crop["M"][i].cpu().numpy()
        assert (np.abs(gm - want["M"]) <= 1e-6 * np.maximum(1.0, np.abs(want["M"]))).all(), (gm, want["M"])
        assert want["mask"].sum() > 100
    print("recentre_fp64", json.dumps(dict(size=[H, W], frames=n, mask_pixels_near_a_tie=ties)))


def test_on_axis_frame_at_the_template_camera_is_crop_resize_pad():
    rng = np.random.default_rng(5)
    H, W = 480, 640
    n = 4
    P = [np.eye(4) for _ in range(n)]
    masks = []
    for i in range(n):
        P[i][:3, :3] = rot(rng.normal(size=3), rng.uniform(0, 360))
        P[i][:3, 3] = [0.0, 0.0, rng.uniform(300, 900)]
        m = _ellipse(rng, H, W, np.asarray(render.TEMPLATE_K), P[i])
        m[rng.integers(100, 380), rng.integers(100, 540)] = 1                  # stray pixels inside the frame
        masks.append(m)
    rgb = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    hinv = np.stack([onboarding.recentre(render.TEMPLATE_K, p)[2] for p in P])
    src = np.stack([onboarding.mask_box(m) for m in masks])
    m_dev = torch.as_tensor(np.stack(masks)).to(DEV)
    boxes = onboarding.recentre_boxes(m_dev, hinv, src)
    assert boxes.cpu().numpy().tolist() == src.tolist()
    got = onboarding.recentre_crop(torch.as_tensor(rgb).to(DEV), m_dev, hinv, boxes)
    want = crop_resize_pad(boxes, torch.as_tensor(rgb).permute(0, 3, 1, 2).float().to(DEV), 224,
                           mask=m_dev.float(), in_div=255.0, mean=CLIP_MEAN, std=CLIP_STD)
    assert torch.equal(got["mask"], want["mask"])
    assert float((got["images"] - want["images"]).abs().max()) <= 1e-6
    assert torch.equal(got["M"], want["M"])


def _textured_spheroid():
    V, F = spheroid(60.0, 40.0, 24, 48)
    col = 0.5 + 0.5 * np.stack([np.sin(V[:, 0] / 9.0), np.cos(V[:, 1] / 7.0), np.sin(V[:, 2] / 5.0 + 1.0)], 1)
    return dict(vertices=V, faces=F, vertex_color=col.astype(np.float32))


def _crop_stats(a, b):
    """Mask IoU of two crops and the mean |RGB| difference (in [0, 1] units) over their common mask eroded by 3 px."""
    ma, mb = a["mask"] > 0.5, b["mask"] > 0.5
    iou = float((ma & mb).sum() / max(1, (ma | mb).sum()))
    both = (ma & mb).float()[None, None]
    core = -torch.nn.functional.max_pool2d(-both, 7, 1, 3)[0, 0] > 0.5
    std = torch.tensor(CLIP_STD, device=DEV)[:, None, None]
    diff = ((a["images"] - b["images"]) * std).abs()[:, core]
    return iou, float(diff.mean()) if diff.numel() else float("inf")


def _recentre_render(mesh, P, K, H, W, hinv):
    r = render.render_templates(mesh, torch.as_tensor(P, dtype=torch.float32)[None], K, size=(H, W), device=DEV)
    rgb = (r["rgba"][0, :3].permute(1, 2, 0) * 255).round().to(torch.uint8)[None]
    mask = (r["rgba"][0, 3] > 0).to(torch.uint8)[None]
    src = onboarding.mask_box(mask[0].cpu().numpy())[None]
    boxes = onboarding.recentre_boxes(mask, hinv[None], src)
    b = boxes[0].tolist()
    if b[2] <= b[0]:
        raise ValueError("empty re-centred mask")
    return onboarding.recentre_crop(rgb, mask, hinv[None], boxes), b


def test_recentred_render_matches_a_render_at_the_virtual_pose():
    """H and the virtual pose must agree: a frame rendered off-axis at a HOPE camera and re-centred shows what a
    render at the virtual pose with the template camera shows.  R_v transposed or H not inverted breaks it."""
    mesh = _textured_spheroid()
    rng = np.random.default_rng(11)
    stats, wrong = [], []
    for k in range(4):
        while True:                        # the whole object inside the 1920 x 1080 frame, 20 px from its edges
            P = _off_axis_pose(rng, 25.0, rng.uniform(450, 700))
            p = K_HOPE @ P[:3, 3]
            r = K_HOPE[0, 0] * 60.0 / P[2, 3]
            if 20 + r < p[0] / p[2] < 1900 - r and 20 + r < p[1] / p[2] < 1060 - r:
                break
        Rv, V, hinv = onboarding.recentre(K_HOPE, P)
        got, gbox = _recentre_render(mesh, P, K_HOPE, 1080, 1920, hinv)
        d = render.render_templates(mesh, torch.as_tensor(V, dtype=torch.float32)[None], render.TEMPLATE_K, device=DEV)
        want = crop_resize_pad(d["boxes"], (d["rgba"][:, :3] * 255).round(), 224, mask=d["rgba"][:, 3],
                               in_div=255.0, mean=CLIP_MEAN, std=CLIP_STD)
        wbox = d["boxes"][0].tolist()
        assert 0 < wbox[0] and wbox[2] < 640 and 0 < wbox[1] and wbox[3] < 480     # the direct render is not clipped
        iou, drgb = _crop_stats(dict(images=got["images"][0], mask=got["mask"][0]),
                                dict(images=want["images"][0], mask=want["mask"][0]))
        sides = max(abs((gbox[2] - gbox[0]) - (wbox[2] - wbox[0])), abs((gbox[3] - gbox[1]) - (wbox[3] - wbox[1])))
        corner = max(abs(a - b) for a, b in zip(gbox, wbox))        # both boxes on the virtual camera's pixel grid
        stats.append(dict(iou=iou, rgb=drgb, side_px=sides, corner_px=corner,
                          off_deg=float(np.degrees(np.arccos(P[2, 3] / np.linalg.norm(P[:3, 3]))))))
        Kt_inv = np.linalg.inv(np.asarray(render.TEMPLATE_K))
        for name, bad in (("transposed_Rv", K_HOPE @ Rv @ Kt_inv), ("H_not_inverted", np.linalg.inv(hinv))):
            try:
                b, bbox = _recentre_render(mesh, P, K_HOPE, 1080, 1920, bad)
                w_iou, w_rgb = _crop_stats(dict(images=b["images"][0], mask=b["mask"][0]),
                                           dict(images=want["images"][0], mask=want["mask"][0]))
                w_corner = max(abs(a - b) for a, b in zip(bbox, wbox))
            except (_lib.GigaPoseNativeError, ValueError):
                w_iou, w_rgb, w_corner = 0.0, float("inf"), float("inf")
            wrong.append(dict(map=name, iou=w_iou, rgb=w_rgb, corner_px=w_corner))
    print("recentre_geometry", json.dumps(dict(right=stats, wrong=wrong)))
    # bars from the measurement on an H100 (DESIGN.md, row f16): IoU >= 0.974, RGB <= 0.033, box corners within 1 px
    for s in stats:
        assert s["iou"] >= 0.95 and s["rgb"] <= 0.05 and s["side_px"] <= 3 and s["corner_px"] <= 3, s
    # a wrong map still shows the object, distorted, so the crops alone tell it apart weakly (IoU 0.67-0.95); on the
    # virtual grid its box lands 205-5812 px away from the render's
    for w in wrong:
        assert w["corner_px"] > 50, w


# ---------------------------------------------------------------------------------------------------- end to end
K_ONB = np.array([[620.0, 0, 331.0], [0, 615.0, 236.5], [0, 0, 1]])


def _render_view(mesh, P, K, rng, H=480, W=640):
    r = render.render_templates(mesh, torch.as_tensor(P, dtype=torch.float32)[None], K, size=(H, W), device=DEV)
    a = r["rgba"][0, 3].cpu().numpy() > 0
    col = (r["rgba"][0, :3].permute(1, 2, 0).cpu().numpy() * 255).round().astype(np.uint8)
    rgb = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    rgb[a] = col[a]
    return rgb, a, np.round(r["depth"][0].cpu().numpy()).astype(np.uint16)


def _write_onboarding(ds, obj, name, frames):
    from PIL import Image
    d = os.path.join(ds, "onboarding_static", name)
    os.makedirs(os.path.join(d, "rgb"))
    os.makedirs(os.path.join(d, "mask_visib"))
    gt, cam = {}, {}
    for im, (rgb, mask, P, K) in enumerate(frames):
        Image.fromarray(rgb).save(os.path.join(d, "rgb", f"{im:06d}.png"))
        Image.fromarray(mask.astype(np.uint8) * 255).save(os.path.join(d, "mask_visib", f"{im:06d}_000000.png"))
        gt[str(im)] = [dict(obj_id=obj, cam_R_m2c=P[:3, :3].reshape(-1).tolist(), cam_t_m2c=P[:3, 3].tolist())]
        cam[str(im)] = dict(cam_K=np.asarray(K).reshape(-1).tolist(), depth_scale=1.0)
    for fname, v in (("scene_gt.json", gt), ("scene_camera.json", cam)):
        with open(os.path.join(d, fname), "w") as f:
            json.dump(v, f)


def _static_tree(root, rng, tpl, planted_view):
    """A 'ycbv' tree of two objects: onboarding_static up / down scenes of off-centre renders, one frame of object 1
    exactly at template pose `planted_view` with the template camera, and a test image identical to that frame."""
    ds = os.path.join(root, "ycbv")
    models = {1: spheroid(40.0, 25.0, 16, 32), 2: tetra(60.0)}
    meshes = {}
    for o, (V, F) in models.items():
        col = 0.5 + 0.5 * np.stack([np.sin(V[:, 0] / (6.0 + o)), np.cos(V[:, 1] / (5.0 + o)), np.sin(V[:, 2] / 4.0)], 1)
        meshes[o] = dict(vertices=V, faces=F, vertex_color=col.astype(np.float32))
    planted = None
    for o in models:
        for half, sign in (("up", 1.0), ("down", -1.0)):
            frames = []
            for k in range(10):
                z = sign * rng.uniform(0.1, 0.95)
                ph = rng.uniform(0, 2 * np.pi)
                cam = np.array([np.sqrt(1 - z * z) * np.cos(ph), np.sqrt(1 - z * z) * np.sin(ph), z])
                fwd = -cam
                up = np.array([0.0, 0.0, 1.0]) if abs(fwd[2]) < 0.99 else np.array([0.0, 1.0, 0.0])
                x = np.cross(up, fwd)
                x /= np.linalg.norm(x)
                R = np.stack([x, np.cross(fwd, x), fwd])
                P = np.eye(4)
                P[:3, :3] = rot(rng.normal(size=3), rng.uniform(-8, 8)) @ R            # off-centre: the camera looks
                P[:3, 3] = P[:3, :3] @ (-cam * 450.0)                                  # up to 8 deg past the origin
                rgb, mask, _ = _render_view(meshes[o], P, K_ONB, rng)
                frames.append((rgb, mask, P, K_ONB))
            if o == 1 and half == "up":
                P = np.asarray(tpl[planted_view], np.float64)
                rgb, mask, depth = _render_view(meshes[o], P, np.asarray(render.TEMPLATE_K), rng)
                planted = (len(frames), rgb, mask, P, depth)
                frames.append((rgb, mask, P, np.asarray(render.TEMPLATE_K)))
            _write_onboarding(ds, o, f"obj_{o:06d}_{half}", frames)
    # the test split: image 0 is the planted frame, image 1 shows object 2 off-centre
    idx, rgb0, mask0, P0, depth0 = planted
    P1 = np.eye(4)
    P1[:3, :3] = rot([1, 2, 3], 40)
    P1[:3, 3] = [60.0, -30.0, 500.0]
    rgb1, mask1, depth1 = _render_view(meshes[2], P1, np.asarray(render.TEMPLATE_K), rng)
    scenes, dets, targets = {1: {}}, [], []
    for im, (rgb, mask, P, depth, o) in enumerate(((rgb0, mask0, P0, depth0, 1), (rgb1, mask1, P1, depth1, 2))):
        bop_path = os.path.join(ds, "test", "000001", "rgb")
        os.makedirs(bop_path, exist_ok=True)
        from PIL import Image
        Image.fromarray(rgb).save(os.path.join(bop_path, f"{im:06d}.png"))
        x1, y1, x2, y2 = onboarding.mask_box(mask).tolist()
        dets.append(dict(scene_id=1, image_id=im, category_id=o, score=0.9, time=0.1, bbox=[x1, y1, x2 - x1, y2 - y1],
                         segmentation=dict(size=list(mask.shape), counts=binary_mask_to_rle(mask)["counts"])))
        scenes[1][im] = dict(gt=[(o, P[:3, :3], P[:3, 3])], visib=[1.0], K=np.asarray(render.TEMPLATE_K),
                             depth_scale=1.0, png=depth)
        targets.append((1, im, o, 1))
    info = {o: dict(diameter=float(np.linalg.norm(V.max(0) - V.min(0)))) for o, (V, _) in models.items()}
    write_tree(ds, models, info, scenes, targets)
    d = os.path.join(root, "default_detections", "core19_model_based_unseen", "cnos-fastsam")
    os.makedirs(d)
    with open(os.path.join(d, "cnos-fastsam_ycbv-test_synthetic.json"), "w") as f:
        json.dump(dets, f)
    return ds, idx


def test_static_run_writes_a_complete_csv_and_retrieves_the_planted_frame(tmp_path):
    from gigapose_b200.synth import fibonacci_view_poses
    rng = np.random.default_rng(21)
    tpl = fibonacci_view_poses(24, 450.0).double().numpy()
    ds, planted_idx = _static_tree(str(tmp_path), rng, tpl, planted_view=5)
    np.save(str(tmp_path / "poses.npy"), tpl.astype(np.float32))
    model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)
    out = str(tmp_path / "run")
    csv = bop_run.run(model, ds, out, "localization", template_poses=str(tmp_path / "poses.npy"), onboarding="static")
    assert csv.endswith("_bop_run_static.csv")
    with open(csv) as f:
        rows = [line.split(",") for line in f.read().splitlines()[1:]]
    assert sorted((int(r[1]), int(r[2])) for r in rows) == [(0, 1), (1, 2)]
    for r in rows:
        assert len(r) == 7 and all(np.isfinite(float(v)) for v in r[3].split() + r[4].split() + r[5].split())
    res = bop_eval.evaluate(csv, ds, "test", device=DEV)
    assert np.isfinite(res["ar"])
    views = model.onboarding_views["ycbv"]
    frame_ids, gaps = views["frame_ids"], views["gap_deg"]
    assert len(frame_ids) == 2 and all(len(f) == 24 for f in frame_ids)
    # the up scene comes after the down scene: the planted frame's index within object 1's frames
    planted = 10 + planted_idx
    assert frame_ids[0][5] == planted and gaps[0][5] < 1e-4
    # the planted test image: its detection's top-1 template is one built from the planted frame
    p = bop_run.plan(ds, "localization")
    from PIL import Image
    rgb = torch.as_tensor(np.asarray(Image.open(os.path.join(ds, "test", "000001", "rgb", "000000.png"))))
    batch = bop_run.image_batch(p, 0, rgb, torch.device(DEV))
    model.log_dir = str(tmp_path / "probe")
    os.makedirs(os.path.join(model.log_dir, "predictions"), exist_ok=True)
    _, kept = model.eval_retrieval(batch, idx_batch=0, dataset_name="ycbv")
    top1 = int(kept.id_src[0, 0])
    print("static_e2e", json.dumps(dict(top1=top1, frame=int(frame_ids[0][top1]), planted=planted,
                                        gap_max=[float(g.max()) for g in gaps], ar=res["ar"])))
    assert frame_ids[0][top1] == planted
    # the template crops come back from the frames: view 5's is the planted frame's crop, i.e. the test image's
    rgb_t, mask_t = model.template_crops("ycbv", 0, [5])
    assert torch.equal(mask_t[0], batch.tar_mask[0])
    assert float((rgb_t[0] - batch.tar_img[0]).abs().max()) <= 1e-5
