"""Row f9 on the GPU: gp_crop_resize_pad_rle bit-identical to gp_crop_resize_pad on the decoded masks, its device memory
on a HOPE-shaped image, and `bop_run.run` end to end on a synthetic BOP tree against a hand-driven run of the same
model on dense masks."""
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from bop_tree import spheroid, tetra, write_tree
from gigapose_b200 import bop_eval, bop_run, render
from gigapose_b200.preprocess import crop_detections_rle, preprocess_queries
from oracle.bop_run_port import binary_mask_to_rle, rle_to_binary_mask, rle_to_string

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bits(t):
    return t.contiguous().view(torch.int32)


def _boxes(rng, n, H, W):
    """The edge cases first (clipped at each edge, fully outside, zero width, larger than the image, and the identity /
    doubling index paths of outputs with rh + rw <= 128), then random boxes."""
    special = [[-30, 50, 200, 300], [100, -40, 300, 200], [W - 100, 100, W + 80, 300], [100, H - 60, 260, H + 90],
               [W + 10, 20, W + 200, 200], [50, 60, 50, 200], [-100, -100, W + 100, H + 100],
               [W - 40, H - 50, W - 40 + 224, H - 50 + 224], [W - 20, H - 30, W + 92, H + 82]]
    out = []
    for i in range(n):
        if i < len(special):
            out.append(special[i])
            continue
        x, y = rng.integers(-50, W, 2) if i % 3 else rng.integers(0, W // 2, 2)
        w, h = rng.integers(1, max(W, H) // (1 + i % 4), 2)
        out.append([int(x), int(y), int(x + w), int(y + h)])
    return np.array(out, np.int64)


def _counts(rng, i, H, W):
    """Run lengths of detection i: ellipses, noise at several densities, empty, full, runs past H * W, runs ending
    before H * W."""
    kind = i % 7
    n = H * W
    if kind == 4:
        return [0, n]
    if kind == 5:
        c = binary_mask_to_rle(rng.random((H, W)) < 0.02)["counts"]
        return c + [7, 1000, 3]                        # past H * W: cut off
    if kind == 6:
        return [int(rng.integers(0, n // 2)), int(rng.integers(1, n // 4))]      # the rest is zeros
    if kind == 3:
        return [n]
    yy, xx = np.mgrid[:H, :W]
    cy, cx = rng.uniform(0, H), rng.uniform(0, W)
    ry, rx = rng.uniform(5, H / 2), rng.uniform(5, W / 2)
    m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
    if kind == 2:
        m ^= rng.random((H, W)) < 0.05
    return binary_mask_to_rle(m)["counts"]


def _case(H, W, n, m, seed, many_runs=False):
    rng = np.random.default_rng(seed)
    rgb = torch.as_tensor(rng.integers(0, 256, (m, H, W, 3), dtype=np.uint8))
    counts = [_counts(rng, i, H, W) for i in range(n)]
    if many_runs:
        counts[-1] = binary_mask_to_rle(rng.random((H, W)) < 0.5)["counts"]
        assert len(counts[-1]) > 50000
    idx = np.arange(n) % m
    return rgb, counts, _boxes(rng, n, H, W), idx


def _both(rgb, counts, boxes, idx):
    H, W = rgb.shape[1:3]
    flat = np.concatenate([np.asarray(c, np.int32) for c in counts]) if counts else np.zeros(0, np.int32)
    off = np.concatenate([[0], np.cumsum([len(c) for c in counts])])
    rle = crop_detections_rle(rgb.to(DEV), flat, off, boxes, idx)
    dense = torch.stack([torch.as_tensor(rle_to_binary_mask(dict(size=[H, W], counts=c))) for c in counts]).float()
    ref = preprocess_queries(rgb.to(DEV).permute(0, 3, 1, 2), dense.to(DEV), torch.as_tensor(boxes),
                             torch.as_tensor(idx))
    return rle, ref


@pytest.mark.parametrize("H,W,n,m,many", [(480, 640, 1, 1, False), (480, 640, 23, 3, True), (480, 640, 200, 3, False),
                                           (1080, 1920, 100, 3, False), (1080, 1920, 9, 1, True)])
def test_rle_crop_is_bit_identical_to_the_dense_crop(H, W, n, m, many):
    rgb, counts, boxes, idx = _case(H, W, n, m, seed=n + H, many_runs=many)
    rle, ref = _both(rgb, counts, boxes, idx)
    for k in ("tar_img", "tar_mask", "tar_M"):
        assert rle[k].shape == ref[k].shape
        diff = float((rle[k] - ref[k]).abs().max())
        assert torch.equal(_bits(rle[k]), _bits(ref[k])), f"{k}: largest difference {diff}"
    assert float(rle["tar_mask"].sum()) > 0


def test_more_than_one_group_of_detections():
    """Detections go to the device in groups of 256: 300 detections take two groups of launches."""
    rgb, counts, boxes, idx = _case(120, 160, 300, 2, seed=3)
    rle, ref = _both(rgb, counts, boxes, idx)
    for k in ("tar_img", "tar_mask", "tar_M"):
        assert torch.equal(_bits(rle[k]), _bits(ref[k])), k


def test_rle_path_device_memory_on_a_hope_shaped_image():
    H, W, n = 1080, 1920, 100
    rgb, counts, boxes, idx = _case(H, W, n, 1, seed=77)
    flat = np.concatenate([np.asarray(c, np.int32) for c in counts])
    off = np.concatenate([[0], np.cumsum([len(c) for c in counts])])
    dense = torch.stack([torch.as_tensor(rle_to_binary_mask(dict(size=[H, W], counts=c))) for c in counts]).float()

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = fn()
        torch.cuda.synchronize()
        used = torch.cuda.max_memory_allocated() - base
        nbytes = sum(v.numel() * v.element_size() for v in out.values())
        del out
        return used, nbytes

    rle_peak, outputs = peak(lambda: crop_detections_rle(rgb.to(DEV), flat, off, boxes, idx))
    dense_peak, _ = peak(lambda: preprocess_queries(rgb.to(DEV).permute(0, 3, 1, 2), dense.to(DEV),
                                                    torch.as_tensor(boxes), torch.as_tensor(idx)))
    print("bop_run_memory", json.dumps(dict(rle_peak=rle_peak, dense_peak=dense_peak, outputs=outputs)))
    assert rle_peak < outputs + (64 << 20)
    assert dense_peak - rle_peak >= n * H * W * 4


# ---------------------------------------------------------------------------------------------------- end to end
def write_rgb(root, scene_id, im_id, rgb, split="test"):
    """An 8-bit RGB image at <split>/<scene>/rgb/<im>.png (the test images the runner reads)."""
    from PIL import Image
    d = os.path.join(root, split, f"{scene_id:06d}", "rgb")
    os.makedirs(d, exist_ok=True)
    Image.fromarray(np.asarray(rgb, np.uint8)).save(os.path.join(d, f"{im_id:06d}.png"))


K_SCENE = np.array([[600.0, 0, 320.0], [0, 600.0, 240.0], [0, 0, 1]])


def _synthetic_tree(root, rng):
    """A 'ycbv' tree of two objects and three RGB images rendered at the ground-truth poses, with a CNOS-style
    detection file of RLE-encoded render masks (list and compressed-string counts, one distractor per image)."""
    ds = os.path.join(root, "ycbv")
    models = {1: tetra(60.0), 2: spheroid(40.0, 25.0, 12, 24)}
    info = {o: dict(diameter=float(np.linalg.norm(V.max(0) - V.min(0)))) for o, (V, _) in models.items()}
    scenes, dets, targets = {1: {}}, [], []
    H, W = 480, 640
    for im in range(3):
        rgb = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
        depth = np.zeros((H, W), np.uint16)
        gts = []
        for j, (o, (V, F)) in enumerate(models.items()):
            pose = np.eye(4, dtype=np.float32)
            pose[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
            if np.linalg.det(pose[:3, :3]) < 0:
                pose[:3, 0] *= -1
            pose[:3, 3] = [(-120.0 if j == 0 else 120.0) + rng.uniform(-20, 20), rng.uniform(-40, 40), 700.0]
            r = render.render_templates(dict(vertices=V, faces=F, constant_color=[0.9, 0.6, 0.3]),
                                        torch.as_tensor(pose)[None], K_SCENE, size=(H, W), device=DEV)
            a = r["rgba"][0, 3].cpu().numpy() > 0.5
            col = (r["rgba"][0, :3].permute(1, 2, 0).cpu().numpy() * 255).round().astype(np.uint8)
            rgb[a] = col[a]
            depth[a] = np.round(r["depth"][0].cpu().numpy()[a]).astype(np.uint16)
            gts.append((o, pose[:3, :3], pose[:3, 3]))
            x1, y1, x2, y2 = r["boxes"][0].tolist()
            counts = binary_mask_to_rle(a)["counts"]
            dets.append(dict(scene_id=1, image_id=im, category_id=o, score=0.9 - 0.1 * j, time=0.2 + 0.01 * im,
                             bbox=[x1, y1, x2 - x1, y2 - y1],
                             segmentation=dict(size=[H, W], counts=counts if j == 0 else rle_to_string(counts))))
            targets.append((1, im, o, 1))
        blob = np.zeros((H, W), bool)
        blob[200:260, 300:380] = True
        dets.append(dict(scene_id=1, image_id=im, category_id=1, score=0.3, time=0.2 + 0.01 * im,
                         bbox=[300.0, 200.0, 80.0, 60.0], segmentation=dict(size=[H, W], counts=binary_mask_to_rle(blob)["counts"])))
        write_rgb(ds, 1, im, rgb)
        scenes[1][im] = dict(gt=gts, visib=[1.0, 1.0], K=K_SCENE, depth_scale=1.0, png=depth)
    write_tree(ds, models, info, scenes, targets)
    with open(os.path.join(ds, "test_targets_bop24.json"), "w") as f:
        json.dump([dict(scene_id=1, im_id=im) for im in range(3)], f)
    d = os.path.join(root, "default_detections", "core19_model_based_unseen", "cnos-fastsam")
    os.makedirs(d)
    with open(os.path.join(d, "cnos-fastsam_ycbv-test_synthetic.json"), "w") as f:
        json.dump(dets, f)
    return ds


def _hand_driven(model, ds, setting, out):
    """The loop without the runner's RLE path: dense decoded masks through `preprocess_queries`, then eval_retrieval and
    the csv writer."""
    import src.megapose.utils.tensor_collection as tc
    from PIL import Image
    from src.utils.inout import save_predictions_from_batched_predictions
    p = bop_run.plan(ds, setting)
    os.makedirs(os.path.join(out, "predictions"))
    model.log_dir = out
    for i, (s, im) in enumerate(p["images"]):
        key = f"{s:06d}_{im:06d}"
        rgb = np.asarray(Image.open(os.path.join(ds, "test", f"{s:06d}", "rgb", f"{im:06d}.png")))
        dets, tl = p["detections"][key], p["test_list"][key]
        H, W = rgb.shape[:2]
        masks = []
        for d in dets:
            c = d["segmentation"]["counts"]
            c = bop_run.rle_from_string(c) if isinstance(c, str) else c
            masks.append(torch.as_tensor(rle_to_binary_mask(dict(size=[H, W], counts=c))).float())
        n = len(dets)
        q = preprocess_queries(torch.as_tensor(rgb).permute(2, 0, 1)[None].to(DEV), torch.stack(masks).to(DEV),
                               bop_run.xywh_to_xyxy([d["bbox"] for d in dets]), torch.zeros(n, dtype=torch.int64))
        infos = pd.DataFrame(dict(label=[str(d["category_id"]) for d in dets], scene_id=[s] * n, view_id=[im] * n,
                                  batch_im_id=np.zeros(n, np.int64)))
        K = torch.as_tensor(p["cameras"][s][im]).float().to(DEV).expand(n, 3, 3).contiguous()
        batch = tc.PandasTensorCollection(infos=infos, tar_img=q["tar_img"], tar_mask=q["tar_mask"], tar_K=K,
                                          tar_M=q["tar_M"])
        batch.test_list = tc.PandasTensorCollection(infos=pd.DataFrame(dict(
            im_id=[im] * len(tl), scene_id=[s] * len(tl), obj_id=[t["obj_id"] for t in tl],
            inst_count=[t["inst_count"] for t in tl], detection_time=[dets[0]["time"]] * len(tl))))
        model.eval_retrieval(batch, idx_batch=i, dataset_name=p["name"])
    save_predictions_from_batched_predictions(os.path.join(out, "predictions"), dataset_name=p["name"],
                                              model_name=model.model_name, run_id="hand", is_refined=False)
    return os.path.join(out, "predictions", f"large-pbrreal-rgb-mmodel_{p['name']}-test_hand.csv")


def _rows(path):
    with open(path) as f:
        return [line.split(",") for line in f.read().splitlines()[1:]]


def test_run_writes_the_csv_of_a_hand_driven_run(tmp_path):
    from gigapose_b200.synth import fibonacci_view_poses
    rng = np.random.default_rng(9)
    ds = _synthetic_tree(str(tmp_path), rng)
    np.save(str(tmp_path / "poses.npy"), fibonacci_view_poses(24, 400.0).numpy())
    model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)
    det_time = {(1, im): 0.2 + 0.01 * im for im in range(3)}
    for setting in ("localization", "detection"):
        out = str(tmp_path / f"run_{setting}")
        csv = bop_run.run(model, ds, out, setting, template_poses=str(tmp_path / "poses.npy"))
        hand = _hand_driven(model, ds, setting, str(tmp_path / f"hand_{setting}"))
        got, want = _rows(csv), _rows(hand)
        assert len(got) == (6 if setting == "localization" else 9) and len(got) == len(want)
        assert [r[:6] for r in got] == [r[:6] for r in want]       # scene, image, object, score, R, t
        for r in got:
            assert float(r[6]) >= det_time[(int(r[0]), int(r[1]))]
        if setting == "localization":
            res = bop_eval.evaluate(csv, ds, "test", device=DEV)
            scores = [res["ar"], res["ar_vsd"], res["ar_mssd"], res["ar_mspd"]]
        else:
            res = bop_eval.evaluate_detection(csv, ds, "test", device=DEV)
            scores = [res["map"], res["map_mssd"], res["map_mspd"]]
        print("bop_run_e2e", setting, json.dumps(scores))
        assert all(np.isfinite(scores))
    with pytest.raises(bop_run.BopRunError, match="already holds prediction files"):
        bop_run.run(model, ds, str(tmp_path / "run_detection"), "detection")
