"""Row f11 end to end: `bop_run --refine-depth H --refine-masks` on a synthetic LM-O tree whose instances stand
partly behind occluders, with the masks CNOS would give (the visible pixels) as run-length encodings."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

from bop_tree import tetra, write_tree
from gigapose_b200 import _lib, bop_eval, bop_run
from icp_scenes import DEV, H, W, perturb, pose, render_depth, rot
from oracle.bop_run_port import binary_mask_to_rle, rle_to_binary_mask
from test_gpu_depth_score import K_SCENE, OBJECTS, _rows
from test_gpu_icp import errors

pytestmark = pytest.mark.gpu


def _occluded_lmo_tree(root, n_images=2):
    """test_gpu_depth_score's LM-O tree with, per instance, a slab 120 mm in front of it over the left 30 % of its
    pixels, sigma = 1 mm noise and 10 % missing pixels; each detection's mask is its visible pixels."""
    from PIL import Image
    ds = os.path.join(root, "lmo")
    models = {o: tetra(40.0 + o) for o in bop_run.LMO_INDEX_TO_ID}
    meshes = {o: f() for o, (f, _, _, _) in OBJECTS.items()}
    for o, m in meshes.items():
        models[o] = (m["vertices"], m["faces"])
    info = {o: dict(diameter=float(np.linalg.norm(V.max(0) - V.min(0)))) for o, (V, _) in models.items()}
    Kf = K_SCENE.astype(np.float32)
    plane = dict(vertices=np.array([[-2e3, -2e3, 950], [2e3, -2e3, 950], [2e3, 2e3, 950], [-2e3, 2e3, 950]], np.float32),
                 faces=np.array([[0, 1, 2], [0, 2, 3]], np.int32))
    scenes, dets, targets, truths, visible = {2: {}}, [], [], {}, {}
    rng = np.random.default_rng(4)
    for im in range(n_images):
        depth = render_depth(plane, np.eye(4, dtype=np.float32), Kf).cpu().numpy()
        rgb = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
        gts = []
        for j, (o, (_, t, axis, deg)) in enumerate(OBJECTS.items()):
            T = pose(rot(axis, deg + 20 * im), np.asarray(t) + [0.0, 10.0 * im, 15.0 * im])
            dobj = render_depth(meshes[o], T, Kf).cpu().numpy()
            a = dobj > 0
            depth = np.where(a, dobj, depth)
            ys, xs = np.nonzero(a)
            x_cut = int(np.sort(xs)[int(0.3 * len(xs))])
            depth[ys.min():ys.max() + 1, xs.min():x_cut] = float(T[2, 3]) - 120.0
            vis = a.copy()
            vis[ys.min():ys.max() + 1, xs.min():x_cut] = False
            rgb[a] = (40 + 90 * j, 200 - 60 * j, 90)
            vy, vx = np.nonzero(vis)
            dets.append(dict(scene_id=2, image_id=im, category_id=o, score=0.9 - 0.1 * j, time=0.25 + 0.01 * im,
                             bbox=[int(vx.min()), int(vy.min()), int(vx.max() - vx.min() + 1), int(vy.max() - vy.min() + 1)],
                             segmentation=dict(size=[H, W], counts=binary_mask_to_rle(vis)["counts"])))
            gts.append((o, T[:3, :3], T[:3, 3]))
            targets.append((2, im, o, 1))
            truths[(im, o)], visible[(im, o)] = T, vis
        depth = depth + rng.normal(size=depth.shape)
        depth[rng.random(depth.shape) < 0.1] = 0
        d = os.path.join(ds, "test", "000002", "rgb")
        os.makedirs(d, exist_ok=True)
        Image.fromarray(rgb).save(os.path.join(d, f"{im:06d}.png"))
        scenes[2][im] = dict(gt=gts, visib=[0.7] * len(gts), K=K_SCENE, depth_scale=1.0,
                             png=np.round(np.clip(depth, 0, None)).astype(np.uint16))
    write_tree(ds, models, info, scenes, targets)
    d = os.path.join(root, "default_detections", "core19_model_based_unseen", "cnos-fastsam")
    os.makedirs(d)
    import json
    with open(os.path.join(d, "cnos-fastsam_lmo-test_synthetic.json"), "w") as f:
        json.dump(dets, f)
    return ds, truths, visible


def test_bop_run_with_masked_refinement(tmp_path):
    import src.megapose.utils.tensor_collection as tc
    from gigapose_b200.synth import fibonacci_view_poses
    from src.utils.inout import save_predictions_from_batched_predictions
    ds, truths, visible = _occluded_lmo_tree(str(tmp_path))
    np.save(str(tmp_path / "poses.npy"), fibonacci_view_poses(24, 400.0).numpy())
    model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)

    # --- the runner with seeded weights: each kept instance gets its own mask, the csv name and layout
    calls, orig = [], model.refine_depth

    def spy(name, kept, depth, **kw):
        calls.append((np.asarray(kept.infos.label).astype(int).tolist(), kw.get("masks"), kw.get("mask_normals", False),
                      tuple(depth.shape), tuple(kw["K"].shape)))
        return orig(name, kept, depth, **kw)
    model.refine_depth = spy
    plain = bop_run.run(model, ds, str(tmp_path / "plain"), template_poses=str(tmp_path / "poses.npy"))
    unmasked_out, masked_out = str(tmp_path / "unmasked"), str(tmp_path / "masked")
    _, unmasked = bop_run.run(model, ds, unmasked_out, refine_hypotheses=2)
    n_unmasked = len(calls)
    coarse, masked = bop_run.run(model, ds, masked_out, refine_hypotheses=2, refine_masks=True)
    model.refine_depth = orig
    assert masked.endswith("_bop_run_icp_masked.csv") and unmasked.endswith("_bop_run_icp.csv")
    assert os.path.dirname(masked) == os.path.join(masked_out, "refined_predictions")
    assert not os.path.exists(os.path.join(masked_out, "refined_predictions", os.path.basename(unmasked)))
    c_rows, m_rows, u_rows, p_rows = _rows(coarse), _rows(masked), _rows(unmasked), _rows(plain)
    assert len(m_rows) == len(u_rows) == 4
    assert [r[:6] for r in c_rows] == [r[:6] for r in p_rows]                 # the coarse csv: every column but `time`
    assert [r[:3] for r in m_rows] == [r[:3] for r in u_rows]                 # scene, image, dataset object id
    assert all(m is None and not mn for _, m, mn, _, _ in calls[:n_unmasked])
    for i, (labels, masks, mask_normals, dshape, kshape) in enumerate(calls[n_unmasked:]):
        assert mask_normals and dshape == (1, H, W) and kshape == (3, 3)
        off = masks["offsets"]
        assert len(off) == len(labels) + 1
        for j, lab in enumerate(labels):
            got = rle_to_binary_mask(dict(size=[H, W], counts=masks["counts"][off[j]:off[j + 1]].tolist()))
            assert np.array_equal(got, visible[(i, bop_run.LMO_INDEX_TO_ID[lab - 1])]), (i, j, lab)
    for i in range(2):
        cn = np.load(os.path.join(masked_out, "predictions", f"{i}.npz"))
        rn = np.load(os.path.join(masked_out, "refined_predictions", f"{i}.npz"))
        rt = float(rn["refinement_time"][0])
        assert rt > 0 and (rn["refinement_time"] == rt).all()
        for j, hyp in enumerate(rn["hypothesis"]):
            same = np.array_equal(rn["poses"][j].view(np.int32), cn["poses"][j, hyp].view(np.int32))
            assert same == (rn["icp_status"][j] != _lib.ICP_OK)
    for c, r in zip(c_rows, m_rows):
        assert float(r[6]) > float(c[6])                                     # time + refinement_time
    with pytest.raises(bop_run.BopRunError, match="refine_masks needs"):
        bop_run.run(model, ds, str(tmp_path / "never"), refine_masks=True)

    # --- planted predictions through refine_image, as `run` calls it: masked against maskless on the occluded instances
    p = bop_run.plan(ds, depth=True)
    outs = {k: str(tmp_path / f"planted_{k}") for k in ("maskless", "masked")}
    err = {k: [] for k in outs}
    for i, (s, im) in enumerate(p["images"]):
        objs = list(OBJECTS)
        poses = np.stack([np.stack([perturb(truths[(im, o)], [0.2, 1, 0.4], 8.0, [9.0, -8.0, 9.0]),
                                    perturb(truths[(im, o)], [-0.4, 0.2, 1], 7.0, [5.0, 9.0, 12.0])]) for o in objs])
        labels = [bop_run.LMO_ID_TO_INDEX[o] for o in objs]
        key = bop_run._key(s, im)
        x = bop_run.image_inputs(p["detections"][key], p["test_list"][key], "lmo", (H, W), key)
        for k, out in outs.items():
            os.makedirs(os.path.join(out, "predictions"), exist_ok=True)
            pred = tc.PandasTensorCollection(
                infos=pd.DataFrame(dict(label=[str(v) for v in labels], scene_id=[s] * 2, view_id=[im] * 2)),
                pred_poses=torch.as_tensor(poses).to(DEV), scores=torch.tensor([[0.9, 0.8], [0.7, 0.6]], device=DEV))
            test_list = tc.PandasTensorCollection(infos=pd.DataFrame(dict(obj_id=labels, inst_count=[1, 1],
                                                                          detection_time=[0.25, 0.25])))
            selected, kept = model.filter_and_save(pred, test_list, 0.05, os.path.join(out, "predictions", f"{i}.npz"))
            depth = bop_eval.load_depth(ds, "test", s, im, p["depth_scale"][s][im])
            masks = bop_run.select_rle((x["counts"], x["offsets"]), selected) if k == "masked" else None
            bop_run.refine_image(model, p, i, kept, depth, 2, out, masks)
            rn = np.load(os.path.join(out, "refined_predictions", f"{i}.npz"))
            for j, o in enumerate(rn["object_id"]):
                err[k].append(errors(rn["poses"][j], truths[(im, int(o))]))
    e = {k: np.array(v) for k, v in err.items()}
    print("planted, per instance (mm, deg):", {k: np.round(v, 3).tolist() for k, v in e.items()})
    assert e["masked"][:, 0].mean() < e["maskless"][:, 0].mean() and e["masked"][:, 1].mean() < e["maskless"][:, 1].mean()
    res = {}
    for k, out in outs.items():
        rid = "planted_icp_masked" if k == "masked" else "planted_icp"
        d = os.path.join(out, "refined_predictions")
        save_predictions_from_batched_predictions(d, dataset_name="lmo", model_name="large", run_id=rid, is_refined=True)
        csv = os.path.join(d, f"large-pbrreal-rgb-mmodel_lmo-test_{rid}.csv")
        res[k] = bop_eval.evaluate(csv, ds, "test", out_dir=os.path.join(out, "refined"), device=DEV)
        bop_run._evaluate(csv, ds, "localization", os.path.join(out, "refined_cli"), DEV)   # what --evaluate runs
    print("planted AR:", {k: {m: r[m] for m in ("ar", "ar_vsd", "ar_mssd", "ar_mspd")} for k, r in res.items()})
    assert res["masked"]["n_targets"] == 4 and np.isfinite(res["masked"]["ar"])
