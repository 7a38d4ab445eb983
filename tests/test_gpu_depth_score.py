"""Row f10 on the GPU: gp_depth_score bit for bit against its numpy restatement (oracle/depth_score_port.py), the ranking
of refined hypotheses on rendered scenes, `GigaPose.refine_depth(rank=...)`, and a depth-refined `bop_run` on a
synthetic LM-O tree.  The scenes are synthetic: they show that the plumbing and the selection work, not accuracy on BOP
data."""
import itertools
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from bop_tree import tetra, write_tree
from gigapose_b200 import _lib, bop_eval, bop_run, icp
from icp_scenes import (DEV, H, K, T_ASM, T_ELL, W, assembly, ellipsoid, noisy_occluded_scene, perturb, pose, render_depth,
                        rot, scene)
from oracle.bop_run_port import binary_mask_to_rle
from oracle.depth_score_port import depth_score

pytestmark = pytest.mark.gpu


def _kernel(frame_idx, depth, rendered, boxes, tol, n_hyp):
    """gp_depth_score through the ABI on host arrays -> host arrays."""
    n = len(rendered)
    F, Hh, Ww = depth.shape
    dev = [torch.as_tensor(np.ascontiguousarray(a)).to(DEV) for a in
           (np.asarray(frame_idx, np.int32), depth, rendered, np.asarray(boxes, np.int64))]
    counts = torch.full((n, 4), -7, dtype=torch.int32, device=DEV)
    score = torch.full((n,), -7.0, device=DEV)
    best = torch.full((n // n_hyp,), -7, dtype=torch.int32, device=DEV)
    _lib.check(_lib.load().gp_depth_score(F, n // n_hyp, n_hyp, Hh, Ww, *[t.data_ptr() for t in dev], float(tol),
                                          counts.data_ptr(), score.data_ptr(), best.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return counts.cpu().numpy(), score.cpu().numpy(), best.cpu().numpy()


def _same(got, want):
    for name, g, w in zip(("counts", "score", "best"), got, want):
        assert g.dtype == w.dtype and g.shape == w.shape, name
        assert np.array_equal(g.view(np.int32), w.view(np.int32)), f"{name}: {int((g.view(np.int32) != w.view(np.int32)).sum())} differ"


def _maps(rng, Hh, Ww, n_det, n_hyp, F=3):
    """Integer-valued measured depths (so that a planted offset of 15 is a difference of exactly 15 in fp32) with 0,
    negative and NaN pixels; renders = the frame's depth plus offsets from {0, +-15, +-16, +-300}, 40 % background."""
    n = n_det * n_hyp
    depth = rng.integers(500, 1500, (F, Hh, Ww)).astype(np.float32)
    hole = rng.random(depth.shape)
    depth[hole < 0.05] = 0
    depth[(hole >= 0.05) & (hole < 0.07)] = -20.0
    depth[(hole >= 0.07) & (hole < 0.09)] = np.nan
    frame_idx = rng.integers(0, F, n_det)
    base = np.nan_to_num(np.abs(depth[np.repeat(frame_idx, n_hyp)]), nan=700.0)
    rendered = (base + rng.choice(np.array([0, 15, -15, 16, -16, 300, -300], np.float32), (n, Hh, Ww))).astype(np.float32)
    rendered[rng.random(rendered.shape) < 0.4] = 0
    x0, y0 = rng.integers(-5, Ww - 1, n), rng.integers(-5, Hh - 1, n)
    boxes = np.stack([x0, y0, x0 + rng.integers(1, Ww, n), y0 + rng.integers(1, Hh, n)], 1).astype(np.int64)
    special = [[0, 0, Ww, Hh], [0, 3, 5, Hh - 2], [2, 0, Ww - 3, 4], [Ww - 6, 1, Ww, Hh - 1], [1, Hh - 4, Ww - 1, Hh],
               [-9, -9, Ww + 9, Hh + 9], [4, 4, 4, 9], [9, 4, 3, 9], [4, 9, 9, 2], [Ww + 3, 0, Ww + 9, 5], [6, 7, 7, 8]]
    for i, b in enumerate(special[:n]):
        boxes[n - 1 - i] = b
    if n > 1:
        rendered[0] = 0                                       # an all-background render: score 0
    return frame_idx, depth, rendered, boxes


@pytest.mark.parametrize("Hh,Ww,n_det,n_hyp", [(17, 17, 1, 1), (17, 17, 11, 3), (480, 640, 100, 1), (480, 640, 37, 3),
                                               (480, 640, 20, 5), (1080, 1920, 4, 5), (1080, 1920, 1, 3)])
def test_kernel_matches_the_port_bit_for_bit(Hh, Ww, n_det, n_hyp):
    rng = np.random.default_rng(Hh + n_det)
    frame_idx, depth, rendered, boxes = _maps(rng, Hh, Ww, n_det, n_hyp)
    seen = np.zeros(4, np.int64)
    results = []
    # differences of exactly 15 in both directions, with the tolerance at 15 and one float32 ulp either side of it
    for tol in (np.float32(15), np.nextafter(np.float32(15), np.float32(16)), np.nextafter(np.float32(15), np.float32(0))):
        got = _kernel(frame_idx, depth, rendered, boxes, tol, n_hyp)
        _same(got, depth_score(frame_idx, depth, rendered, boxes, tol, n_hyp))
        seen += got[0].sum(0)
        results.append(got[0])
    assert (seen > 0).all(), seen                             # consistent, behind, front and missing all occur
    assert np.array_equal(results[0], results[1]) and not np.array_equal(results[0], results[2])
    assert results[2][:, 0].sum() < results[0][:, 0].sum()    # below the tolerance, the +-15 pixels leave `consistent`
    if len(rendered) > 1:
        assert got[0][0].tolist() == [0, 0, 0, 0] and got[1][0] == 0


def test_ties_go_to_the_lowest_index_and_an_invalid_frame_is_marked():
    depth = np.full((1, 20, 20), 100, np.float32)
    depth[0, 15:] = 0
    P, Q, R = (np.zeros((20, 20), np.float32) for _ in range(3))
    P[:10], Q[:5], R[:] = 100, 100, 200                        # P and Q score 1 with different counts, R scores 0
    Q[15:] = 100                                               # missing pixels do not change Q's score
    orders = [(R, P, Q), (R, Q, P), (P, Q, R), (Q, P, R), (R, R, R)]
    rendered = np.stack([m for o in orders for m in o])
    boxes = np.tile(np.array([0, 0, 20, 20], np.int64), (len(rendered), 1))
    got = _kernel([0] * len(orders), depth, rendered, boxes, 15.0, 3)
    _same(got, depth_score([0] * len(orders), depth, rendered, boxes, 15.0, 3))
    assert got[2].tolist() == [1, 1, 0, 0, 0]
    assert got[0][1].tolist() == [200, 0, 0, 0] and got[0][2].tolist() == [100, 0, 0, 100]
    assert got[1][:3].tolist() == [0.0, 1.0, 1.0] and got[0][0].tolist() == [0, 0, 300, 100]
    bad = _kernel([0, 1, -1, 0, 0], depth, rendered, boxes, 15.0, 3)
    _same(bad, depth_score([0, 1, -1, 0, 0], depth, rendered, boxes, 15.0, 3))
    assert bad[2].tolist() == [1, -1, -1, 0, 0] and (bad[0][3:9] == -1).all() and np.isnan(bad[1][3:9]).all()


def test_one_launch_per_call():
    lib = _lib.load()
    rng = np.random.default_rng(5)
    for n_det, n_hyp in ((1, 1), (100, 5)):
        args = _maps(rng, 64, 48, n_det, n_hyp)
        before = lib.gp_launch_count()
        _kernel(*args, 15.0, n_hyp)
        assert lib.gp_launch_count() - before == 1


# ---------------------------------------------------------------------------------------------------- ranking
def _errors(T, Tt):
    dR = T[:3, :3].astype(np.float64) @ Tt[:3, :3].astype(np.float64).T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    return float(np.linalg.norm(T[:3, 3].astype(np.float64) - Tt[:3, 3])), float(ang)


def _hypotheses(Tt):
    """[truth turned 180 degrees about the view axis and shifted 8 mm, truth off by 4 degrees / 6 mm, truth pushed onto
    the background plane]: index 1 is the good one."""
    return [perturb(Tt, [0, 0, 1], 180.0, [0.0, 0.0, 8.0]), perturb(Tt, [1, 0.2, 0.3], 4.0, [3.0, -4.0, 3.3]),
            perturb(Tt, [0, 1, 0], 5.0, [0.0, 0.0, 150.0])]


def _rank(mesh, hyps, d):
    """Every order of the three hypotheses as one detection each: refine_icp (no masks) then score_hypotheses."""
    orders = list(itertools.permutations(range(3)))
    T0 = torch.as_tensor(np.stack([hyps[j] for o in orders for j in o])).to(DEV)
    dm = icp.device_meshes([mesh], DEV)
    n = len(T0)
    out, st, _, _ = icp.refine_icp(dm, np.zeros(n, np.int64), T0, d, torch.as_tensor(K), np.zeros(n, np.int64))
    counts, score, best = icp.score_hypotheses(dm, np.zeros(n, np.int64), out, d, torch.as_tensor(K),
                                               np.zeros(n, np.int64), 3)
    return orders, out.cpu().numpy().reshape(-1, 3, 4, 4), st.cpu().numpy().reshape(-1, 3), \
        counts.cpu().numpy().reshape(-1, 3, 4), score.cpu().numpy().reshape(-1, 3), best.cpu().numpy()


@pytest.mark.parametrize("name,bar_deg,margin_bar", [("ellipsoid", 0.1, 0.6), ("assembly", 0.2, 0.4)])
def test_the_refined_good_hypothesis_wins_in_every_order(name, bar_deg, margin_bar):
    """The bars on the winner's pose are those of test_gpu_icp.py's noiseless scenes.  Measured on an H100: the good
    hypothesis scores 0.999 / 0.998 (ellipsoid / assembly), the flipped one 0.255 / 0.521 after its own refinement, the
    one on the background plane 0.000 / 0.012; the smallest margins are 0.744 and 0.477."""
    mesh, Tt = (ellipsoid(), T_ELL) if name == "ellipsoid" else (assembly(), T_ASM)
    d, _ = scene(mesh, Tt)
    orders, out, st, counts, score, best = _rank(mesh, _hypotheses(Tt), d)
    margins = []
    for i, o in enumerate(orders):
        good = o.index(1)
        assert int(best[i]) == good, (o, score[i])
        assert int(st[i, good]) == _lib.ICP_OK
        et, er = _errors(out[i, good], Tt)
        assert et < 0.5 and er < bar_deg, (et, er)
        margins.append(float(score[i, good] - np.delete(score[i], good).max()))
    by_hyp = {j: float(score[0, orders[0].index(j)]) for j in range(3)}
    print(f"depth_score_margin {name}: scores flipped {by_hyp[0]:.4f} good {by_hyp[1]:.4f} background {by_hyp[2]:.4f}, "
          f"smallest margin {min(margins):.4f}")
    assert min(margins) > margin_bar
    same = np.stack([_hypotheses(Tt)[1]] * 3)
    dm = icp.device_meshes([mesh], DEV)
    _, s, b = icp.score_hypotheses(dm, np.zeros(3, np.int64), torch.as_tensor(same).to(DEV), d, torch.as_tensor(K),
                                   np.zeros(3, np.int64), 3)
    assert int(b[0]) == 0 and float(s[0]) == float(s[1]) == float(s[2])


def test_occlusion_does_not_flip_the_ranking():
    """sigma = 1 mm noise, 10 % missing pixels and an occluder over 30 % of the object: the occluder's pixels count as
    `front` for every hypothesis, the holes as `missing`, and the good hypothesis still wins in every order (measured
    on an H100: by 0.469 at least; its counts are 4881 consistent, 83 behind, 2276 front, 516 missing)."""
    mesh = ellipsoid()
    d, _ = noisy_occluded_scene(mesh, T_ELL)
    orders, out, st, counts, score, best = _rank(mesh, _hypotheses(T_ELL), d)
    margins = []
    for i, o in enumerate(orders):
        good = o.index(1)
        assert int(best[i]) == good, (o, score[i])
        assert (counts[i, :, 2] > 0).all() and (counts[i, :, 3] > 0).all()
        assert counts[i, good, 2] > 0.15 * counts[i, good].sum()
        margins.append(float(score[i, good] - np.delete(score[i], good).max()))
    print(f"depth_score_margin occluded ellipsoid: smallest margin {min(margins):.4f}, good counts "
          f"{counts[0, orders[0].index(1)].tolist()}")
    assert min(margins) > 0.4


# ---------------------------------------------------------------------------------------------------- refine_depth
def _bits(t):
    return t.contiguous().view(torch.uint8) if t.dtype != torch.bool else t


def test_refine_depth_rank_adds_three_tensors_and_changes_nothing_else(tmp_path):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    dev = torch.device(DEV)
    model = bench.build_models(dev)
    model.log_dir = str(tmp_path)
    templates = bench.SyntheticTemplates(2, 8, dev)
    model.template_datasets = {"synthetic": templates}
    batch, _, _ = bench.make_queries(templates, 3, seed=4)
    pred = model.retrieve(batch, "synthetic")
    meshes = [ellipsoid(), assembly()]
    model.attach_meshes("synthetic", meshes)
    lab = np.asarray(pred.infos.label).astype(int) - 1
    truths = [T_ELL if o == 0 else T_ASM for o in lab]
    depth = torch.stack([scene(meshes[o], T)[0] for o, T in zip(lab, truths)])
    k = pred.pred_poses.shape[1]
    # hypothesis 1 is the good one; 0 is flipped, the rest lie behind the background plane
    coarse = torch.stack([torch.as_tensor(np.stack(
        [_hypotheses(T)[0], _hypotheses(T)[1]] + [perturb(T, [1, 0.2, 0.3], 9.0 + 3 * j, [20.0, -2.0, 200.0 + 9 * j])
                                                  for j in range(k - 2)])) for T in truths]).to(dev)
    pred.pred_poses = coarse
    Kf = torch.as_tensor(K).expand(len(lab), 3, 3)
    frames = np.arange(len(lab))
    for h in (1, 3):
        plain = model.refine_depth("synthetic", pred, depth, frames, hypotheses=h, K=Kf)
        off = model.refine_depth("synthetic", pred, depth, frames, hypotheses=h, K=Kf, rank=False)
        on = model.refine_depth("synthetic", pred, depth, frames, hypotheses=h, K=Kf, rank=True)
        assert set(off._tensors) == set(plain._tensors)
        assert set(on._tensors) - set(plain._tensors) == {"depth_counts", "depth_score", "best_hypothesis"}
        assert "depth_score" not in pred._tensors
        for name, t in plain._tensors.items():
            assert torch.equal(_bits(t), _bits(off._tensors[name])) and torch.equal(_bits(t), _bits(on._tensors[name])), name
        assert on.depth_counts.shape == (len(lab), h, 4) and on.depth_counts.dtype == torch.int32
        assert on.depth_score.shape == (len(lab), h) and on.best_hypothesis.dtype == torch.int64
        assert on.best_hypothesis.tolist() == [0 if h == 1 else 1] * len(lab)
        # scored on the final poses: the same numbers from score_hypotheses on pred_poses[:, :h]
        c, s, b = icp.score_hypotheses(model.meshes["synthetic"], np.repeat(lab, h), on.pred_poses[:, :h].reshape(-1, 4, 4),
                                       depth, Kf, np.repeat(frames, h), h)
        assert torch.equal(c.reshape(-1, h, 4), on.depth_counts) and torch.equal(s.reshape(-1, h), on.depth_score)
        assert torch.equal(b.long(), on.best_hypothesis)


# ---------------------------------------------------------------------------------------------------- bop_run
K_SCENE = np.array([[600.0, 0, 320.0], [0, 600.0, 240.0], [0, 0, 1]])
OBJECTS = {5: (ellipsoid, [-110.0, -10.0, 700.0], [0.3, 1.0, 0.2], 35.0),
           9: (assembly, [120.0, 30.0, 760.0], [1.0, -0.4, 0.5], 50.0)}


def _lmo_tree(root, n_images=2):
    """An 'lmo' tree (the eight LM-O object ids, so that the index -> id remap is exercised): objects 5 and 9 stand in
    front of a plane in every image; RGB, 16-bit depth in mm, and CNOS-style detections of the render masks."""
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
    scenes, dets, targets, truths = {2: {}}, [], [], {}
    rng = np.random.default_rng(2)
    for im in range(n_images):
        depth = render_depth(plane, np.eye(4, dtype=np.float32), Kf)
        rgb = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
        gts = []
        for j, (o, (_, t, axis, deg)) in enumerate(OBJECTS.items()):
            T = pose(rot(axis, deg + 20 * im), np.asarray(t) + [0.0, 10.0 * im, 15.0 * im])
            dobj = render_depth(meshes[o], T, Kf)
            a = (dobj > 0).cpu().numpy()
            depth = torch.where(dobj > 0, dobj, depth)
            rgb[a] = (40 + 90 * j, 200 - 60 * j, 90)
            ys, xs = np.nonzero(a)
            dets.append(dict(scene_id=2, image_id=im, category_id=o, score=0.9 - 0.1 * j, time=0.25 + 0.01 * im,
                             bbox=[int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1)],
                             segmentation=dict(size=[H, W], counts=binary_mask_to_rle(a)["counts"])))
            gts.append((o, T[:3, :3], T[:3, 3]))
            targets.append((2, im, o, 1))
            truths[(im, o)] = T
        d = os.path.join(ds, "test", "000002", "rgb")
        os.makedirs(d, exist_ok=True)
        Image.fromarray(rgb).save(os.path.join(d, f"{im:06d}.png"))
        scenes[2][im] = dict(gt=gts, visib=[1.0] * len(gts), K=K_SCENE, depth_scale=1.0,
                             png=np.round(depth.cpu().numpy()).astype(np.uint16))
    write_tree(ds, models, info, scenes, targets)
    d = os.path.join(root, "default_detections", "core19_model_based_unseen", "cnos-fastsam")
    os.makedirs(d)
    with open(os.path.join(d, "cnos-fastsam_lmo-test_synthetic.json"), "w") as f:
        json.dump(dets, f)
    return ds, truths


def _rows(path):
    with open(path) as f:
        return [line.split(",") for line in f.read().splitlines()[1:]]


def test_bop_run_with_depth_refinement(tmp_path):
    import src.megapose.utils.tensor_collection as tc
    from gigapose_b200.synth import fibonacci_view_poses
    from src.utils.inout import save_predictions_from_batched_predictions
    ds, truths = _lmo_tree(str(tmp_path))
    np.save(str(tmp_path / "poses.npy"), fibonacci_view_poses(24, 400.0).numpy())
    model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)

    # --- the runner with seeded weights: the plumbing, whatever the ICP makes of junk poses
    plain = bop_run.run(model, ds, str(tmp_path / "plain"), template_poses=str(tmp_path / "poses.npy"))
    out = str(tmp_path / "refined_run")
    coarse, refined = bop_run.run(model, ds, out, refine_hypotheses=2)
    assert isinstance(plain, str) and os.path.exists(coarse) and os.path.exists(refined)
    assert refined.endswith("_bop_run_icp.csv") and os.path.dirname(refined) == os.path.join(out, "refined_predictions")
    c_rows, r_rows, p_rows = _rows(coarse), _rows(refined), _rows(plain)
    assert len(c_rows) == len(r_rows) == 4
    assert [r[:6] for r in c_rows] == [r[:6] for r in p_rows]                # every column but `time`
    assert [r[:3] for r in c_rows] == [r[:3] for r in r_rows]                # scene, image, dataset object id
    assert sorted({int(r[2]) for r in r_rows}) == [5, 9]
    statuses = []
    for i in range(2):
        cn = np.load(os.path.join(out, "predictions", f"{i}.npz"))
        rn = np.load(os.path.join(out, "refined_predictions", f"{i}.npz"))
        assert rn["object_id"].tolist() == [bop_run.LMO_INDEX_TO_ID[v - 1] for v in cn["object_id"]]
        assert rn["poses"].shape == (len(cn["poses"]), 4, 4) and (rn["hypothesis"] < 2).all()
        for j, hyp in enumerate(rn["hypothesis"]):
            same = np.array_equal(rn["poses"][j].view(np.int32), cn["poses"][j, hyp].view(np.int32))
            assert same == (rn["icp_status"][j] != _lib.ICP_OK), (i, j, rn["icp_status"][j])
            assert rn["scores"][j] == cn["scores"][j, hyp]
            statuses.append(int(rn["icp_status"][j]))
        rt = float(rn["refinement_time"][0])
        assert rt > 0 and (rn["refinement_time"] == rt).all()
        for c, r in zip(c_rows[2 * i:2 * i + 2], r_rows[2 * i:2 * i + 2]):
            assert float(r[6]) == pytest.approx(float(c[6]) + rt, rel=1e-9)
    print("bop_refine_e2e icp statuses with seeded weights:", statuses)
    with pytest.raises(bop_run.BopRunError, match="already holds prediction files"):
        bop_run.run(model, ds, out, refine_hypotheses=2)
    with pytest.raises(bop_run.BopRunError, match="refine_hypotheses 6"):
        bop_run.run(model, ds, str(tmp_path / "never"), refine_hypotheses=6)

    # --- planted predictions through refine_image: hypothesis 0 is the flipped pose on half of the detections
    p = bop_run.plan(ds, depth=True)
    planted = str(tmp_path / "planted")
    os.makedirs(os.path.join(planted, "predictions"))
    expect = []
    for i, (s, im) in enumerate(p["images"]):
        objs = list(OBJECTS)
        hyps = [_hypotheses(truths[(im, o)]) for o in objs]
        flip_first = [(i + j) % 2 == 0 for j in range(len(objs))]
        poses = np.stack([np.stack([h[0], h[1]] if f else [h[1], h[0]]) for h, f in zip(hyps, flip_first)])
        expect.append([1 if f else 0 for f in flip_first])
        labels = [bop_run.LMO_ID_TO_INDEX[o] for o in objs]
        pred = tc.PandasTensorCollection(
            infos=pd.DataFrame(dict(label=[str(v) for v in labels], scene_id=[s] * len(objs), view_id=[im] * len(objs))),
            pred_poses=torch.as_tensor(poses).to(DEV), scores=torch.tensor([[0.9, 0.8], [0.7, 0.6]], device=DEV))
        test_list = tc.PandasTensorCollection(infos=pd.DataFrame(dict(obj_id=labels, inst_count=[1] * len(objs),
                                                                      detection_time=[0.25] * len(objs))))
        _, kept = model.filter_and_save(pred, test_list, 0.05, os.path.join(planted, "predictions", f"{i}.npz"))
        depth = bop_eval.load_depth(ds, "test", s, im, p["depth_scale"][s][im])
        ref = bop_run.refine_image(model, p, i, kept, depth, 2, planted)
        assert ref.best_hypothesis.tolist() == expect[-1], (i, ref.depth_score.tolist())
        assert (ref.icp_status[torch.arange(len(objs)), ref.best_hypothesis] == _lib.ICP_OK).all()
    for d, rid, refd in ((os.path.join(planted, "predictions"), "planted", False),
                         (os.path.join(planted, "refined_predictions"), "planted_icp", True)):
        save_predictions_from_batched_predictions(d, dataset_name="lmo", model_name="large", run_id=rid, is_refined=refd)
    res = [bop_eval.evaluate(os.path.join(planted, d, f"large-pbrreal-rgb-mmodel_lmo-test_{rid}.csv"), ds, "test",
                             device=DEV) for d, rid in (("predictions", "planted"), ("refined_predictions", "planted_icp"))]
    print("bop_refine_planted", json.dumps({k: [r[k] for r in res] for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd")}))
    assert res[0]["n_targets"] == res[1]["n_targets"] == 4
    assert res[1]["ar_mssd"] > res[0]["ar_mssd"] and res[1]["ar_vsd"] > res[0]["ar_vsd"]
    assert [int(r[2]) for r in _rows(os.path.join(planted, "refined_predictions",
                                                  "large-pbrreal-rgb-mmodel_lmo-test_planted_icp.csv"))] == [5, 9, 5, 9]
