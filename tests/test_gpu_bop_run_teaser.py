"""Row f13 end to end: `bop_run --refine-depth H --depth-refiner teaserpp` on the synthetic LM-O tree of
tests/test_gpu_bop_run_masked.py, and `GigaPose.refine_depth(refiner="teaserpp", rank=True)` on planted hypotheses."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

from gigapose_b200 import _lib, bop_eval, bop_run, icp, teaser
from icp_scenes import DEV, perturb
from test_gpu_bop_run_masked import _occluded_lmo_tree
from test_gpu_depth_score import OBJECTS, _rows

pytestmark = pytest.mark.gpu


def test_bop_run_with_the_teaserpp_refiner(tmp_path):
    import src.megapose.utils.tensor_collection as tc
    from gigapose_b200.synth import fibonacci_view_poses
    ds, truths, _ = _occluded_lmo_tree(str(tmp_path))
    np.save(str(tmp_path / "poses.npy"), fibonacci_view_poses(24, 400.0).numpy())
    model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)
    plain = bop_run.run(model, ds, str(tmp_path / "plain"), template_poses=str(tmp_path / "poses.npy"))
    t_out, i_out = str(tmp_path / "teaser"), str(tmp_path / "icp")
    coarse, tcsv = bop_run.run(model, ds, t_out, refine_hypotheses=2, depth_refiner="teaserpp")
    _, icsv = bop_run.run(model, ds, i_out, refine_hypotheses=2)            # the ICP path still runs
    assert tcsv.endswith("_bop_run_teaserpp.csv") and icsv.endswith("_bop_run_icp.csv")
    assert os.path.dirname(tcsv) == os.path.join(t_out, "refined_predictions") and os.path.exists(tcsv)
    c_rows, t_rows, i_rows, p_rows = _rows(coarse), _rows(tcsv), _rows(icsv), _rows(plain)
    assert len(t_rows) == len(i_rows) == 4
    assert [r[:6] for r in c_rows] == [r[:6] for r in p_rows]                 # the coarse csv: every column but `time`
    assert [r[:3] for r in t_rows] == [r[:3] for r in i_rows]                 # scene, image, dataset object id
    for c, r in zip(c_rows, t_rows):
        assert float(r[6]) > float(c[6])                                     # time + refinement_time
    statuses = []
    for i in range(2):
        cn = np.load(os.path.join(t_out, "predictions", f"{i}.npz"))
        rn = np.load(os.path.join(t_out, "refined_predictions", f"{i}.npz"))
        assert "teaser_status" in rn.files and "icp_status" not in rn.files
        for j, hyp in enumerate(rn["hypothesis"]):
            same = np.array_equal(rn["poses"][j].view(np.int32), cn["poses"][j, hyp].view(np.int32))
            assert same == (rn["teaser_status"][j] != _lib.TEASER_OK)
            statuses.append(int(rn["teaser_status"][j]))
    print("teaserpp statuses of the chosen hypotheses:", statuses)
    with pytest.raises(bop_run.BopRunError, match="no masks"):
        bop_run.run(model, ds, str(tmp_path / "never"), refine_hypotheses=2, refine_masks=True,
                    depth_refiner="teaserpp")

    # --- refine_depth(refiner="teaserpp", rank=True) on planted hypotheses equals refine_teaserpp + score_hypotheses
    p = bop_run.plan(ds, depth=True)
    s, im = p["images"][0]
    objs = list(OBJECTS)
    poses = np.stack([np.stack([perturb(truths[(im, o)], [0.2, 1, 0.4], 4.0, [6.0, -5.0, 9.0]),
                                perturb(truths[(im, o)], [1, 0, 0], 0.0, [0.0, 0.0, 12.0]),
                                perturb(truths[(im, o)], [-0.4, 0.2, 1], 3.0, [5.0, 4.0, -8.0])]) for o in objs])
    labels = [bop_run.LMO_ID_TO_INDEX[o] for o in objs]
    pred = tc.PandasTensorCollection(
        infos=pd.DataFrame(dict(label=[str(v) for v in labels], scene_id=[s] * 2, view_id=[im] * 2)),
        pred_poses=torch.as_tensor(poses).to(DEV), scores=torch.tensor([[0.9, 0.8, 0.7], [0.7, 0.6, 0.5]], device=DEV))
    depth = torch.as_tensor(bop_eval.load_depth(ds, "test", s, im, p["depth_scale"][s][im]), device=DEV)
    K = torch.as_tensor(p["cameras"][s][im], dtype=torch.float64).float()
    out = model.refine_depth("lmo", pred, depth, hypotheses=2, K=K, rank=True, refiner="teaserpp")
    for name in ("teaser_status", "teaser_inliers", "teaser_clique", "depth_score"):
        assert tuple(getattr(out, name).shape) == (2, 2), name
    assert tuple(out.depth_counts.shape) == (2, 2, 4) and tuple(out.best_hypothesis.shape) == (2,)
    assert not hasattr(out, "icp_status")
    meshes = model.meshes["lmo"]
    lab = np.repeat(np.asarray(labels) - 1, 2)
    ref = teaser.refine_teaserpp(meshes, lab, pred.pred_poses[:, :2].reshape(-1, 4, 4), depth, K, np.zeros(4, np.int64))
    assert torch.equal(out.pred_poses[:, :2].reshape(-1, 4, 4), ref[0])
    assert torch.equal(out.pred_poses[:, 2], pred.pred_poses[:, 2])           # hypotheses past h untouched
    assert torch.equal(out.teaser_status.reshape(-1), ref[1]) and torch.equal(out.teaser_inliers.reshape(-1), ref[2])
    counts, score, best = icp.score_hypotheses(meshes, lab, ref[0], depth, K, np.zeros(4, np.int64), 2)
    assert torch.equal(out.depth_score.reshape(-1), score) and torch.equal(out.best_hypothesis, best.to(torch.int64))
    with pytest.raises(ValueError, match="no masks"):
        model.refine_depth("lmo", pred, depth, hypotheses=2, K=K, refiner="teaserpp", masks=torch.ones(2, *depth.shape))
