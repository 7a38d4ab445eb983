"""Row f15 on the GPU, on the synthetic 'ycbv' tree of tests/test_gpu_bop_run.py:

- a run onboarded from the generated test templates (`template_poses.template_poses()`, no --template-poses) against
  one onboarded from the reference's level-1 poses x 0.4 (tests/golden/template_poses.npz);
- `python -m torch.distributed.run --nproc-per-node 2 -m gigapose_b200.bop_run`, both ranks on cuda:0, with and
  without --refine-depth 2, against the one-process run: the csvs byte for byte in every column but `time`, the same
  .npz files, the same --evaluate scores."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gigapose_b200 import bop_run
from test_gpu_bop_run import _synthetic_tree

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEM = "large-pbrreal-rgb-mmodel_ycbv-test_bop_run"


def _rows(path):
    """The csv's lines, each without its `time` column (scene_id,im_id,obj_id,score,R,t,time[,instance_id]; R and t
    are space-separated)."""
    with open(path) as f:
        lines = f.read().split("\n")
    return [",".join(r[:6] + r[7:]) for r in (line.split(",") for line in lines)]


def test_generated_templates_run_as_the_reference_level_1_poses(tmp_path, golden_dir):
    ds = _synthetic_tree(str(tmp_path), np.random.default_rng(9))
    fixture = np.load(os.path.join(golden_dir, "template_poses.npz"))["obj_poses_level1"].copy()
    fixture[:, :3, 3] *= 0.4
    csvs = {}
    for which, poses in (("fixture", fixture), ("generated", None)):
        model = bop_run.build_model(DEV, str(tmp_path / "log"), seed=7)
        csvs[which] = bop_run.run(model, ds, str(tmp_path / which), template_poses=poses)
        assert model.engines["ycbv"].T == 162
        del model
        torch.cuda.empty_cache()
    got, want = _rows(csvs["generated"]), _rows(csvs["fixture"])
    assert len(got) == len(want) == 7
    assert got[0] == want[0]
    # The views within a ring of equal elevation come in another order, and the poses differ from the reference's by
    # up to 7.6e-8 rad / 5.5e-5 mm, so a template may round to other fp32 values: each row must keep its scene, image,
    # object and score to 1e-6, and its pose to 1e-5 (R) and 1e-3 mm (t), or else it retrieved another template.
    worst = np.zeros(3)
    for g, w in zip(got[1:], want[1:]):
        g, w = g.split(","), w.split(",")
        assert g[:3] == w[:3]
        diff = np.abs(np.array(" ".join(g[3:]).split(), float) - np.array(" ".join(w[3:]).split(), float))
        assert diff[1:10].max() < 1e-3, f"row {w[:3]}: the generated templates retrieved another template " \
                                        f"(rotation differs by {diff[1:10].max():.3g})"
        worst = np.maximum(worst, [diff[0], diff[1:10].max(), diff[10:13].max()])
    print("generated_vs_fixture_templates", json.dumps(dict(score=worst[0], R=worst[1], t_mm=worst[2])))
    assert worst[0] < 1e-6 and worst[1] < 1e-5 and worst[2] < 1e-3


@pytest.fixture(scope="module")
def tree_and_checkpoint(tmp_path_factory):
    root = tmp_path_factory.mktemp("multi")
    ds = _synthetic_tree(str(root), np.random.default_rng(9))
    model = bop_run.build_model(DEV, str(root / "log"), seed=7)
    ckpt = str(root / "seeded.ckpt")
    torch.save({"state_dict": model.state_dict()}, ckpt)
    del model
    torch.cuda.empty_cache()
    return root, ds, ckpt


def _bop_run(ds, ckpt, out, ranks, extra=()):
    args = ["-m", "gigapose_b200.bop_run", "--dataset-dir", ds, "--checkpoint", ckpt, "--out", out, "--evaluate",
            "--device", DEV, *extra]
    if ranks > 1:
        args = ["-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(ranks)] + args
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, *args], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    scores = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    return scores


def _files(out):
    return {d: sorted(f for f in os.listdir(os.path.join(out, d)) if f.endswith(".npz"))
            for d in ("predictions", "refined_predictions") if os.path.isdir(os.path.join(out, d))}


@pytest.mark.parametrize("refine", [0, 2])
def test_two_ranks_write_the_one_process_csvs(tree_and_checkpoint, refine):
    root, ds, ckpt = tree_and_checkpoint
    extra = ["--refine-depth", str(refine)] if refine else []
    one, two = str(root / f"one_{refine}"), str(root / f"two_{refine}")
    want_scores = _bop_run(ds, ckpt, one, 1, extra)
    got_scores = _bop_run(ds, ckpt, two, 2, extra)
    assert len(want_scores) == (2 if refine else 1)
    assert got_scores == want_scores
    assert _files(two) == _files(one)
    assert _files(one)["predictions"] == ["0.npz", "1.npz", "2.npz"]
    csvs = [os.path.join("predictions", f"{STEM}.csv"), os.path.join("predictions", f"{STEM}MultiHypothesis.csv")]
    if refine:
        csvs.append(os.path.join("refined_predictions", f"{STEM}_icp.csv"))
    for csv in csvs:
        want = _rows(os.path.join(one, csv))
        assert len(want) > 1
        got = _rows(os.path.join(two, csv))
        assert got == want, (csv, [(g, w) for g, w in zip(got, want) if g != w][:2])
    print("bop_run_multi", refine, json.dumps(got_scores))
