"""Row f10 without a GPU: the numpy port of gp_depth_score against a per-pixel loop written from the contract's
sentences, the entry point's argument checks, and the host checks of `bop_run` for a depth-refined run."""
import json
import os

import numpy as np
import pytest

from bop_tree import tetra, write_tree
from gigapose_b200 import _lib, bop_run, build
from oracle.depth_score_port import depth_score


def _brute(frame_idx, depth, rendered, boxes, tol, n_hyp):
    F, H, W = depth.shape
    n = len(rendered)
    counts, score, best = np.zeros((n, 4), np.int32), np.zeros(n, np.float32), np.zeros(len(frame_idx), np.int32)
    for i in range(n):
        d = i // n_hyp
        x0, y0, x1, y1 = (int(v) for v in boxes[i])
        for y in range(max(y0, 0), min(y1, H)):
            for x in range(max(x0, 0), min(x1, W)):
                r, m = rendered[i, y, x], depth[frame_idx[d], y, x]
                if not r > 0:
                    continue
                if not m > 0:
                    counts[i, 3] += 1
                elif np.float32(m - r) > tol:
                    counts[i, 1] += 1
                elif np.float32(r - m) > tol:
                    counts[i, 2] += 1
                else:
                    counts[i, 0] += 1
        den = int(counts[i, :3].sum())
        score[i] = np.float32(counts[i, 0]) / np.float32(den) if den else 0.0
    for d in range(len(frame_idx)):
        s = score[d * n_hyp:(d + 1) * n_hyp]
        best[d] = [j for j in range(n_hyp) if s[j] == s.max()][0]
    return counts, score, best


@pytest.mark.parametrize("n_hyp,seed", [(1, 0), (3, 1), (5, 2)])
def test_port_matches_a_per_pixel_loop(n_hyp, seed):
    rng = np.random.default_rng(seed)
    F, H, W, n_det = 2, 19, 23, 4
    n = n_det * n_hyp
    depth = rng.uniform(400, 440, (F, H, W)).astype(np.float32)
    depth[rng.random(depth.shape) < 0.1] = 0
    depth[0, 3, 4], depth[1, 5, 6] = np.nan, -3.0
    rendered = (depth[rng.integers(0, F, n)] + rng.choice([-20, -15, 0, 15, 20], (n, H, W))).astype(np.float32)
    rendered[rng.random(rendered.shape) < 0.4] = 0
    boxes = np.stack([rng.integers(-3, W // 2, n), rng.integers(-3, H // 2, n), rng.integers(W // 2, W + 4, n),
                      rng.integers(H // 2, H + 4, n)], 1).astype(np.int64)
    boxes[0] = [5, 5, 5, 9]                                  # empty
    if n > 2:
        boxes[2] = [7, 8, 8, 9]                              # one pixel
        rendered[n - 1] = rendered[n - 2]                    # a tie inside the last detection: the lower index wins
        boxes[n - 1] = boxes[n - 2]
    frame_idx = rng.integers(0, F, n_det)
    got = depth_score(frame_idx, depth, rendered, boxes, 15.0, n_hyp)
    want = _brute(frame_idx, depth, rendered, boxes, np.float32(15.0), n_hyp)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g.view(np.int32), w.view(np.int32))
    assert (got[0] > 0).any(0).all()                         # every class occurs
    if n_hyp > 1:
        assert got[2][-1] != n_hyp - 1


def test_port_marks_a_frame_index_out_of_range():
    depth = np.ones((1, 4, 4), np.float32)
    counts, score, best = depth_score([1, 0], depth, np.ones((2, 4, 4), np.float32), [[0, 0, 4, 4]] * 2, 1.0, 1)
    assert (counts[0] == -1).all() and np.isnan(score[0]) and best[0] == -1
    assert counts[1].tolist() == [16, 0, 0, 0] and score[1] == 1 and best[1] == 0


def test_gp_depth_score_rejects_bad_arguments_without_a_gpu():
    build.build()
    lib = _lib.load()
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first
    good = dict(n_frames=1, n_det=2, n_hyp=3, height=480, width=640, frame_idx=fake, depth=fake, rendered=fake,
                boxes=fake, tolerance=15.0, counts=fake, score=fake, best=fake)
    cases = [(dict(n_hyp=0), b"n_hyp 0"), (dict(n_det=0), b"n_det 0"), (dict(n_det=-2), b"n_det -2"),
             (dict(n_frames=0), b"n_frames 0"), (dict(height=0), b"image size"), (dict(width=-640), b"image size"),
             (dict(width=8193), b"image size"), (dict(tolerance=-1.0), b"tolerance"),
             (dict(tolerance=float("nan")), b"tolerance"), (dict(tolerance=float("inf")), b"tolerance")]
    cases += [({k: None}, b"null") for k in ("frame_idx", "depth", "rendered", "boxes", "counts", "score", "best")]
    before = lib.gp_launch_count()
    for kw, word in cases:
        rc = lib.gp_depth_score(*dict(good, **kw).values(), None)
        assert rc == -1 and word in lib.gp_last_error(), (kw, rc, lib.gp_last_error())
    assert lib.gp_launch_count() == before


def _tree(root, with_depth):
    ds = os.path.join(root, "ycbv")
    K = np.array([[600.0, 0, 320.0], [0, 600.0, 240.0], [0, 0, 1]])
    image = dict(gt=[(1, np.eye(3), [0, 0, 700.0])], visib=[1.0], K=K, depth_scale=0.5, png=np.zeros((4, 4), np.uint16))
    write_tree(ds, {1: tetra()}, {1: dict(diameter=70.0)}, {1: {0: image, 3: image}}, [(1, 0, 1, 1), (1, 3, 1, 1)])
    if not with_depth:
        os.remove(os.path.join(ds, "test", "000001", "depth", "000003.png"))
    dets = [dict(scene_id=1, image_id=im, category_id=1, score=0.5, time=0.1, bbox=[0, 0, 2, 2],
                 segmentation=dict(size=[4, 4], counts=[0, 4, 12])) for im in (0, 3)]
    path = os.path.join(root, "dets.json")
    with open(path, "w") as f:
        json.dump(dets, f)
    return ds, path


def test_plan_names_a_missing_depth_file(tmp_path):
    ds, dets = _tree(str(tmp_path / "a"), with_depth=True)
    p = bop_run.plan(ds, detections=dets, depth=True)
    assert p["depth_scale"] == {1: {0: 0.5, 3: 0.5}}
    ds, dets = _tree(str(tmp_path / "b"), with_depth=False)
    assert bop_run.plan(ds, detections=dets)["images"] == [(1, 0), (1, 3)]        # an RGB run does not need it
    with pytest.raises(bop_run.BopRunError, match=r"depth[/\\]000003\.png not found"):
        bop_run.plan(ds, detections=dets, depth=True)


def test_refine_depth_flag_is_checked_by_the_parser(capsys):
    base = ["--dataset-dir", "d", "--checkpoint", "c", "--template-poses", "p"]
    assert bop_run.parser().parse_args(base).refine_depth == 0
    assert bop_run.parser().parse_args(base + ["--refine-depth", "0"]).refine_depth == 0
    assert bop_run.parser().parse_args(base + ["--refine-depth", str(bop_run.TOP_K)]).refine_depth == bop_run.TOP_K
    for bad in ("-1", str(bop_run.TOP_K + 1), "two"):
        with pytest.raises(SystemExit):
            bop_run.parser().parse_args(base + ["--refine-depth", bad])
        assert "--refine-depth" in capsys.readouterr().err
