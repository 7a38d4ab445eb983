"""Row f12 on the GPU against the independent fp64 evaluator (tests/add_fp64.py): gp_bop_add's errors within their
derived bars on objects of 1 to 100 000 vertices, every mutated definition failing against the kernel on the golden
tree, and evaluate_add end to end on a larger synthetic tree (symmetric objects, repeated instances, score ties,
invisible ground truths).  Worst ratios to the bars and the mutation margins are printed (pytest -s) for DESIGN.md."""
import json

import numpy as np
import pytest

import add_fp64 as af
from bop_tree import rot, spheroid, write_tree
from gigapose_b200 import bop_eval
from test_gpu_add_eval import case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _report(name, obj):
    print(name, json.dumps(obj))


def test_kernel_within_the_fp64_bars():
    c = case()
    worst = np.zeros(3)
    for p in range(c["bad"]):
        o, f = c["obj"][p], c["frame"][p]
        V = c["vertices"][c["vo"][o]:c["vo"][o + 1]]
        pe, pg = c["pe"][p].astype(np.float64), c["pg"][p].astype(np.float64)     # the poses the kernel was given
        want = np.array(af.errors(V, pe, pg, c["K"][f].astype(np.float64)))
        bar = np.array(af.bars(V, pe, pg, c["K"][f].astype(np.float64)))
        worst = np.maximum(worst, np.abs(c["kernel"][p] - want) / bar)
    _report("f12 kernel / fp64 bar (add, adds, proj)", worst.tolist())
    assert (worst <= 1).all()


@pytest.fixture(scope="module")
def golden_fx(golden_dir, tmp_path_factory):
    tree, models, faces, results, ref = af.golden(golden_dir)
    root = str(tmp_path_factory.mktemp("add_tree"))
    af.write_golden_tree(root, tree, models, faces)
    fx = dict(tree=tree, models=models, results=results, root=root, setup=bop_eval.prepare(results, root))
    fx["res"] = bop_eval.evaluate_add(results, root, device=DEV)
    return fx


def test_every_mutation_fails_against_the_kernel(golden_fx):
    fx, res = golden_fx, golden_fx["res"]
    base = af.disagreement(af.evaluate(fx["tree"], fx["models"], fx["results"]), res, res["errors"], fx)
    assert not af.failed(base), base
    margins = {"none": base}
    for mut in af.MUTATIONS:
        d = af.disagreement(af.evaluate(fx["tree"], fx["models"], fx["results"], (mut,)), res, res["errors"], fx)
        margins[mut] = d
        assert af.failed(d), mut
    _report("f12 mutation margins", {k: dict(pair=v["pair"], recall=len(v["recall"]), auc=len(v["auc"]),
                                             matched=v["matched"]) for k, v in margins.items()})


def larger_tree(seed=5):
    """4 images, 3 objects (one plain and non-uniform, one with a continuous symmetry, one with a discrete one),
    2-3 instances of each per image, some under the visibility cut, 1-2 estimates per instance with score ties and a
    wrong-instance estimate."""
    rng = np.random.default_rng(seed)
    V1 = np.concatenate([rng.normal(size=(1200, 3)) * 8, rng.uniform(-70, 70, (600, 3))]).astype(np.float32)
    V2, F2 = spheroid(45.0, 30.0, n_lat=16, n_lon=64)
    half = rng.uniform(-50, 50, (400, 3))
    V3 = np.concatenate([half, half * [-1, -1, 1]]).astype(np.float32)         # symmetric under 180 deg about z
    tri = np.array([[0, 1, 2]], np.int32)
    models = {1: (V1, tri), 2: (V2, F2), 3: (V3, tri)}
    flip = np.diag([-1.0, -1.0, 1.0, 1.0])
    info = {1: dict(diameter=float(2 * np.linalg.norm(V1, axis=1).max())),
            2: dict(diameter=90.0, symmetries_continuous=[dict(axis=[0, 0, 1], offset=[0, 0, 0])]),
            3: dict(diameter=float(2 * np.linalg.norm(V3, axis=1).max()), symmetries_discrete=[flip.ravel().tolist()])}
    scenes, targets, results = {2: {}}, [], []
    for im in range(4):
        K = np.array([[600.0 + 20 * im, 1.5 * (im % 2), 320], [0, 605.0, 240], [0, 0, 1]])
        gt, visib = [], []
        for o in (1, 2, 3):
            n = 2 + (im + o) % 2
            for k in range(n):
                R = rot(rng.normal(size=3), rng.uniform(0, 360))
                t = np.array([rng.uniform(-250, 250), rng.uniform(-200, 200), rng.uniform(800, 1600)])
                gt.append((o, R, t))
                visib.append(0.05 if (k == 1 and im % 2 == 0) else float(rng.uniform(0.2, 1)))
                for e in range(1 + (k + im) % 2):
                    dR = rot(rng.normal(size=3), rng.uniform(0, 12 if e == 0 else 40))
                    dt = rng.normal(size=3) * (3, 10, 30)[(k + e + im) % 3]
                    score = round(float(rng.uniform(0.1, 1)), 1)          # rounded: ties happen
                    results.append(dict(scene_id=2, im_id=im, obj_id=o, score=score, R=(R @ dR).tolist(),
                                        t=(t + dt).tolist(), time=1.0))
            targets.append((2, im, o, n))
        scenes[2][im] = dict(gt=gt, visib=visib, K=K, depth_scale=1.0, png=np.zeros((8, 8), np.uint16))
    return models, info, scenes, targets, results


def test_evaluate_add_equals_the_fp64_evaluator_on_a_larger_tree(tmp_path):
    models, info, scenes, targets, results = larger_tree()
    write_tree(str(tmp_path), models, info, scenes, targets)
    scores = [r["score"] for r in results]
    assert len(set(scores)) < len(scores)                                       # score ties
    res = bop_eval.evaluate_add(results, str(tmp_path), device=DEV)
    tree = dict(info=info, scenes={2: {im: dict(gt=v["gt"], visib=v["visib"], K=v["K"]) for im, v in scenes[2].items()}},
                targets=targets)
    mv = {o: m[0] for o, m in models.items()}
    fx = dict(tree=tree, models=mv, results=results, setup=bop_eval.prepare(results, str(tmp_path)))
    ref = af.evaluate(tree, mv, results)
    # no matched error within a bar of its threshold (recalls must then agree exactly)
    for m, thr in (("add(-s)", None), ("add-s", None), ("proj", 5.0)):
        th = np.array([0.1 * info[o]["diameter"] for o in ref["target_obj"]]) if thr is None else thr
        e = ref["matched"][m]
        fin = np.isfinite(e)
        assert (np.abs(e[fin] - (th[fin] if thr is None else th)) > 1e-3).all(), m
        if thr is None:
            assert (np.abs(e[fin] - 100.0) > 1e-3).all(), m                    # the AUC cap, 0.1 m
    d = af.disagreement(ref, res, res["errors"], fx)
    _report("f12 larger tree", dict(n_pairs=len(res["errors"]["group"]), n_targets=res["n_targets"], worst_pair=d["pair"],
                                    recalls=res["recall"], aucs=res["auc"]))
    assert not af.failed(d), d
    assert res["n_targets"] == ref["n_targets"] and res["n_targets"] >= 20
