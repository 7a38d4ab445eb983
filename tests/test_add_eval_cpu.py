"""Row f12 without a GPU: bop_eval.add_scores against the reference's matches, recalls and AUCs on the golden tree
(tests/golden/add_reference.*, from oracle/make_golden_add.py), oracle/add_port.py against the fp64 evaluator
(tests/add_fp64.py) and the reference's fp32 dists_add*, the fp64 evaluator against the reference, every mutated
definition failing against the port, and the --task add flag."""
import numpy as np
import pytest

import add_fp64 as af
from gigapose_b200 import bop_eval
from oracle import add_port

METRICS = ("add(-s)", "add-s", "proj")


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
    tree, models, faces, results, ref = af.golden(golden_dir)
    root = str(tmp_path_factory.mktemp("add_tree"))
    af.write_golden_tree(root, tree, models, faces)
    setup = bop_eval.prepare(results, root)
    return dict(tree=tree, models=models, results=results, ref=ref, root=root, setup=setup)


def reference_errors(fx):
    """The reference's per-candidate errors in the layout compute_add_errors returns."""
    c, groups = fx["ref"]["cand"], fx["setup"]["groups"]
    out = dict(group=[], est=[], gt=[], add=[], adds=[], proj=[])
    for i, e in enumerate(c["csv_id"]):
        r = fx["results"][e]
        gi = next(g for g, G in enumerate(groups) if (G["scene_id"], G["im_id"], G["obj_id"]) ==
                  (r["scene_id"], r["im_id"], r["obj_id"]))
        out["group"].append(gi)
        out["est"].append(e)
        out["gt"].append(c["gt_inst"][i])
        for m in ("add", "adds", "proj"):
            out[m].append(c[m][i])
    return {k: np.asarray(v) for k, v in out.items()}


def port_errors(setup, tree, models, results):
    """oracle/add_port.py's errors of every pair compute_add_errors would compute."""
    rows = bop_eval._pair_rows(setup["groups"], range(len(setup["groups"])), setup["images"])
    out = dict(group=rows["group"], est=rows["est"], gt=rows["gt"])
    errs = []
    for gi, e, k in zip(rows["group"], rows["est"], rows["gt"]):
        g = setup["groups"][gi]
        V, Pe, Pg, K = af.pair_args(dict(results=results, tree=tree, models=models), e, g["scene_id"], g["im_id"], k)
        errs.append(add_port.add_errors(V, Pe.astype(np.float32), Pg.astype(np.float32), K))
    errs = np.asarray(errs).reshape(-1, 3)
    return dict(out, add=errs[:, 0], adds=errs[:, 1], proj=errs[:, 2])


def test_add_scores_on_the_reference_errors_give_the_reference_scores(fx):
    s = bop_eval.add_scores(fx["setup"], reference_errors(fx))
    ref = fx["ref"]
    assert s["n_targets"] == ref["n_targets"] == 9
    for m in METRICS:
        got = sorted((int(e), int(k), float(err))
                     for (gi, k), e, err in zip(s["target_gt"], s["matched_est"][m], s["matched"][m]) if e >= 0)
        assert got == sorted((a, b, c) for a, b, c in ref["matches"][m]), m
        assert s["recall"][m] == ref["recall"][m], m
        for o, v in s["objects"].items():
            assert v["recall"][m] == ref["recall_objects"][m][str(o)], (m, o)
    for m in ("add(-s)", "add-s"):
        assert af.close_auc(s["auc"][m], ref["auc"][m], 0.0), (m, s["auc"][m], ref["auc"][m])
        for o, v in s["objects"].items():
            assert af.close_auc(v["auc"][m], ref["auc_objects"][m][str(o)], 0.0), (m, o)
    # the planted cases
    assert np.isnan(s["objects"][3]["auc"]["add-s"]) and not np.isnan(s["objects"][1]["auc"]["add(-s)"])
    assert 100.0 in s["matched"]["add(-s)"].tolist() and 100.0078125 in s["matched"]["add(-s)"].tolist()
    assert np.isinf(s["matched"]["add(-s)"]).sum() == 1


def test_match_min_error_rule():
    v = np.array([True, True, False, True])
    err = np.array([[5.0, 5.0, 0.0, 9.0], [np.nan, 1.0, 0.0, np.inf], [np.inf, np.nan, 0.0, 7.0], [1.0, 1.0, 1.0, 1.0]])
    e, a = bop_eval.match_min_error(err, v)
    # row 0 takes gt 0 (a tie: the lowest index), row 1 gt 1 (NaN / inf never match), row 2 gt 3, row 3 nothing left
    assert a.tolist() == [0, 1, -1, 2] and e.tolist() == [5.0, 1.0, np.inf, 7.0]


def test_port_within_the_fp64_bars_and_the_reference_fp32(fx):
    c, worst = fx["ref"]["cand"], np.zeros(3)
    worst_ref = np.zeros(3)
    for i, e in enumerate(c["csv_id"]):
        r = fx["results"][e]
        V, Pe, Pg, K = af.pair_args(fx, e, r["scene_id"], r["im_id"], c["gt_inst"][i])
        got = np.array(add_port.add_errors(V, Pe.astype(np.float32), Pg.astype(np.float32), K))
        want = np.array(af.errors(V, Pe, Pg, K))
        bar = np.array(af.bars(V, Pe, Pg, K))
        worst = np.maximum(worst, np.abs(got - want) / bar)
        worst_ref = np.maximum(worst_ref, np.abs(got - np.array([c["add"][i], c["adds"][i], c["proj"][i]])) / (2 * bar))
    print("port / fp64 bar (add, adds, proj):", worst.tolist(), "port vs reference fp32 / 2 bars:", worst_ref.tolist())
    assert (worst <= 1).all() and (worst_ref <= 1).all()


def test_kdtree_equals_brute_force():
    rng = np.random.default_rng(3)
    a, b = rng.normal(size=(300, 3)) * 50, rng.normal(size=(257, 3)) * 50
    assert np.array_equal(af.nn_kdtree(a, b), af.nn_brute(a, b))


def test_port_terms_exact_cases():
    V = np.array([[0, 0, 0], [10, 0, 0], [0, 20, 0]], np.float32)
    P = af.pose(np.eye(3), [1, 2, 500]).astype(np.float32)
    K = np.array([[500, 3, 320], [0, 500, 240], [0, 0, 1]], np.float32)
    assert add_port.add_errors(V, P, P, K) == (0.0, 0.0, 0.0)
    Q = P.copy()
    Q[0, 3] += 7
    add, adds, proj = add_port.add_errors(V, Q, P, K)
    assert add == 7.0 and adds == 17.0 / 3.0                 # (10, 0, 0)'s nearest estimated point is (7, 0, 0)
    assert add_port.chunked_mean(np.arange(2500, dtype=np.float32)) == 1249.5


def test_fp64_evaluator_equals_the_reference(fx):
    got = af.evaluate(fx["tree"], fx["models"], fx["results"])
    ref = fx["ref"]
    assert got["n_targets"] == ref["n_targets"]
    for m in METRICS:
        assert got["recall"][m] == ref["recall"][m], m
    # AUC is 10 x a sum of (interval x accuracy) with accuracies <= 1: moving each error by at most e moves it by
    # at most 10 x 2 e (metres); e = the largest fp32 / fp64 difference of the matched errors
    e = max(abs(a - b) for m in ("add(-s)", "add-s") for a, b in
            zip(sorted(x for x in got["matched"][m] if np.isfinite(x)), sorted(x[2] for x in ref["matches"][m])))
    for m in ("add(-s)", "add-s"):
        assert af.close_auc(got["auc"][m], ref["auc"][m], 20 * e / 1000 + 1e-15), m
        for o, v in got["objects"].items():
            assert af.close_auc(v["auc"][m], ref["auc_objects"][m][str(o)], 20 * e / 1000 + 1e-15), (m, o)


def test_port_scores_agree_with_fp64_and_every_mutation_fails(fx):
    errors = port_errors(fx["setup"], fx["tree"], fx["models"], fx["results"])
    scores = bop_eval.add_scores(fx["setup"], errors)
    base = af.disagreement(af.evaluate(fx["tree"], fx["models"], fx["results"]), scores, errors, fx)
    assert not af.failed(base), base
    for mut in af.MUTATIONS:
        d = af.disagreement(af.evaluate(fx["tree"], fx["models"], fx["results"], (mut,)), scores, errors, fx)
        print("mutation", mut, d)
        assert af.failed(d), mut


def test_task_add_parses_and_localization_stays_the_default(monkeypatch, tmp_path):
    seen = []
    monkeypatch.setattr(bop_eval, "evaluate_add", lambda *a, **k: seen.append(("add", a, k)) or dict(scores={}))
    monkeypatch.setattr(bop_eval, "evaluate", lambda *a, **k: seen.append(("loc", a, k)) or
                        {k: 0 for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd", "n_targets", "average_time_per_image")})
    csv = str(tmp_path / "x.csv")
    bop_eval.main(["--results", csv, "--dataset-dir", "D", "--task", "add", "--out", "O"])
    bop_eval.main(["--results", csv, "--dataset-dir", "D"])
    assert [s[0] for s in seen] == ["add", "loc"]
    assert seen[0][1] == (csv, "D", "test") and seen[0][2] == dict(out_dir="O")
    assert seen[1][2] == dict(out_dir=str(tmp_path))
