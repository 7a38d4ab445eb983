"""TEST INFRASTRUCTURE ONLY -- regenerates tests/golden/add_reference.{json,npz} (row f12).

Drives the reference's own vendored MegaPose pieces (dists_add, dists_add_symmetric, project_points, get_top_n_ids
with targets, add_valid_gt(visib_gt_min=0.1), get_candidate_matches, match_poses, compute_auc_posecnn) on a seeded
synthetic BOP tree, and stores the tree (in the form tests/bop_tree.write_tree takes) with the reference's per-pair
errors, matches, recalls and AUCs.  The meter that combined these pieces is not in the reference: the recall here is
(matches with error < threshold) / (valid ground truths of the targets), and the AUC takes the matched error of every
valid ground truth in metres, inf when unmatched.

The tree plants the cases the tests need: an ADD of exactly 100 mm = 0.1 x the declared 1000 mm diameter and = 0.1 m
(the strict recall `<` and the AUC cap's `>`), one just above (100 + 2^-7 mm), a target where minimum-error matching
gives a ground truth an error above 0.1 d although another estimate was below it, a ground truth under the visibility
cut, an object that declares only a continuous symmetry, an object with no target within 0.1 m, a rotated estimate on
a non-uniformly sampled object (the two nearest-neighbour directions differ), K01 != 0 in one frame, and no score
ties.

    python -m oracle.make_golden_add
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.ref_import import _ReferenceImports  # noqa: E402
from bop_tree import rot, spheroid  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
METRICS = ("add(-s)", "add-s", "proj")


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3] = np.asarray(R, np.float64)
    T[:3, 3] = t
    return T


class _Stub(types.ModuleType):
    """A module whose every attribute is another stub: enough for import-time references."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Stub(f"{self.__name__}.{name}")


def fixture(seed=12):
    """-> dict(models {obj: (V, F)}, info, scenes, targets, results) for write_tree (results as load_bop_results dicts
    with list-valued R, t)."""
    rng = np.random.default_rng(seed)
    # obj 1: integer coordinates (transforms by R = I and integer translations are exact in fp32), non-uniform: a dense
    # cluster and a sparse shell
    dense = rng.integers(-20, 21, (500, 3))
    sparse = rng.integers(-150, 151, (300, 3))
    V1 = np.unique(np.concatenate([dense, sparse]), axis=0).astype(np.float32)
    V2, F2 = spheroid(40.0, 25.0, n_lat=12, n_lon=48)              # exact 7.5 degree symmetry about z
    V3 = rng.uniform(-60, 60, (300, 3)).astype(np.float32)
    tri = np.array([[0, 1, 2]], np.int32)
    models = {1: (V1, tri), 2: (V2, F2), 3: (V3, tri)}
    info = {1: dict(diameter=1000.0),                               # 0.1 d = 100 exactly in fp64
            2: dict(diameter=80.0, symmetries_continuous=[dict(axis=[0, 0, 1], offset=[0, 0, 0])]),
            3: dict(diameter=169.7)}
    I = np.eye(3)
    K1 = np.array([[600.0, 0, 320], [0, 600.0, 240], [0, 0, 1]])
    K2 = np.array([[580.0, 2.5, 330], [0, 590.0, 250], [0, 0, 1]])
    png = np.zeros((8, 8), np.uint16)
    A, B, C = np.array([300.0, 0, 2000]), np.array([-500.0, 0, 2000]), np.array([0.0, 400, 2000])
    D, E, H = np.array([-200.0, 0, 1800]), np.array([200.0, 0, 1800]), np.array([0.0, 900, 1800])
    RF, F_, G = rot([1, 2, 0.5], 40), np.array([0.0, -300, 1500]), np.array([150.0, -300, 1500])
    R3, T3 = rot([0.3, -1, 0.2], 25), np.array([-100.0, 200, 1700])
    scenes = {1: {
        1: dict(gt=[(1, I, B), (1, I, A), (1, I, C), (3, R3, T3), (3, I, [400.0, -300, 2100])], visib=[0.8, 0.9, 0.05, 0.7, 0.6],
                K=K1, depth_scale=1.0,
                png=png),
        2: dict(gt=[(1, I, D), (1, I, E), (1, I, H), (2, RF, F_), (2, I, G)], visib=[0.9, 0.6, 0.5, 0.7, 0.4], K=K2,
                depth_scale=1.0, png=png)}}
    targets = [(1, 1, 1, 2), (1, 1, 3, 2), (1, 2, 1, 3), (1, 2, 2, 2)]
    ests = [  # (im, obj, score, R, t)
        (1, 1, 0.95, I, A + [100.0, 0, 0]),               # ADD exactly 100 mm = 0.1 d = 0.1 m
        (1, 1, 0.90, I, B + [0, 100.0078125, 0]),         # just above
        (1, 1, 0.50, I, C),                               # dropped by inst_count (and C is under the visibility cut)
        (1, 3, 0.80, R3, T3 + [0, 0, 300.0]),             # obj 3: no target within 0.1 m, one target missed
        (2, 1, 0.90, I, D + [150.0, 0, 0]),               # takes D at 150 > 0.1 d ...
        (2, 1, 0.85, I, D + [-50.0, 0, 0]),               # ... though this one is at 50; it takes E at 450
        (2, 1, 0.70, rot([0, 1, 1], 20) @ I, H + [5.0, -3, 4]),    # rotated: ADD-S's direction matters
        (2, 2, 0.92, RF @ rot([0, 0, 1], 30), F_ + [1.0, 2, -1]),  # about the symmetry axis: ADD-S small, ADD not
        (2, 2, 0.60, I, G + [0, 0, 40.0]),
    ]
    results = [dict(scene_id=1, im_id=im, obj_id=o, score=s, R=np.asarray(R).tolist(), t=np.asarray(t).tolist(),
                    time=1.0) for im, o, s, R, t in ests]
    return dict(models=models, info=info, scenes=scenes, targets=targets, results=results)


def main():
    fx = fixture()
    import pandas as pd
    # transform_ops imports pinocchio (through transform.py) and transforms3d at module level; neither is called here
    stubs = {name: _Stub(name) for name in ("pinocchio", "transforms3d")}
    with _ReferenceImports(stubs) as ctx:
        dist = ctx.import_reference("src.megapose.lib3d.distances")
        geo = ctx.import_reference("src.megapose.lib3d.camera_geometry")
        mu = ctx.import_reference("src.megapose.evaluation.meters.utils")
        preds = pd.DataFrame([dict(scene_id=r["scene_id"], view_id=r["im_id"], label=r["obj_id"], score=r["score"],
                                   csv_id=i) for i, r in enumerate(fx["results"])])
        tg = pd.DataFrame([dict(scene_id=s, view_id=i, label=o, inst_count=n) for s, i, o, n in fx["targets"]])
        keep = mu.get_top_n_ids(preds, group_keys=("scene_id", "view_id", "label"), top_key="score", targets=tg)
        preds = preds.iloc[np.sort(np.asarray(keep, np.int64))].reset_index(drop=True)
        gts = []
        for s, i, o, _ in fx["targets"]:
            sc = fx["scenes"][s][i]
            for k, (go, R, t) in enumerate(sc["gt"]):
                if go == o:
                    gts.append(dict(scene_id=s, view_id=i, label=o, visib_fract=sc["visib"][k], gt_inst=k))
        gts = mu.add_valid_gt(pd.DataFrame(gts), visib_gt_min=0.1)
        n_targets = int(gts["valid"].sum())
        cand = mu.get_candidate_matches(preds, gts)
        err = {m: [] for m in ("add", "adds", "proj")}
        for _, c in cand.iterrows():
            r = fx["results"][int(c["csv_id"])]
            sc = fx["scenes"][int(c["scene_id"])][int(c["view_id"])]
            _, Rg, tg_ = sc["gt"][int(c["gt_inst"])]
            Pe = torch.as_tensor(_pose(r["R"], r["t"]), dtype=torch.float32)[None]
            Pg = torch.as_tensor(_pose(Rg, tg_), dtype=torch.float32)[None]
            pts = torch.as_tensor(fx["models"][int(c["label"])][0], dtype=torch.float32)[None]
            err["add"].append(dist.dists_add(Pe, Pg, pts).norm(dim=-1).mean().item())
            err["adds"].append(dist.dists_add_symmetric(Pe, Pg, pts).norm(dim=-1).mean().item())
            K = torch.as_tensor(sc["K"], dtype=torch.float32)[None]
            err["proj"].append((geo.project_points(pts, K, Pe) - geo.project_points(pts, K, Pg)).norm(dim=-1).mean().item())
        sym = {o: bool(v.get("symmetries_continuous") or v.get("symmetries_discrete")) for o, v in fx["info"].items()}
        per_metric = {"add(-s)": [e_s if sym[int(l)] else e_a for e_a, e_s, l in zip(err["add"], err["adds"], cand["label"])],
                      "add-s": err["adds"], "proj": err["proj"]}
        out = dict(n_targets=n_targets, cand=dict(csv_id=cand["csv_id"].astype(int).tolist(),
                                                  gt_inst=cand["gt_inst"].astype(int).tolist(),
                                                  label=cand["label"].astype(int).tolist(), **err),
                   matches={}, recall={}, auc={}, auc_objects={}, recall_objects={})
        valid = gts[gts["valid"]].reset_index(drop=True)
        for m in METRICS:
            c = cand.copy()
            c["error"] = np.asarray(per_metric[m], np.float64)
            mt = mu.match_poses(c)
            pairs = [(int(preds.loc[int(p), "csv_id"]),
                      int(gts.loc[int(g), "gt_inst"]), float(e))
                     for p, g, e in zip(mt["pred_id"], mt["gt_id"], mt["error"])]
            out["matches"][m] = sorted(pairs)
            got = {(int(gts.loc[int(g), "view_id"]), int(gts.loc[int(g), "gt_inst"])): float(e)
                   for g, e in zip(mt["gt_id"], mt["error"])}
            target_err = np.array([got.get((int(v), int(k)), np.inf) for v, k in zip(valid["view_id"], valid["gt_inst"])])
            labels = valid["label"].to_numpy().astype(int)
            thr = np.array([0.1 * fx["info"][int(l)]["diameter"] for l in labels]) if m != "proj" else np.full(len(labels), 5.0)
            out["recall"][m] = float(np.count_nonzero(target_err < thr) / n_targets)
            out["recall_objects"][m] = {str(o): float(np.count_nonzero((target_err < thr)[labels == o]) /
                                                      np.count_nonzero(labels == o)) for o in sorted(set(labels))}
            if m != "proj":
                out["auc"][m] = float(mu.compute_auc_posecnn(target_err / 1000.0))
                out["auc_objects"][m] = {str(o): float(mu.compute_auc_posecnn(target_err[labels == o] / 1000.0))
                                         for o in sorted(set(labels))}
    tree = dict(info={str(k): v for k, v in fx["info"].items()}, targets=fx["targets"], results=fx["results"],
                scenes={str(s): {str(i): dict(gt=[(o, np.asarray(R).tolist(), np.asarray(t).tolist()) for o, R, t in v["gt"]],
                                              visib=v["visib"], K=np.asarray(v["K"]).tolist())
                                 for i, v in ims.items()} for s, ims in fx["scenes"].items()})
    with open(os.path.join(OUT, "add_reference.json"), "w") as f:
        json.dump(dict(tree=tree, reference=out), f, indent=1)
    np.savez_compressed(os.path.join(OUT, "add_reference.npz"),
                        **{f"V{o}": V for o, (V, _) in fx["models"].items()},
                        **{f"F{o}": F for o, (_, F) in fx["models"].items()})
    print(json.dumps(dict(n_targets=out["n_targets"], recall=out["recall"], auc=out["auc"],
                          auc_objects=out["auc_objects"]), indent=1))


if __name__ == "__main__":
    main()
