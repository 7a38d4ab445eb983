"""An independent fp64 evaluator of row f12 (ADD, ADD-S, proj; ADD(-S) / ADD-S / proj recalls and PoseCNN's AUC),
written from the definitions: ADD = mean |P_est x - P_gt x|; ADD-S = mean over the ground-truth points of the distance
to the nearest estimated point (scipy's cKDTree in fp64, the BOP toolkit's method, cross-checked by brute force);
proj = mean pixel distance with u = (K00 x + K01 y) / z + K02, v = K11 y / z + K12; ADD(-S) = ADD-S for an object
with declared symmetries; per target the top inst_count estimates by score (csv order on ties), ground truths valid at
visib_fract >= 0.1, minimum-error matching without a threshold, recall = matched errors < threshold over the valid
ground truths, and the AUC up to 0.1 m as the upper step sum of the accuracy curve.

It imports neither oracle/add_port.py nor bop_eval's matching or AUC code.  It takes a tree in the in-memory form that
tests/bop_tree.write_tree writes (plus the model vertices and the results list), so the dataset readers are crossed.

`mutate` names a wrong definition, for the tests that check each one fails:
  nn_swap            ADD-S with the nearest ground-truth point of each estimated point
  rms                root mean square instead of the mean
  no_k01             K01 ignored in the projection
  add_for_continuous ADD(-S) takes ADD for an object that declares only continuous symmetries
  le_threshold       recall counts error <= threshold
  auc_ge_cap         the AUC drops errors >= 0.1 m (so exactly 0.1 m no longer counts)
  first_come         each estimate takes the first unmatched valid ground truth, whatever its error
  bop_matching       each estimate takes the best unmatched valid ground truth below the threshold (BOP 2019's rule)
  drop_unmatched_auc the AUC is over the matched targets only
  count_invisible    ground truths under the visibility cut are targets and matchable
"""
import numpy as np
from scipy.spatial import cKDTree

U32 = 2.0 ** -24                # unit roundoff of fp32
VISIB_MIN = 0.1
AUC_CAP = 0.1                   # metres
METRICS = ("add(-s)", "add-s", "proj")


def _apply(P, V):
    P = np.asarray(P, np.float64).reshape(4, 4)
    return np.asarray(V, np.float64) @ P[:3, :3].T + P[:3, 3]


def _proj(K, X, k01=True):
    K = np.asarray(K, np.float64).reshape(3, 3)
    u = ((K[0, 0] * X[:, 0] + (K[0, 1] * X[:, 1] if k01 else 0.0)) / X[:, 2]) + K[0, 2]
    v = K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2]
    return np.stack([u, v], 1)


def nn_brute(query, points):
    """Distance of each query row to its nearest row of points, by brute force."""
    q, p = np.asarray(query, np.float64), np.asarray(points, np.float64)
    return np.sqrt(((q[:, None, :] - p[None, :, :]) ** 2).sum(-1).min(1))


def nn_kdtree(query, points):
    return cKDTree(np.asarray(points, np.float64)).query(np.asarray(query, np.float64), k=1)[0]


def errors(V, pose_est, pose_gt, K, mutate=()):
    """-> (ADD, ADD-S, proj) in fp64."""
    e, g = _apply(pose_est, V), _apply(pose_gt, V)
    mean = (lambda d: float(np.sqrt(np.mean(d ** 2)))) if "rms" in mutate else (lambda d: float(np.mean(d)))
    add = mean(np.linalg.norm(e - g, axis=1))
    adds = mean(nn_kdtree(e, g) if "nn_swap" in mutate else nn_kdtree(g, e))
    k01 = "no_k01" not in mutate
    proj = mean(np.linalg.norm(_proj(K, e, k01) - _proj(K, g, k01), axis=1))
    return add, adds, proj


def bars(V, pose_est, pose_gt, K):
    """fp32 error bars of (ADD, ADD-S, proj) against fp64.  A transformed coordinate ((A0 x + A1 y) + A2 z) + A3 has at
    most 4 roundings, each within u of a partial sum bounded by |t| + r (r = the largest vertex norm, |R| = 1), so every
    coordinate is within 4 u (|t| + r); a difference of two within 8 u (|t_est| + |t_gt| + 2 r) plus its own rounding,
    and the norm (3 roundings on squares, one sqrt) keeps it within 2x that.  The min of values each within b is within b
    of the fp64 min, so ADD-S has ADD's bar.  proj: u = (K00 x + K01 y) / z + K02 with x, y, z each within the
    coordinate bar c and z >= z_min: |du| <= ((|K00| + |K01|) (1 + m) + |K11| (1 + m)) c / z_min + 8 u max(|u|, |v|),
    m = max (|x| + |y|) / z."""
    V = np.asarray(V, np.float64)
    r = float(np.linalg.norm(V, axis=1).max())
    te, tg = np.linalg.norm(np.asarray(pose_est, np.float64).reshape(4, 4)[:3, 3]), \
        np.linalg.norm(np.asarray(pose_gt, np.float64).reshape(4, 4)[:3, 3])
    c = 4 * U32 * (max(te, tg) + r)
    b3 = 2 * (2 * c + 8 * U32 * (te + tg + 2 * r))
    K = np.asarray(K, np.float64).reshape(3, 3)
    e, g = _apply(pose_est, V), _apply(pose_gt, V)
    z = min(e[:, 2].min(), g[:, 2].min())
    m = max((np.abs(e[:, :2]).sum(1) / e[:, 2]).max(), (np.abs(g[:, :2]).sum(1) / g[:, 2]).max())
    uv = np.abs(np.concatenate([_proj(K, e), _proj(K, g)])).max()
    bp = 2 * (2 * ((abs(K[0, 0]) + abs(K[0, 1]) + abs(K[1, 1])) * (1 + m) * c / z + 8 * U32 * uv))
    return b3, b3, bp


def auc(errors_m, ge_cap=False):
    """Area under the accuracy curve up to AUC_CAP, x 1 / AUC_CAP, as the upper step sum: over the distinct kept errors
    d_1 < d_2 < ... (kept: <= AUC_CAP, or < with ge_cap), the interval (d_{k-1}, d_k] (d_0 = 0) counts the accuracy
    (first rank of d_k) / n, and (d_last, AUC_CAP] the accuracy of all kept errors.  NaN when none is kept."""
    d = np.sort(np.asarray(errors_m, np.float64))
    n = len(d)
    keep = (d < AUC_CAP) if ge_cap else (d <= AUC_CAP)
    kd = d[keep]
    if len(kd) == 0:
        return float("nan")
    area, prev = 0.0, 0.0
    for k, x in enumerate(kd):
        if x != prev:
            area += (x - prev) * ((k + 1) / n)
            prev = x
    area += (AUC_CAP - prev) * (len(kd) / n)
    return area / AUC_CAP


def _match(err, valid, mutate, thr):
    """Per ground truth: the matched error (inf when unmatched)."""
    out = np.full(len(valid), np.inf)
    for row in err:
        free = [j for j in range(len(valid)) if valid[j] and np.isinf(out[j]) and not np.isnan(row[j])
                and np.isfinite(row[j])]
        if "first_come" in mutate:
            pick = free[:1]
        elif "bop_matching" in mutate:
            below = [j for j in free if row[j] < thr]
            pick = [min(below, key=lambda j: (row[j], j))] if below else []
        else:
            pick = [min(free, key=lambda j: (row[j], j))] if free else []
        for j in pick:
            out[j] = row[j]
    return out


def evaluate(tree, models, results, mutate=()):
    """tree: dict(info {obj: models_info entry}, scenes {scene: {im: dict(gt [(obj, R, t)], visib, K)}}, targets
    [(scene, im, obj, inst_count)]); models {obj: V [N,3]}; results: dicts (scene_id, im_id, obj_id, score, R, t).
    -> dict(pairs {(csv index, scene, im, gt index): (add, adds, proj)}, matched {metric: [errors per target]},
    target_obj, n_targets, recall {metric}, auc {metric}, objects {obj: dict(recall, auc)})."""
    info = tree["info"]
    pairs, matched, tobj, thr_all = {}, {m: [] for m in ("add(-s)", "add-s", "proj")}, [], {m: [] for m in
                                                                                        ("add(-s)", "add-s", "proj")}
    for s, im, o, n in tree["targets"]:
        sc = tree["scenes"][s][im]
        idx = [i for i, r in enumerate(results) if (r["scene_id"], r["im_id"], r["obj_id"]) == (s, im, o)]
        idx = sorted(idx, key=lambda i: (-results[i]["score"], i))[:n]
        gts = [k for k, g in enumerate(sc["gt"]) if g[0] == o]
        valid = np.array([sc["visib"][k] >= VISIB_MIN or "count_invisible" in mutate for k in gts], bool)
        sym = bool(info[o].get("symmetries_discrete")) or bool(info[o].get("symmetries_continuous"))
        if "add_for_continuous" in mutate and not info[o].get("symmetries_discrete"):
            sym = False
        tabs = {m: np.full((len(idx), len(gts)), np.inf) for m in matched}
        for a, i in enumerate(idx):
            r = results[i]
            Pe = np.eye(4)
            Pe[:3, :3], Pe[:3, 3] = np.asarray(r["R"], np.float64).reshape(3, 3), np.asarray(r["t"], np.float64)
            for b, k in enumerate(gts):
                Pg = np.eye(4)
                Pg[:3, :3], Pg[:3, 3] = np.asarray(sc["gt"][k][1], np.float64).reshape(3, 3), sc["gt"][k][2]
                e = errors(models[o], Pe, Pg, sc["K"], mutate)
                pairs[(i, s, im, k)] = e
                tabs["add(-s)"][a, b] = e[1] if sym else e[0]
                tabs["add-s"][a, b] = e[1]
                tabs["proj"][a, b] = e[2]
        d = float(info[o]["diameter"])
        th = {"add(-s)": 0.1 * d, "add-s": 0.1 * d, "proj": 5.0}
        for m in matched:
            matched[m] += list(_match(tabs[m], valid, mutate, th[m])[valid])
            thr_all[m] += [th[m]] * int(valid.sum())
        tobj += [o] * int(valid.sum())
    tobj = np.array(tobj)
    matched = {m: np.array(v) for m, v in matched.items()}
    thr_all = {m: np.array(v) for m, v in thr_all.items()}

    def scores(sel):
        n = int(sel.sum())
        hit = {m: (matched[m][sel] <= thr_all[m][sel]) if "le_threshold" in mutate else (matched[m][sel] < thr_all[m][sel])
               for m in matched}
        rec = {m: float(np.count_nonzero(h) / max(n, 1)) for m, h in hit.items()}
        au = {}
        for m in ("add(-s)", "add-s"):
            e = matched[m][sel] / 1000.0
            if "drop_unmatched_auc" in mutate:
                e = e[np.isfinite(e)]
            au[m] = auc(e, "auc_ge_cap" in mutate)
        return rec, au

    rec, au = scores(np.ones(len(tobj), bool))
    objects = {int(o): dict(zip(("recall", "auc"), scores(tobj == o))) for o in sorted(set(tobj.tolist()))}
    return dict(pairs=pairs, matched=matched, target_obj=tobj, n_targets=len(tobj), recall=rec, auc=au,
                objects=objects)


# ---------------------------------------------------------------------------------------------------- the golden tree
def golden(golden_dir):
    """tests/golden/add_reference.{json,npz} -> (tree, models {obj: V}, faces {obj: F}, results, reference) with int
    keys, in the form `evaluate` and tests/bop_tree.write_tree take."""
    import json
    import os
    with open(os.path.join(golden_dir, "add_reference.json")) as f:
        d = json.load(f)
    z = np.load(os.path.join(golden_dir, "add_reference.npz"))
    t = d["tree"]
    tree = dict(info={int(k): v for k, v in t["info"].items()},
                targets=[tuple(x) for x in t["targets"]],
                scenes={int(s): {int(i): dict(gt=[(o, np.asarray(R), np.asarray(tt)) for o, R, tt in v["gt"]],
                                              visib=v["visib"], K=np.asarray(v["K"]))
                                 for i, v in ims.items()} for s, ims in t["scenes"].items()})
    models = {o: z[f"V{o}"] for o in tree["info"]}
    faces = {o: z[f"F{o}"] for o in tree["info"]}
    return tree, models, faces, t["results"], d["reference"]


def write_golden_tree(root, tree, models, faces):
    """The golden tree as a BOP dataset directory (8 x 8 empty depth images: no metric here reads them)."""
    from bop_tree import write_tree
    scenes = {s: {i: dict(v, depth_scale=1.0, png=np.zeros((8, 8), np.uint16)) for i, v in ims.items()}
              for s, ims in tree["scenes"].items()}
    write_tree(root, {o: (models[o], faces[o]) for o in models}, tree["info"], scenes, tree["targets"])


# ---------------------------------------------------------------------------------------------------- comparisons
def pose(R, t):
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64)
    return P


def pair_args(fx, e, s, im, k):
    """(V, P_est, P_gt, K) of result e against ground truth k of image (s, im); fx holds results, tree, models."""
    r = fx["results"][e]
    o, R, t = fx["tree"]["scenes"][s][im]["gt"][k]
    return fx["models"][o], pose(r["R"], r["t"]), pose(R, t), fx["tree"]["scenes"][s][im]["K"]


def close_auc(a, b, bar):
    return (np.isnan(a) and np.isnan(b)) or abs(a - b) <= bar


MUTATIONS = ("nn_swap", "rms", "no_k01", "add_for_continuous", "le_threshold", "auc_ge_cap", "first_come",
             "bop_matching", "drop_unmatched_auc", "count_invisible")


def disagreement(fp64, scores, errors, fx_like):
    """How a (possibly mutated) fp64 evaluation disagrees with bop_eval's scores on the port's (or kernel's) errors
    (fx_like holds setup, results, tree, models):
    -> dict(pair = worst per-pair |diff| / bar, recall = recalls that differ, auc = AUCs beyond their bar, matched =
    targets whose matched error differs beyond the largest pair bar or whose match differs)."""
    setup = fx_like["setup"]
    worst, max_bar = 0.0, 0.0
    for p in range(len(errors["group"])):
        g = setup["groups"][int(errors["group"][p])]
        key = (int(errors["est"][p]), g["scene_id"], g["im_id"], int(errors["gt"][p]))
        V, Pe, Pg, K = pair_args(fx_like, key[0], key[1], key[2], key[3])
        bar = np.array(bars(V, Pe, Pg, K))
        max_bar = max(max_bar, float(bar.max()))
        got = np.array([errors["add"][p], errors["adds"][p], errors["proj"][p]])
        worst = max(worst, float((np.abs(got - np.array(fp64["pairs"][key])) / bar).max()))
    rec = [m for m in METRICS if fp64["recall"][m] != scores["recall"][m]]
    rec += [(m, o) for o, v in scores["objects"].items() for m in METRICS
            if o in fp64["objects"] and fp64["objects"][o]["recall"][m] != v["recall"][m]]
    n_matched = 0
    if len(fp64["matched"]["proj"]) != len(scores["matched"]["proj"]):
        n_matched = -1
    else:
        for m in METRICS:
            a, b = fp64["matched"][m], scores["matched"][m]
            both = np.isfinite(a) & np.isfinite(b)
            n_matched += int((np.isfinite(a) != np.isfinite(b)).sum() +
                             (np.abs(a[both] - b[both]) > max_bar).sum())
    # an AUC moves by at most 10 x 2 e when every error moves by at most e metres (see the fp64 / reference test)
    ab = 20 * max_bar / 1000
    auc = [m for m in ("add(-s)", "add-s") if not close_auc(fp64["auc"][m], scores["auc"][m], ab)]
    auc += [(m, o) for o, v in scores["objects"].items() for m in ("add(-s)", "add-s")
            if o in fp64["objects"] and not close_auc(fp64["objects"][o]["auc"][m], v["auc"][m], ab)]
    return dict(pair=worst, recall=rec, auc=auc, matched=n_matched)


def failed(d):
    return d["pair"] > 1 or d["recall"] or d["auc"] or d["matched"] != 0
