"""An independent fp64 evaluator of the BOP metrics, the scenes it is compared on, and the bars of the comparison.  Shared
by tests/test_bop_fp64_cpu.py (against oracle/bop_port.py and oracle/bop24_port.py) and tests/test_gpu_bop_fp64.py
(against csrc/bop_eval.cu and bop_eval.evaluate / evaluate_detection).

It is written from the published definitions, not from the kernels: VSD from Hodan et al., "On Evaluation of 6D Object
Pose Estimation" / "BOP: Benchmark for 6D Object Pose Estimation" (ECCV 2016 / 2018), MSSD and MSPD from Hodan et al.,
"BOP Challenge 2020 on 6D Object Localization", the BOP 2019 / 2024 evaluation rules and COCO's average precision
(Lin et al., ECCV 2014).  It imports nothing from oracle/ or gigapose_b200, reads no files, and takes the scenes in the
in-memory form tests/bop_tree.write_tree writes (so the dataset readers are crossed too).  It does not render: depth
renders come from a callable, so that what is under test is the metric.

  VSD    over every pixel where either render is non-zero (no other pixel can be visible), in float64 from the caller's
         float32 depths: the distance of depth z at pixel (u, v) is |K^-1 (u, v, 1) z| with (u, v) the integer column and
         row (the renderer's pixel centre) and K's focal lengths and principal point;
         visib_gt = d_gt > 0 and (d_gt - d_test <= delta or d_test = 0), visib_est likewise or (visib_gt and d_est > 0),
         cost = pixels of the intersection with |d_gt - d_est| / diameter >= tau, e = (cost + union - inter) / union,
         1 when the union is empty.
  MSSD   min over the symmetry transforms S of max over the vertices x of |P_est x - P_gt S x|; MSPD the same over the
  MSPD   projections with the full K (K @ p, divided by its third row).  The transforms: the identity and the declared
         discrete symmetries D; each continuous symmetry (axis a, offset o) gives n = ceil(pi / 0.01) rotations R_k by
         2 pi k / n about the line through o along a, x -> R_k x + (o - R_k o), composed as C_k D (D first).
  AR     per target (image, object): the inst_count highest-scoring estimates (stable on ties), the ground truths of the
         object, valid when visib_fract >= 0.1; per threshold, estimates in descending score order each take the
         unmatched valid ground truth with the smallest error strictly below it; recall = matched / valid targets;
         MSPD thresholds are theta x (image width / 640).
  AP     per target image the 100 highest-scoring estimates (stable on ties) of which those of objects with a valid
         ground truth count; per (image, object) the same greedy matching, with ignored ground truths (visib < 0.1)
         matchable after the valid ones and their estimates ignored; per object and threshold COCO's AP over its estimates
         ranked by score over all images: precision envelope by a reverse cumulative maximum, then the envelope at the
         first rank reaching each of the 101 recall points (searchsorted), mean over the points.

Bars.  The kernels compute in float32; every comparison here allows exactly their rounding, counted per operation with
u = 2^-24 (as in tests/render_fp64.py):
  distance  X = ((u - cx) z) / fx: 3 roundings; X^2, Y^2: 7u; their sum 8u, plus z^2 and one more sum: 9u relative of
            the radicand; the square root halves it and adds u: 5.5u relative, under DIST_ULPS ulp(d).  Where X = Y = 0
            exactly (the principal point at an integer pixel) the float32 distance is |z| exactly: bar 0.
  VSD       a pixel is ambiguous when its delta or tau comparison lies within the float32 error of its operands (the
            distances' bars, the rounding of their difference, of the division by the diameter, and float32(tau) - tau).
            Kernel counts may differ from these only on ambiguous pixels, and e by 3 n_amb / (union - n_amb).
  MSSD/MSPD float32 rounding of the inputs and transforms: POSE_BAR_MSSD u (|t| + radius) and POSE_BAR_MSPD u (the sum of
            |K| entries).
  Recall/AP must be exact where no pair's error lies within its bar of a threshold (the scenes assert it); AP is a mean
            of 101 terms, so it allows the rounding of a sequential sum, 101 x 2^-53.

Mutations.  Every definition above has flags that change one rule (MUTATIONS); the tests show that each mutated
definition fails against the kernels, with a recorded margin."""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

U = 2.0 ** -24
DELTA = 15.0
TAUS = tuple(i / 20 for i in range(1, 11))
THETA_VSD = THETA_MSSD = TAUS
THETA_MSPD = tuple(5.0 * i for i in range(1, 11))
VISIB_MIN = 0.1
SYM_STEP = 0.01
MAX_PER_IMAGE = 100
RECALL_POINTS = np.linspace(0.0, 1.0, 101)
DIST_ULPS = 6.0                 # 5.5u relative, counted above; the measured float32 error is printed by the CPU test
POSE_BAR_MSSD = 8.0             # about 4x the largest error measured (DESIGN.md, row f7)
POSE_BAR_MSPD = 2.5

VSD_MUTATIONS = ("pixel_centre_half", "depth_not_distance", "strict_delta", "missing_not_visible",
                 "no_gt_visible_term", "no_diameter", "empty_union_zero")
POSE_MUTATIONS = ("sym_dc", "offset_sign", "ignore_k01")
AR_MUTATIONS = ("theta_le", "keep_all", "count_invisible", "first_come", "mspd_unscaled")
AP_MUTATIONS = ("no_interpolation", "ignored_as_fp", "cap_after_filter", "mspd_unscaled")
FP, TP, IGNORED = 0, 1, 2


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------- VSD
def distances(z, us, vs, K, mutation=None):
    """Distances from the camera centre of float32 depths z at columns us, rows vs -> (d, bar) float64."""
    z = np.asarray(z, np.float32).astype(np.float64)
    K = np.asarray(K, np.float32).astype(np.float64).reshape(3, 3)
    h = 0.5 if mutation == "pixel_centre_half" else 0.0
    x = (us + h - K[0, 2]) / K[0, 0]
    y = (vs + h - K[1, 2]) / K[1, 1]
    d = z if mutation == "depth_not_distance" else z * np.sqrt(x * x + y * y + 1.0)
    exact = (z == 0) | ((us == K[0, 2]) & (vs == K[1, 2]))
    return d, np.where(exact, 0.0, DIST_ULPS * ulp32(d))


def _sub_bar(a, b, bar_a, bar_b):
    """Error bound of float32(a32 - b32) against a - b: the operands' bars plus the rounding of the difference (exact,
    and then 0 when it is representable, where both operands are exact float32 values)."""
    diff = a - b
    exact = (bar_a == 0) & (bar_b == 0)
    return bar_a + bar_b + np.where(exact, np.abs(diff.astype(np.float32).astype(np.float64) - diff), ulp32(diff))


def vsd(depth_test, K, est_depth, gt_depth, diameter, delta=DELTA, taus=TAUS, mutation=None):
    """One (estimate, ground truth) pair on one image -> dict(counts int64 [2 + n_tau] (inter, union, cost per tau),
    errors float64 [n_tau], n_amb (ambiguous pixels), bar [n_tau] (the bound of e), exact (e is a float32 value))."""
    H, W = np.shape(depth_test)
    idx = np.flatnonzero((np.asarray(est_depth).reshape(-1) > 0) | (np.asarray(gt_depth).reshape(-1) > 0))
    vs, us = (idx // W).astype(np.float64), (idx % W).astype(np.float64)
    dt, bt = distances(np.asarray(depth_test).reshape(-1)[idx], us, vs, K, mutation)
    dg, bg = distances(np.asarray(gt_depth).reshape(-1)[idx], us, vs, K, mutation)
    de, be = distances(np.asarray(est_depth).reshape(-1)[idx], us, vs, K, mutation)
    missing = dt == 0 if mutation != "missing_not_visible" else np.zeros(len(idx), bool)

    def visible(d, b):
        diff = d - dt
        ok = diff < delta if mutation == "strict_delta" else diff <= delta
        bar = _sub_bar(d, dt, b, bt)
        amb = (d > 0) & (dt > 0) & (bar > 0) & (np.abs(diff - delta) <= bar)
        return (d > 0) & (ok | missing), amb

    vg, amb_g = visible(dg, bg)
    ve, amb_e = visible(de, be)
    if mutation != "no_gt_visible_term":
        ve = ve | (vg & (de > 0))
    inter, union = vg & ve, vg | ve
    diam = 1.0 if mutation == "no_diameter" else float(diameter)
    c = np.abs(dg - de) / diam
    c_bar = _sub_bar(dg, de, bg, be) / diam + ulp32(c)
    amb = amb_g | amb_e
    maybe = inter | amb                    # only these pixels' tau comparisons can change a count
    costs = []
    for t in taus:
        costs.append(int(np.count_nonzero(inter & (c >= t))))
        amb |= maybe & (np.abs(c - t) <= c_bar + abs(float(np.float32(t)) - t))
    ni, nu, na = int(inter.sum()), int(union.sum()), int(amb.sum())
    if nu == 0:
        errors = np.full(len(taus), 0.0 if mutation == "empty_union_zero" else 1.0)
        return dict(counts=np.array([ni, nu] + costs, np.int64), errors=errors, n_amb=na,
                    bar=np.zeros(len(taus)) if na == 0 else np.ones(len(taus)), exact=na == 0)
    frac = [Fraction(ct + nu - ni, nu) for ct in costs]
    errors = np.array([float(f) for f in frac])
    exact = na == 0 and all(Fraction(float(np.float32(float(f)))) == f for f in frac)
    if na:
        bar = np.full(len(taus), 3.0 * na / max(nu - na, 1) + 2 * ulp32(1.0))
    else:                                  # counts exact: one float32 rounding of the rational, 0 when representable
        bar = np.array([0.0 if Fraction(float(np.float32(float(f)))) == f else float(ulp32(float(f))) for f in frac])
    return dict(counts=np.array([ni, nu] + costs, np.int64), errors=errors, n_amb=na, bar=bar, exact=exact)


# ---------------------------------------------------------------------------------------------------------- MSSD / MSPD
def _rotation(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    c, s = math.cos(angle), math.sin(angle)
    return c * np.eye(3) + s * np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]) + (1 - c) * np.outer(a, a)


def symmetries(info, mutation=None):
    """models_info entry (json form) -> transforms [S, 4, 4] float64."""
    disc = [np.eye(4)] + [np.asarray(s, np.float64).reshape(4, 4) for s in info.get("symmetries_discrete", [])]
    cont = []
    for sym in info.get("symmetries_continuous", []):
        o = np.asarray(sym["offset"], np.float64).reshape(3)
        n = int(math.ceil(math.pi / SYM_STEP))
        for k in range(n):
            T = np.eye(4)
            T[:3, :3] = _rotation(sym["axis"], 2.0 * math.pi * k / n)
            T[:3, 3] = T[:3, :3] @ o - o if mutation == "offset_sign" else o - T[:3, :3] @ o
            cont.append(T)
    if not cont:
        return np.stack(disc)
    if mutation == "sym_dc":
        return np.stack([D @ C for D in disc for C in cont])
    return np.stack([C @ D for D in disc for C in cont])


def project(K, P, mutation=None):
    K = np.array(K, np.float64).reshape(3, 3)
    if mutation == "ignore_k01":
        K[0, 1] = 0.0
    q = P @ K.T
    return q[:, :2] / q[:, 2:]


def mssd_mspd(vertices, syms, pose_est, pose_gt, K, mutation=None):
    """-> (mssd, mspd) float64 over the transforms syms [S, 4, 4]."""
    V = np.asarray(vertices, np.float64)
    Pe, Pg = np.asarray(pose_est, np.float64).reshape(4, 4), np.asarray(pose_gt, np.float64).reshape(4, 4)
    e = V @ Pe[:3, :3].T + Pe[:3, 3]
    pe = project(K, e, mutation)
    mssd = mspd = math.inf
    for S in np.asarray(syms, np.float64).reshape(-1, 4, 4):
        A = Pg @ S
        g = V @ A[:3, :3].T + A[:3, 3]
        mssd = min(mssd, float(np.sqrt(((e - g) ** 2).sum(1)).max()))
        mspd = min(mspd, float(np.sqrt(((pe - project(K, g, mutation)) ** 2).sum(1)).max()))
    return mssd, mspd


def pose_bars(vertices, pose_est, pose_gt, K):
    """Float32 error bounds of (mssd, mspd): relative to the translation plus the object's radius, and to K."""
    r = float(np.sqrt((np.asarray(vertices, np.float64) ** 2).sum(1)).max())
    t = max(np.linalg.norm(np.asarray(pose_est)[:3, 3]), np.linalg.norm(np.asarray(pose_gt)[:3, 3]))
    k = float(np.abs(np.asarray(K, np.float64)).sum())
    return POSE_BAR_MSSD * U * (t + r), POSE_BAR_MSPD * U * k


# ---------------------------------------------------------------------------------------------------------- scoring
def pose(R, t):
    T = np.eye(4)
    T[:3, :3] = np.asarray(R, np.float64).reshape(3, 3)
    T[:3, 3] = np.asarray(t, np.float64).reshape(3)
    return T


def _order(results, ids):
    """ids by descending score, the csv (list) order on ties."""
    ids = list(ids)
    keys = np.array([results[i]["score"] for i in ids], np.float64)
    return [ids[j] for j in np.lexsort((np.arange(len(ids)), -keys))]


def greedy(errors, valid, th, mutation=None, ignored=False):
    """errors [n_est, n_gt] in estimate order, valid [n_gt] -> per estimate the matched ground truth or -1, and whether it
    was a valid one.  With `ignored` (the detection task) the other ground truths are tried after the valid ones."""
    n_est, n_gt = np.shape(errors)
    taken = np.zeros(n_gt, bool)
    out = []
    for a in range(n_est):
        got = (-1, False)
        for want in ((True, False) if ignored else (True,)):
            ok = (np.asarray(valid) == want) & ~taken
            ok &= (np.asarray(errors[a]) <= th) if mutation == "theta_le" else (np.asarray(errors[a]) < th)
            if ok.any():
                j = int(np.flatnonzero(ok)[0]) if mutation == "first_come" else \
                    int(np.flatnonzero(ok)[np.argmin(np.asarray(errors[a])[ok])])
                taken[j] = True
                got = (j, want)
                break
        out.append(got)
    return out


def _margin(err, bar, thresholds):
    """Smallest |err - theta| / bar over the thresholds; inf for a bar of 0 (an exact value, decided alike even on a
    threshold)."""
    d = np.min(np.abs(np.asarray(thresholds, np.float64) - err))
    return math.inf if bar == 0 else d / bar


def evaluate_bop19(tree, results, render, delta=DELTA, taus=TAUS, mutation=None):
    """BOP 2019 average recall.  tree: dict(models {obj: (V, F)}, info {obj: models_info entry}, scenes {scene: {im:
    dict(gt [(obj, R, t)], visib, K, depth_scale, png)}}, targets [(scene, im, obj, inst_count)]); results: dicts
    (scene_id, im_id, obj_id, score, R, t); render(obj, pose [4,4], K, H, W) -> float32 depth.  -> dict(ar, ar_vsd,
    ar_mssd, ar_mspd, recall_vsd [n_tau, n_theta], recall_mssd, recall_mspd, n_targets, pairs (per pair: target, est,
    gt, the three errors and their bars), margin (the smallest distance of an error to a threshold, in bars))."""
    ths_vsd, ths_mssd = np.asarray(THETA_VSD), np.asarray(THETA_MSSD)
    m_vsd, m_mssd, m_mspd = np.zeros((len(taus), len(ths_vsd))), np.zeros(len(ths_mssd)), np.zeros(len(THETA_MSPD))
    n_targets, pairs, margin = 0, [], math.inf
    renders = {}
    for ti, (s, im, o, inst_count) in enumerate(tree["targets"]):
        sc = tree["scenes"][s][im]
        png = np.asarray(sc["png"])
        H, W = png.shape
        r = 1.0 if mutation == "mspd_unscaled" else W / 640.0
        depth = (png.astype(np.float64) * sc["depth_scale"]).astype(np.float32)
        ests = [i for i, x in enumerate(results) if (x["scene_id"], x["im_id"], x["obj_id"]) == (s, im, o)]
        ests = _order(results, ests)
        if mutation != "keep_all":
            ests = ests[:inst_count]
        gts = [k for k, g in enumerate(sc["gt"]) if g[0] == o]
        valid = np.array([mutation == "count_invisible" or sc["visib"][k] >= VISIB_MIN for k in gts], bool)
        n_targets += int(valid.sum())
        if not ests or not gts:
            continue
        V, F = tree["models"][o]
        info = tree["info"][o]
        syms = symmetries(info)
        K = np.asarray(sc["K"], np.float64)
        E = dict(vsd=np.zeros((len(ests), len(gts), len(taus))), mssd=np.zeros((len(ests), len(gts))),
                 mspd=np.zeros((len(ests), len(gts))))
        for a, e in enumerate(ests):
            Pe = pose(results[e]["R"], results[e]["t"])
            for b, k in enumerate(gts):
                Pg = pose(sc["gt"][k][1], sc["gt"][k][2])
                for key, P in (("e", Pe), ("g", Pg)):
                    rk = (o, P.tobytes(), K.tobytes(), H, W)
                    if rk not in renders:
                        renders[rk] = render(o, P, K, H, W)
                v = vsd(depth, K, renders[(o, Pe.tobytes(), K.tobytes(), H, W)],
                        renders[(o, Pg.tobytes(), K.tobytes(), H, W)], info["diameter"], delta, taus, mutation)
                ms, mp = mssd_mspd(V, syms, Pe, Pg, K)
                bs, bp = pose_bars(V, Pe, Pg, K)
                E["vsd"][a, b], E["mssd"][a, b], E["mspd"][a, b] = v["errors"], ms, mp
                pairs.append(dict(target=ti, est=e, gt=k, vsd=v["errors"], vsd_bar=v["bar"], n_amb=v["n_amb"],
                                  counts=v["counts"], mssd=ms, mssd_bar=bs, mspd=mp, mspd_bar=bp))
                margin = min([margin, _margin(ms, bs, ths_mssd * info["diameter"]),
                              _margin(mp, bp, np.asarray(THETA_MSPD) * r)] +
                             [_margin(v["errors"][t], v["bar"][t], ths_vsd) for t in range(len(taus))])
        for t in range(len(taus)):
            for j, th in enumerate(ths_vsd):
                m_vsd[t, j] += sum(1 for g, _ in greedy(E["vsd"][:, :, t], valid, th, mutation) if g >= 0)
        for j, th in enumerate(ths_mssd):
            m_mssd[j] += sum(1 for g, _ in greedy(E["mssd"], valid, th * info["diameter"], mutation) if g >= 0)
        for j, th in enumerate(THETA_MSPD):
            m_mspd[j] += sum(1 for g, _ in greedy(E["mspd"], valid, th * r, mutation) if g >= 0)
    n = max(n_targets, 1)
    rv, rs, rp = m_vsd / n, m_mssd / n, m_mspd / n
    a = (float(rv.mean()), float(rs.mean()), float(rp.mean()))
    return dict(ar=sum(a) / 3.0, ar_vsd=a[0], ar_mssd=a[1], ar_mspd=a[2], recall_vsd=rv, recall_mssd=rs,
                recall_mspd=rp, n_targets=n_targets, pairs=pairs, margin=margin)


def average_precision(labels, n_valid, mutation=None):
    """COCO AP of one ranked label sequence (FP / TP / IGNORED): the precision envelope by a reverse cumulative maximum,
    searchsorted on the recall points."""
    lab = np.asarray(labels, np.int64).reshape(-1)
    if mutation == "ignored_as_fp":
        lab = np.where(lab == IGNORED, FP, lab)
    tp, fp = np.cumsum(lab == TP).astype(np.float64), np.cumsum(lab == FP).astype(np.float64)
    if not len(lab):
        return 0.0
    recall = tp / n_valid
    precision = tp / (tp + fp + np.spacing(1.0))
    if mutation != "no_interpolation":
        precision = np.maximum.accumulate(precision[::-1])[::-1]
    at = np.searchsorted(recall, RECALL_POINTS, side="left")
    q = np.where(at < len(lab), precision[np.minimum(at, len(lab) - 1)], 0.0)
    return math.fsum(q) / len(q)


def evaluate_bop24(tree, results, max_per_image=MAX_PER_IMAGE, mutation=None):
    """BOP 2024 6D-detection mAP.  tree as evaluate_bop19's with `images` [(scene, im)] in place of targets.  -> dict(map,
    map_mssd, map_mspd, ap_mssd / ap_mspd [n_obj, T], objects, labels {result index: int8 [2, T]}, margin)."""
    scenes, T = tree["scenes"], len(THETA_MSSD)
    n_valid = {}
    for s, im in tree["images"]:
        for g, v in zip(scenes[s][im]["gt"], scenes[s][im]["visib"]):
            if v >= VISIB_MIN:
                n_valid[g[0]] = n_valid.get(g[0], 0) + 1
    objects = sorted(n_valid)
    labels, margin = {}, math.inf
    for s, im in tree["images"]:
        sc = scenes[s][im]
        W = np.asarray(sc["png"]).shape[1]
        r = 1.0 if mutation == "mspd_unscaled" else W / 640.0
        K = np.asarray(sc["K"], np.float64)
        ests = _order(results, [i for i, x in enumerate(results) if (x["scene_id"], x["im_id"]) == (s, im)])
        if mutation == "cap_after_filter":
            ests = [i for i in ests if results[i]["obj_id"] in n_valid][:max_per_image]
        else:
            ests = [i for i in ests[:max_per_image] if results[i]["obj_id"] in n_valid]
        for o in objects:
            est = [i for i in ests if results[i]["obj_id"] == o]
            gts = [k for k, g in enumerate(sc["gt"]) if g[0] == o]
            if not est:
                continue
            valid = np.array([sc["visib"][k] >= VISIB_MIN for k in gts], bool)
            V = tree["models"][o][0]
            info = tree["info"][o]
            syms = symmetries(info)
            err = np.zeros((2, len(est), len(gts)))
            for a, e in enumerate(est):
                Pe = pose(results[e]["R"], results[e]["t"])
                for b, k in enumerate(gts):
                    Pg = pose(sc["gt"][k][1], sc["gt"][k][2])
                    err[:, a, b] = mssd_mspd(V, syms, Pe, Pg, K)
                    bs, bp = pose_bars(V, Pe, Pg, K)
                    margin = min(margin, _margin(err[0, a, b], bs, np.asarray(THETA_MSSD) * info["diameter"]),
                                 _margin(err[1, a, b], bp, np.asarray(THETA_MSPD) * r))
            for e in est:
                labels[e] = np.zeros((2, T), np.int8)
            for m, ths in enumerate((np.asarray(THETA_MSSD) * info["diameter"], np.asarray(THETA_MSPD) * r)):
                for t, th in enumerate(ths):
                    for e, (j, ok) in zip(est, greedy(err[m], valid, th, ignored=True)):
                        labels[e][m, t] = FP if j < 0 else (TP if ok else IGNORED)
    ap = np.zeros((len(objects), 2, T))
    for k, o in enumerate(objects):
        ranked = _order(results, [e for e in labels if results[e]["obj_id"] == o])
        for m in range(2):
            for t in range(T):
                ap[k, m, t] = average_precision([labels[e][m, t] for e in ranked], n_valid[o], mutation)
    a = (float(ap[:, 0].mean()), float(ap[:, 1].mean()))
    return dict(map=(a[0] + a[1]) / 2.0, map_mssd=a[0], map_mspd=a[1], ap_mssd=ap[:, 0], ap_mspd=ap[:, 1],
                objects=objects, labels=labels, margin=margin)


# ---------------------------------------------------------------------------------------------------------- scenes
def rot(axis, deg):
    return _rotation(axis, math.radians(deg))


def blob(radii=(80.0, 55.0, 40.0), n_lat=40, n_lon=72):
    """A bumpy, asymmetric closed surface (mm) -> (V f32, F i32)."""
    th = np.linspace(0, np.pi, n_lat)[1:-1, None]
    ph = np.arange(n_lon)[None] * (2 * np.pi / n_lon)
    bump = 1 + 0.1 * np.sin(3 * th) * np.cos(2 * ph) + 0.06 * np.cos(5 * ph + 1.0) * np.sin(th) ** 2
    ring = np.stack([radii[0] * np.sin(th) * np.cos(ph) * bump, radii[1] * np.sin(th) * np.sin(ph) * bump,
                     radii[2] * np.cos(th) * bump + 0 * ph], -1).reshape(-1, 3)
    V = np.concatenate([ring, [[0, 0, radii[2]], [0, 0, -radii[2]]]]).astype(np.float32)
    F, L = [], n_lat - 2
    for i in range(L - 1):
        for j in range(n_lon):
            p, q = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            F += [[p, p + n_lon, q], [q, p + n_lon, q + n_lon]]
    top, bot = len(V) - 2, len(V) - 1
    for j in range(n_lon):
        F += [[top, j, (j + 1) % n_lon], [bot, (L - 1) * n_lon + (j + 1) % n_lon, (L - 1) * n_lon + j]]
    return V, np.array(F, np.int32)


def plate(x0, x1, y0, y1):
    """A flat rectangle in the z = 0 plane, facing the camera."""
    V = np.array([[x0, y0, 0], [x1, y0, 0], [x1, y1, 0], [x0, y1, 0]], np.float32)
    return V, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def diameter(V):
    V = np.asarray(V, np.float64)
    return float(max(np.sqrt(((V[i:i + 512, None] - V[None]) ** 2).sum(-1)).max() for i in range(0, len(V), 512)))


def vsd_frames(H, W, render, seed=0, n_renders=20):
    """Frames for gp_bop_vsd: three general frames, each with its own K and n_renders views of one object (its ground
    truth, perturbed estimates, views clipped on each border and partly outside, one pushed behind the measured surface,
    one empty), every ordered pair of distinct views and three identical ones; measured depth = the ground truth's minus a
    ramp across it (the delta comparison crosses inside), an occluder, 4 % missing pixels.  A fourth frame has its
    principal point on a pixel, where the measured depth is the ground truth's minus exactly delta and elsewhere 1 mm:
    the delta comparisons decided by equality, and two occluded views whose union is empty.  render(V, F, pose, K, H, W)
    -> float32 depth.  -> dict(depth [F, H, W], K [F, 3, 3], renders [R, H, W], pairs int [n, 3] (frame, est, gt),
    diameter [n], mesh)."""
    rng = np.random.default_rng(seed)
    V, F = blob()
    diam = diameter(V)
    Ks = [np.array([[0.75 * W, 0, W // 2], [0, 0.75 * W, H // 2], [0, 0, 1]]),
          np.array([[0.45 * W, 0, W / 2 + 3.37], [0, 0.46 * W, H / 2 - 2.71], [0, 0, 1]]),
          np.array([[1.1 * W, 0, 0.47 * W + 0.3], [0, 1.1 * W, 0.52 * H + 0.6], [0, 0, 1]]),
          np.array([[0.8 * W, 0, W // 2], [0, 0.8 * W, H // 2], [0, 0, 1]])]
    Ks = [K.astype(np.float32) for K in Ks]
    depth, renders, pairs = [], [], []
    for f, K in enumerate(Ks):
        fx = float(K[0, 0])
        z = fx * 2 * 80.0 / (0.16 * W)                       # the object spans about 16 % of the width
        uv = [(0.5, 0.5), (0.8, 0.4), (0.35, 0.6), (0.5, 0.5)][f]
        c = np.array([(uv[0] * W - K[0, 2]) * z / fx, (uv[1] * H - K[1, 2]) * z / K[1, 1], z])
        if f == 3:
            c[:2] = 0.0
        R0 = rot(rng.normal(size=3), rng.uniform(0, 180))
        poses = [pose(R0, c)]
        if f < 3:
            for _ in range(n_renders - 8):
                poses.append(pose(rot(rng.normal(size=3), rng.uniform(1, 12)) @ R0,
                                  c + rng.normal(size=3) * [8, 8, 20]))
            for bu, bv in ((0.0, 0.5), (1.0, 0.5), (0.5, 0.0), (0.5, 1.0)):    # centred on each border
                poses.append(pose(R0, [(bu * W - K[0, 2]) * z / fx, (bv * H - K[1, 2]) * z / K[1, 1], z]))
            poses.append(pose(R0, c + [0, 0, 60.0]))                       # behind the measured surface
            poses.append(pose(R0, c * [1, 1, -1]))                         # behind the camera: empty
        else:
            poses += [pose(R0, c + [0, 0, 1.0]), pose(R0, c + [0, 0, 30.0]), pose(R0, c + [0, 0, 40.0])]
        base = len(renders)
        rs = [np.asarray(render(V, F, P, K, H, W), np.float32) for P in poses]
        renders += rs
        g = rs[0]
        if f < 3:
            us = np.arange(W)[None]
            cols = np.nonzero(g.any(0))[0]
            ramp = -25.0 + 50.0 * (us - cols.min()) / max(cols.max() - cols.min(), 1)
            d = np.full((H, W), np.float32(z + 250.0))
            d = np.where(g > 0, g - ramp, d).astype(np.float32)
            ys, xs = np.nonzero(g)
            d[ys.min():(ys.min() + ys.max()) // 2, xs.min():(xs.min() + xs.max()) // 2] = np.float32(z - 150.0)
            d[rng.random((H, W)) < 0.04] = 0
            n = len(rs)
            pairs += [(f, base + i, base + j) for i in range(n) for j in range(n) if i != j]
            pairs += [(f, base + i, base + i) for i in range(3)] + [(f, base + n - 1, base + n - 1)]
        else:
            d = np.full((H, W), np.float32(1.0))
            cy, cx = int(K[1, 2]), int(K[0, 2])
            assert g[cy, cx] > 0
            d[cy, cx] = g[cy, cx] - np.float32(DELTA)
            assert float(g[cy, cx]) - float(d[cy, cx]) == DELTA
            pairs += [(f, base + 1, base), (f, base, base + 1), (f, base, base), (f, base + 2, base + 3)]
        depth.append(d.astype(np.float32))
    pairs = np.array(pairs, np.int64)
    return dict(depth=np.stack(depth), K=np.stack(Ks), renders=np.stack(renders), pairs=pairs,
                diameter=np.full(len(pairs), diam), mesh=(V, F))


def compare_vsd(kernel_counts, kernel_errors, ref):
    """One pair: kernel counts / errors against a `vsd` result -> (count excess over n_amb, error ratio to the bar)."""
    excess = int(np.abs(np.asarray(kernel_counts, np.int64) - ref["counts"]).max()) - ref["n_amb"]
    d = np.abs(np.asarray(kernel_errors, np.float64) - ref["errors"])
    ratio = float(np.max(np.where(ref["bar"] > 0, d / np.where(ref["bar"] > 0, ref["bar"], 1), np.where(d > 0, np.inf, 0))))
    return excess, ratio


def pose_objects():
    """Objects for gp_bop_mssd_mspd, models_info entries in json form -> [(V, info)]:
    0: 10 002 vertices, a discrete symmetry (90 deg about x through o, so that C D and D C differ) and a continuous one
       about z through o = (20, -12, 0): 2 x 315 = 630 transforms, the last chunk of 8 partial;
    1: no symmetry (1 transform); 2: 8 discrete symmetries about z (9 transforms)."""
    import bop_tree
    o = np.array([20.0, -12.0, 0.0])
    V0 = (bop_tree.spheroid(60.0, 35.0, n_lat=102, n_lon=100)[0] + o).astype(np.float32)
    D = np.eye(4)
    D[:3, :3] = rot([1, 0, 0], 90)
    D[:3, 3] = o - D[:3, :3] @ o
    info0 = dict(diameter=diameter(V0[::7]), symmetries_discrete=[D.ravel().tolist()],
                 symmetries_continuous=[dict(axis=[0, 0, 1], offset=o.tolist())])
    V1 = blob(n_lat=20, n_lon=36)[0]
    V2 = bop_tree.spheroid(40.0, 25.0, n_lat=12, n_lon=48)[0]
    steps = []
    for k in range(1, 9):
        S = np.eye(4)
        S[:3, :3] = rot([0, 0, 1], 45.0 * k)
        steps.append(S.ravel().tolist())
    return [(V0, info0), (V1, dict(diameter=diameter(V1))), (V2, dict(diameter=80.0, symmetries_discrete=steps))]


POSE_KS = [np.array([[1390.5, 20.0, 964.9], [0, 1387.0, 522.2], [0, 0, 1]], np.float32),      # skewed
           np.array([[572.4, 0, 325.3], [0, 573.6, 242.0], [0, 0, 1]], np.float32)]


def pose_cases(objects, seed=1):
    """(object, frame, pose_est, pose_gt) float64: estimates on a symmetry (one of C_k D, one of C_k), perturbed ones and
    identical ones, both frames."""
    rng = np.random.default_rng(seed)
    cases = []
    for o, (V, info) in enumerate(objects):
        S = symmetries(info)
        for f in range(2):
            for k in range(4):
                Pg = pose(rot(rng.normal(size=3), rng.uniform(0, 180)), rng.normal(size=3) * [80, 60, 0] + [0, 0, 700 + 150 * k])
                if k == 0:
                    Pe = Pg.copy()
                elif k == 1:                                         # C_k D (the last one when there is no C)
                    Pe = Pg @ S[len(S) // 2 + 37 if len(S) > 315 else len(S) - 1]
                elif k == 2 and len(S) > 315:
                    Pe = Pg @ S[37]                                  # C_37 alone (D = identity)
                else:
                    Pe = pose(rot(rng.normal(size=3), rng.uniform(1, 10)) @ Pg[:3, :3], Pg[:3, 3] + rng.normal(size=3) * 5)
                cases.append((o, f, Pe, Pg))
    return cases


def _res(s, im, o, score, P):
    return dict(scene_id=s, im_id=im, obj_id=o, score=float(score), R=np.asarray(P)[:3, :3].copy(),
                t=np.asarray(P)[:3, 3].reshape(3, 1).copy(), time=0.25)


def ar_tree(render, seed=2):
    """A BOP 2019 tree at 400 x 240 (r = 0.625): two images with their own K; an asymmetric blob (two close instances,
    one under the visibility cut), a plate whose estimate, shifted by 10 px over missing depth, has a VSD of exactly
    1/4 = theta, a spheroid with a discrete flip and a continuous symmetry about an axis off its origin; repeated
    instances, score ties, an estimate of an object without a target, 101 extra estimates in one image.  -> (tree,
    results); tree as evaluate_bop19 takes it (the arguments of bop_tree.write_tree)."""
    import bop_tree
    rng = np.random.default_rng(seed)
    H, W = 240, 400
    Ks = [np.array([[300.0, 0, 200.0], [0, 300.0, 120.0], [0, 0, 1]]),
          np.array([[310.0, 0, 197.3], [0, 305.0, 118.6], [0, 0, 1]])]
    o3 = np.array([6.0, -4.0, 0.0])
    flip = np.eye(4)
    flip[:3, :3] = rot([1, 0, 0], 180)
    flip[:3, 3] = o3 - flip[:3, :3] @ o3
    Vb, Fb = blob((50.0, 35.0, 25.0), 24, 48)
    Vs, Fs = bop_tree.spheroid(40.0, 25.0, n_lat=14, n_lon=48)
    models = {1: (Vb, Fb), 2: plate(-71.0, 69.0, -51.0, 49.0), 3: ((Vs + o3).astype(np.float32), Fs)}
    info = {1: dict(diameter=100.0), 2: dict(diameter=172.0),
            3: dict(diameter=80.0, symmetries_discrete=[flip.ravel().tolist()],
                    symmetries_continuous=[dict(axis=[0, 0, 1], offset=o3.tolist())])}
    Ra, Rb, Rc = rot([1, 2, 0], 40), rot([0, 1, 1], 70), rot([1, 0, 0], 30)
    gts = {0: [(1, Ra, [-60.0, -40, 700]), (1, Ra, [-30.0, -40, 700]), (1, Rb, [80.0, 50, 800]), (2, np.eye(3), [0.0, 0, 600]),
               (3, Rc, [90.0, -50, 650])],
           1: [(1, Rb, [-50.0, 20, 650]), (3, Rc, [40.0, -40, 700]), (3, Rb, [-60.0, 50, 750]), (1, Ra, [70.0, 40, 800])]}
    visib = {0: [0.8, 0.7, 0.05, 0.9, 0.6], 1: [0.9, 0.5, 0.7, 0.08]}
    scenes = {1: {}}
    for im in (0, 1):
        K = Ks[im]
        d = np.full((H, W), 1500.0)
        for o, R, t in gts[im]:
            r = np.asarray(render(*models[o], pose(R, t), K, H, W), np.float64)
            d = np.where((r > 0) & (r < d), r, d)
        d[rng.random((H, W)) < 0.03] = 0
        if im == 0:
            d[90:150, 150:250] = 0                              # no depth under the plate and its estimate
        scenes[1][im] = dict(gt=[(o, R, np.asarray(t)) for o, R, t in gts[im]], visib=visib[im], K=K, depth_scale=0.1,
                             png=np.round(d / 0.1).astype(np.uint16))
    targets = [(1, 0, 1, 2), (1, 0, 2, 1), (1, 0, 3, 1), (1, 1, 1, 1), (1, 1, 3, 2)]
    G = lambda im, k: pose(gts[im][k][1], gts[im][k][2])
    turn = lambda P, S: P @ S
    S3 = symmetries(info[3])
    res = [_res(1, 0, 1, 0.9, pose(Ra, [-43.0, -40, 700])),          # 17 / 13 mm from the two instances
           _res(1, 0, 1, 0.8, pose(Ra, [-56.0, -40, 700])),          # 4 / 26 mm: greedy by error matches both
           _res(1, 0, 1, 0.75, pose(rot([0, 0, 1], 50) @ Rb, [80.0, 50, 800])),   # on the invisible instance
           _res(1, 0, 2, 0.7, pose(np.eye(3), [20.0, 0, 600])),      # the plate 10 px to the right
           _res(1, 0, 3, 0.6, turn(G(0, 4), S3[315 + 40]) @ pose(rot([0, 1, 0], 2), [1.0, 0, 2])),
           _res(1, 0, 3, 0.6, pose(rot([1, 1, 0], 6) @ Rc, [93.0, -47, 660])),   # a tie: csv order keeps the first
           _res(1, 1, 1, 0.95, pose(rot([1, 0, 0], 25) @ Rb, [-20.0, 20, 690])),  # kept (inst_count 1), poor
           _res(1, 1, 1, 0.5, pose(rot([0, 1, 0], 3) @ Rb, [-48.0, 21, 652])),    # dropped, good
           _res(1, 1, 3, 0.7, turn(G(1, 1), S3[100]) @ pose(np.eye(3), [0.5, 0.5, 3])),
           _res(1, 1, 3, 0.7, pose(rot([0, 0, 1], 4) @ Rb, [-57.0, 52, 748])),
           _res(1, 1, 3, 0.4, pose(rot([1, 0, 0], 9) @ Rc, [44.0, -36, 712])),
           _res(1, 1, 2, 0.99, pose(np.eye(3), [0.0, 0, 600]))]              # object 2 has no target in image 1
    for k in range(101):                                                       # low-scored extras in image 0
        P = pose(rot(rng.normal(size=3), rng.uniform(0, 90)) @ Ra, [-45.0, -40, 700] + rng.normal(size=3) * [30, 20, 40])
        res.append(_res(1, 0, 1, 0.1 * rng.random(), P))
    return dict(models=models, info=info, scenes=scenes, targets=targets), res


def ap_tree(seed=4):
    """A BOP 2024 tree at 400 x 240 (r = 0.625), no depth needed: two images; objects 1 (three instances per image, one
    ignored), 3 (symmetric, offset axis), 2 (only an ignored ground truth: not evaluated) and 4 (no ground truth).
    Image 0 has 103 estimates: 8 of objects 2 and 4 at the top scores, then object 1's, whose lowest-scored one is a
    true positive that a cap applied after dropping the non-evaluated objects would keep; an estimate on an ignored
    ground truth ranks above a false positive; score ties.  -> (tree, results)."""
    rng = np.random.default_rng(seed)
    import bop_tree
    o3 = np.array([6.0, -4.0, 0.0])
    Vs, Fs = bop_tree.spheroid(40.0, 25.0, n_lat=14, n_lon=48)
    Vb, Fb = blob((50.0, 35.0, 25.0), 24, 48)
    models = {1: (Vb, Fb), 2: bop_tree.tetra(60.0), 3: ((Vs + o3).astype(np.float32), Fs), 4: bop_tree.tetra(30.0)}
    flip = np.eye(4)
    flip[:3, :3] = rot([1, 0, 0], 180)
    flip[:3, 3] = o3 - flip[:3, :3] @ o3
    info = {1: dict(diameter=100.0), 2: dict(diameter=85.0), 4: dict(diameter=42.0),
            3: dict(diameter=80.0, symmetries_discrete=[flip.ravel().tolist()],
                    symmetries_continuous=[dict(axis=[0, 0, 1], offset=o3.tolist())])}
    K = np.array([[300.0, 0, 200.0], [0, 300.0, 120.0], [0, 0, 1]])
    R = [rot(rng.normal(size=3), rng.uniform(0, 180)) for _ in range(8)]
    gts = {0: [(1, R[0], [-80.0, -40, 700]), (1, R[1], [0.0, -40, 750]), (1, R[2], [80.0, 40, 800]), (3, R[3], [-60.0, 60, 700]),
               (2, R[4], [60.0, 60, 650])],
           1: [(1, R[5], [-50.0, 20, 650]), (3, R[6], [40.0, -40, 700]), (3, R[7], [-60.0, 50, 750])]}
    visib = {0: [0.8, 0.7, 0.05, 0.9, 0.05], 1: [0.9, 0.5, 0.7]}
    scenes = {1: {im: dict(gt=[(o, Rr, np.asarray(t)) for o, Rr, t in gts[im]], visib=visib[im], K=K, depth_scale=1.0,
                           png=np.zeros((240, 400), np.uint16)) for im in (0, 1)}}
    G = lambda im, k: pose(gts[im][k][1], gts[im][k][2])
    near = lambda P, deg, dt: pose(rot(rng.normal(size=3), deg) @ P[:3, :3], P[:3, 3] + dt)
    S3 = symmetries(info[3])
    res = []
    for k in range(8):                                                          # non-evaluated objects on top
        res.append(_res(1, 0, 2 if k % 2 else 4, 0.99, G(0, 4)))
    res += [_res(1, 0, 1, 0.9, near(G(0, 2), 1, [1, 0, 2])),                   # on the ignored instance
            _res(1, 0, 1, 0.8, near(G(0, 0), 2, [2, 1, 3])),
            _res(1, 0, 1, 0.8, near(G(0, 0), 1, [0, 1, 1])),                   # a tie; the second is a duplicate
            _res(1, 0, 3, 0.75, G(0, 3) @ S3[315 + 60] @ pose(rot([0, 1, 0], 1), [1.0, 0, 1]))]
    for k in range(90):                                                         # far-off false positives
        res.append(_res(1, 0, 1, 0.7 - 0.005 * k, near(G(0, 1), 30, rng.normal(size=3) * 40 + [0, 0, 60])))
    res.append(_res(1, 0, 1, 0.05, near(G(0, 1), 2, [1, 2, 2])))                # 103rd of 103: a TP
    res += [_res(1, 1, 1, 0.6, near(G(1, 0), 3, [3, 2, 8])),
            _res(1, 1, 1, 0.95, near(G(1, 0), 20, [20, 10, 40])),
            _res(1, 1, 3, 0.85, G(1, 1) @ S3[200] @ pose(np.eye(3), [0.5, 0.5, 2])),
            _res(1, 1, 3, 0.85, near(G(1, 2), 4, [4, -2, 9])),
            _res(1, 1, 3, 0.3, near(G(1, 2), 15, [10, 5, 30])),
            _res(1, 1, 4, 0.9, G(1, 0))]
    return dict(models=models, info=info, scenes=scenes, images=[(1, 0), (1, 1)],
                targets=[(1, im, 1, 1) for im in (0, 1)]), res
