"""CPU restatement of the BOP 2024 6D-detection score (gigapose_b200/csrc/bop_eval.cu, header comment, row f8): greedy
matching with ignored ground truths and COCO's interpolated average precision (Lin et al., "Microsoft COCO: Common
Objects in Context", ECCV 2014; pycocotools' evaluateImg / accumulate with iscrowd = 0).  Written from that statement in
plain loops, with the same stated operation order (the AP sum is sequential over the recall thresholds, in fp64), so
that gp_bop_match and gp_bop_average_precision are meant to be bit-identical to it.  The per-pair errors come from
oracle/bop_port.mssd_mspd_fp32.  Test infrastructure, like oracle/port.py; it does not import gigapose_b200."""
from __future__ import annotations

import numpy as np

LABEL_FP, LABEL_TP, LABEL_IGNORED = 0, 1, 2


def detection_labels(err, valid, thresholds):
    """One (image, object) group.  err [n_est, n_gt] with the estimates in descending score order, valid [n_gt] bool,
    thresholds [T] (fp64) -> labels int8 [n_est, T].  Per threshold, each estimate in turn takes the unmatched valid
    ground truth with the smallest error strictly below the threshold (the first on a tie) and is a TP; else the
    unmatched ignored one with the smallest such error, and is ignored; else it is an FP.  NaN never matches."""
    valid = [bool(v) for v in np.asarray(valid).reshape(-1)]
    err = np.asarray(err, np.float64)
    err = err if err.ndim == 2 else err.reshape(-1, len(valid))
    out = np.zeros((err.shape[0], len(thresholds)), np.int8)
    for t, th in enumerate(thresholds):
        taken = [False] * len(valid)
        for a in range(err.shape[0]):
            label = LABEL_FP
            for want, lab in ((True, LABEL_TP), (False, LABEL_IGNORED)):
                best = None
                for j in range(len(valid)):
                    if taken[j] or valid[j] != want or not err[a, j] < th:
                        continue
                    if best is None or err[a, j] < err[a, best]:
                        best = j
                if best is not None:
                    taken[best] = True
                    label = lab
                    break
            out[a, t] = label
    return out


def average_precision(labels, n_valid, recall_thresholds=None):
    """COCO AP of one (object, metric, threshold): labels of the object's estimates ranked by descending score over all
    images.  Cumulative TP / FP (ignored estimates keep their rank and add to neither), recall = TP / n_valid,
    precision = TP / ((TP + FP) + spacing(1)), the precision envelope from the right, q_k = the envelope at the first
    rank with recall >= r_k (0 if none), AP = sequential fp64 sum of q_k / K."""
    rec = np.linspace(0.0, 1.0, 101) if recall_thresholds is None else np.asarray(recall_thresholds, np.float64)
    lab = np.asarray(labels).reshape(-1)
    tp = np.cumsum(lab == LABEL_TP).astype(np.float64)
    fp = np.cumsum(lab == LABEL_FP).astype(np.float64)
    rc = tp / float(n_valid)
    pr = (tp / ((tp + fp) + np.spacing(1))).tolist()
    for i in range(len(pr) - 1, 0, -1):
        if pr[i] > pr[i - 1]:
            pr[i - 1] = pr[i]
    s = 0.0
    for i in np.searchsorted(rc, rec, side="left"):
        s += pr[i] if i < len(pr) else 0.0
    return s / len(rec)


def detection_scores(estimates, gts, errors, theta_mssd, theta_mspd, diameters, r, recall_thresholds=None):
    """The whole score from the pairs' errors.  estimates: kept estimates in csv order, dicts (image, obj, score);
    gts: dicts (image, obj, valid); errors {(estimate index, gt index): (mssd, mspd)} for every pair of the same image
    and object; diameters {obj: diameter}; r = image width / 640.  Evaluated objects: those with a valid gt; estimates of
    other objects take no part.  -> dict(objects, ap [n_obj, 2, T], ap_mssd, ap_mspd [n_obj, T], map_mssd, map_mspd,
    map, labels int8 [n_est, 2, T] (-1 for estimates that take no part))."""
    objects = sorted({g["obj"] for g in gts if g["valid"]})
    T = len(theta_mssd)
    labels = np.full((len(estimates), 2, T), -1, np.int8)
    groups = {}
    for i, e in enumerate(estimates):
        if e["obj"] in objects:
            groups.setdefault((e["image"], e["obj"]), ([], []))[0].append(i)
    for j, g in enumerate(gts):
        if (g["image"], g["obj"]) in groups:
            groups[(g["image"], g["obj"])][1].append(j)
    for (_, o), (ei, gi) in groups.items():
        ei = sorted(ei, key=lambda i: -estimates[i]["score"])             # stable: csv order on ties
        valid = np.array([gts[j]["valid"] for j in gi], bool)
        for m, th in enumerate((np.asarray(theta_mssd) * diameters[o], np.asarray(theta_mspd) * r)):
            err = np.array([[np.float64(errors[(a, b)][m]) for b in gi] for a in ei], np.float64).reshape(len(ei), len(gi))
            labels[ei, m] = detection_labels(err, valid, th)
    ap = np.zeros((len(objects), 2, T))
    for k, o in enumerate(objects):
        ranked = sorted((i for i, e in enumerate(estimates) if e["obj"] == o), key=lambda i: -estimates[i]["score"])
        nv = sum(1 for g in gts if g["obj"] == o and g["valid"])
        for m in range(2):
            for t in range(T):
                ap[k, m, t] = average_precision(labels[ranked, m, t], nv, recall_thresholds)
    ap_mssd, ap_mspd = np.ascontiguousarray(ap[:, 0]), np.ascontiguousarray(ap[:, 1])
    a = (float(np.mean(ap_mssd)), float(np.mean(ap_mspd))) if objects else (0.0, 0.0)
    return dict(objects=objects, ap=ap, ap_mssd=ap_mssd, ap_mspd=ap_mspd, map_mssd=a[0], map_mspd=a[1],
                map=(a[0] + a[1]) / 2.0, labels=labels)
