"""numpy restatement of gp_depth_score (gigapose_b200/csrc/depth_score.cu, whose header comment is the contract): float32
subtractions, integer counts, one float32 division, first maximum.  tests/test_gpu_depth_score.py compares the kernel
with it bit for bit."""
import numpy as np


def depth_score(frame_idx, depth, rendered, boxes, tolerance, n_hyp):
    """frame_idx [n_det]; depth f32 [F,H,W]; rendered f32 [n_det*n_hyp,H,W]; boxes i64 [n_det*n_hyp,4] xyxy, exclusive
    max -> counts i32 [n_det*n_hyp,4] (consistent, behind, front, missing), score f32 [n_det*n_hyp], best i32 [n_det]."""
    depth = np.asarray(depth, np.float32)
    rendered = np.asarray(rendered, np.float32)
    boxes = np.asarray(boxes, np.int64)
    tol = np.float32(tolerance)
    F, H, W = depth.shape
    n_det = len(frame_idx)
    counts = np.zeros((n_det * n_hyp, 4), np.int32)
    score = np.zeros(n_det * n_hyp, np.float32)
    best = np.zeros(n_det, np.int32)
    for d in range(n_det):
        f = int(frame_idx[d])
        rows = slice(d * n_hyp, (d + 1) * n_hyp)
        if not 0 <= f < F:
            counts[rows], score[rows], best[d] = -1, np.array(0x7fffffff, np.uint32).view(np.float32), -1
            continue
        best_score = np.float32(-1.0)
        for j in range(n_hyp):
            i = d * n_hyp + j
            x0, x1 = (int(min(max(v, 0), W)) for v in boxes[i, [0, 2]])
            y0, y1 = (int(min(max(v, 0), H)) for v in boxes[i, [1, 3]])
            if x1 > x0 and y1 > y0:
                r = rendered[i, y0:y1, x0:x1]
                m = depth[f, y0:y1, x0:x1]
                on = r > 0
                with np.errstate(invalid="ignore"):
                    missing = on & ~(m > 0)
                    behind = on & ~missing & ((m - r) > tol)
                    front = on & ~missing & ~behind & ((r - m) > tol)
                consistent = on & ~missing & ~behind & ~front
                counts[i] = [consistent.sum(), behind.sum(), front.sum(), missing.sum()]
            den = int(counts[i, 0]) + int(counts[i, 1]) + int(counts[i, 2])
            score[i] = np.float32(0) if den == 0 else np.float32(int(counts[i, 0])) / np.float32(den)
            if score[i] > best_score:
                best_score, best[d] = score[i], j
    return counts, score, best
