"""CPU restatement of the depth refiner's masked-normal mode (gigapose_b200/csrc/depth_icp.cu, steps 1' and 2', row
f11), on top of oracle/icp_port.py: the target normals of detection d come from the depth smoothed within its mask M_d,
S_d = (G * (D [D > 0] M_d)) / (G * ([D > 0] M_d)), the points from the raw depth, the targets are z > 0 and M_d, and
stages 3-6 are icp_port.refine's with that map and mask.

`scene_masked` is the definition over the whole frame; `scene_masked_box` is what the kernels compute: S_d on the
mask's box grown by MARGIN px and clipped to the frame, the map on the box, reading D and M_d only inside the box."""
from __future__ import annotations

import numpy as np

from oracle import icp_port

F32 = np.float32
MARGIN = 2


def scene_masked(depth, mask, K, unit_per_m=1000.0):
    """Target map f32 [H,W,6] of one detection: points of icp_port.scene(D), normals of icp_port.scene(D M).  The
    normals of icp_port.scene depend on S and K only and its smoothing weights are [D > 0], so feeding it the masked
    depth smooths with the weights [D > 0] M."""
    D = np.asarray(depth, F32)
    masked = np.where(np.asarray(mask) != 0, D, F32(0))
    points = icp_port.scene(D, K, unit_per_m)
    normals = icp_port.scene(masked, K, unit_per_m)
    return np.concatenate([points[..., :3], normals[..., 3:]], -1)


def mask_box(mask):
    """(x0, y0, x1, y1), exclusive max, of the nonzero pixels; (0, 0, 0, 0) for an empty mask."""
    ys, xs = np.nonzero(np.asarray(mask))
    if not len(ys):
        return 0, 0, 0, 0
    return int(xs.min()), int(ys.min()), int(xs.max()) + 1, int(ys.max()) + 1


def _grad_at(S, idx, n, lo):
    """np.gradient(., 2, edge_order=2) along axis 0 of the tile S (whose row 0 is frame index lo) at frame indices
    idx, in the kernel's float32 operation order."""
    x = lambda i: S[i - lo]                                                     # noqa: E731
    out = np.empty((len(idx),) + S.shape[1:], F32)
    for k, i in enumerate(idx):
        if i == 0:
            out[k] = (F32(-0.75) * x(0) + x(1)) + F32(-0.25) * x(2)
        elif i == n - 1:
            out[k] = (F32(0.25) * x(n - 3) + (-x(n - 2))) + F32(0.75) * x(n - 1)
        else:
            out[k] = (x(i + 1) - x(i - 1)) / F32(4)
    return out


def scene_masked_box(depth, mask, K, box=None, unit_per_m=1000.0):
    """The map of `scene_masked` over the mask's box only -> (box, map f32 [y1-y0, x1-x0, 6]); reads depth and mask
    inside the box only (anything outside may be garbage)."""
    D = np.asarray(depth, F32)
    H, W = D.shape
    x0, y0, x1, y1 = mask_box(mask) if box is None else box
    if x1 <= x0 or y1 <= y0:
        return (x0, y0, x1, y1), np.zeros((max(y1 - y0, 0), max(x1 - x0, 0), 6), F32)
    ex0, ey0, ex1, ey1 = max(0, x0 - MARGIN), max(0, y0 - MARGIN), min(W, x1 + MARGIN), min(H, y1 + MARGIN)
    inbox = np.zeros((H, W), bool)
    inbox[y0:y1, x0:x1] = True
    Db = np.where(inbox, D, F32(0))                  # nothing outside the box is read below
    valid = inbox & (np.asarray(mask) != 0) & (Db > 0)
    w = icp_port.gauss_weights()
    rows, cols = np.arange(ey0, ey1), np.arange(ex0, ex1)
    num = np.zeros((len(rows), len(cols)), F32)
    den = np.zeros_like(num)
    for k in range(-icp_port.RADIUS, icp_port.RADIUS + 1):
        r = icp_port._reflect(rows + k, H)
        ok = valid[r][:, ex0:ex1]
        num = np.where(ok, num + w[k + icp_port.RADIUS] * Db[r][:, ex0:ex1], num).astype(F32)
        den = np.where(ok, den + w[k + icp_port.RADIUS], den).astype(F32)
    sn, sd = np.zeros_like(num), np.zeros_like(num)
    for k in range(-icp_port.RADIUS, icp_port.RADIUS + 1):
        j = icp_port._reflect(cols + k, W)
        inside = (j >= ex0) & (j < ex1)                                # columns outside ext hold num = den = 0
        jj = np.clip(j - ex0, 0, len(cols) - 1)
        sn = np.where(inside, sn + w[k + icp_port.RADIUS] * num[:, jj], sn).astype(F32)
        sd = np.where(inside, sd + w[k + icp_port.RADIUS] * den[:, jj], sd).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        S = np.where(sd > 0, sn / sd, F32(0)).astype(F32)             # [ext rows, ext cols]
    bv, bu = np.arange(y0, y1), np.arange(x0, x1)
    gv = _grad_at(S[:, bu - ex0], bv, H, ey0)
    gu = _grad_at(S[bv - ey0].T, bu, W, ex0).T
    z = S[np.ix_(bv - ey0, bu - ex0)]
    K = np.asarray(K, F32)
    fx, cx, fy, cy = K[0, 0], K[0, 2], K[1, 1], K[1, 2]
    a = (bu.astype(F32) - cx)[None, :]
    b = (bv.astype(F32) - cy)[:, None]
    ix, iy = F32(1) / fx, F32(1) / fy
    tux, tuy, tuz = z * ix + (a * ix) * gu, (b * iy) * gu, gu
    tvx, tvy, tvz = (a * ix) * gv, z * iy + (b * iy) * gv, gv
    nx, ny, nz = tuy * tvz - tuz * tvy, tuz * tvx - tux * tvz, tux * tvy - tuy * tvx
    nn = np.sqrt((nx * nx + ny * ny) + nz * nz)
    with np.errstate(divide="ignore", invalid="ignore"):
        n = np.where(nn[..., None] > 0, np.stack([nx, ny, nz], -1) / nn[..., None], F32(0)).astype(F32)
    d = Db[y0:y1, x0:x1]
    ok = (d > F32(0.2) * F32(unit_per_m)) & (d < F32(5) * F32(unit_per_m))
    pts = np.stack([np.where(ok, (a * d) / fx, F32(0)), np.where(ok, (b * d) / fy, F32(0)), np.where(ok, d, F32(0))], -1)
    return (x0, y0, x1, y1), np.concatenate([pts, n], -1).astype(F32)


def refine_masked(depth, mask, rendered, box, K, T0, debug=None, **params):
    """Stages 2-6 of one hypothesis in the masked mode -> icp_port.refine's (pose, status, residual, fitness)."""
    return icp_port.refine(scene_masked(depth, mask, K, params.get("unit_per_m", 1000.0)), rendered, box, K, T0,
                           mask=mask, debug=debug, **params)
