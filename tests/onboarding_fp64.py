"""Row f16's re-centring restated in fp64 numpy, independently of csrc/onboard.cu: the re-centred mask's box found by
sampling a virtual grid that covers the whole frame, and the 224 crop built from ATen's own crop of a coordinate image
(tests/crop_aten.py) followed by the per-pixel map through H^-1, nearest mask, bilinear RGB and the CLIP steps.

Pixel centres are at integer coordinates (csrc/render.cu's convention).  A virtual pixel (c, r) samples the frame at
(x, y) = (s0 / s2, s1 / s2), s = H^-1 (c, r, 1), evaluated in the kernel's operation order, and is outside the frame
when s2 <= 0 or (rint(x), rint(y)) is outside it."""
import numpy as np
import torch

from crop_aten import crop_aten

CLIP_MEAN = np.array([0.48145466, 0.4578275, 0.40821073])
CLIP_STD = np.array([0.26862954, 0.26130258, 0.27577711])


def to_source(hinv, c, r):
    h = np.asarray(hinv, np.float64).reshape(9)
    c, r = np.asarray(c, np.float64), np.asarray(r, np.float64)
    sx = h[0] * c + h[1] * r + h[2]
    sy = h[3] * c + h[4] * r + h[5]
    sw = h[6] * c + h[7] * r + h[8]
    with np.errstate(divide="ignore", invalid="ignore"):
        return sx / sw, sy / sw, sw > 0


def sample(hinv, c, r, H, W):
    """-> x, y, ix, iy, inside of the virtual pixels (c, r)."""
    x, y, front = to_source(hinv, c, r)
    ok = front & (np.abs(x) < 2.0 ** 24) & (np.abs(y) < 2.0 ** 24)
    ix = np.where(ok, np.rint(np.where(ok, x, 0)), -1).astype(np.int64)
    iy = np.where(ok, np.rint(np.where(ok, y, 0)), -1).astype(np.int64)
    inside = ok & (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    return x, y, ix, iy, inside


def near_tie(x, y, eps=1e-6):
    """True where x or y is within eps of a half-integer: its nearest pixel is decided by rounding alone."""
    fx, fy = np.abs(x - np.floor(x) - 0.5), np.abs(y - np.floor(y) - 0.5)
    return (fx < eps) | (fy < eps)


def recentred_box(mask, hinv):
    """xyxy (exclusive max) of the virtual pixels whose nearest frame pixel is a mask pixel, over a grid covering the
    image of the whole frame (widened by 2 px) under H; (0, 0, 0, 0) when there is none."""
    H, W = mask.shape
    Hf = np.linalg.inv(np.asarray(hinv, np.float64).reshape(3, 3))
    corners = np.array([[-1, -1, 1], [W, -1, 1], [-1, H, 1], [W, H, 1]], np.float64) @ Hf.T
    assert (corners[:, 2] > 0).all(), "the frame reaches the virtual camera's horizon"
    uv = corners[:, :2] / corners[:, 2:]
    x0, y0 = np.floor(uv.min(0)).astype(np.int64) - 2
    x1, y1 = np.ceil(uv.max(0)).astype(np.int64) + 2
    r, c = np.mgrid[y0:y1 + 1, x0:x1 + 1]
    _, _, ix, iy, inside = sample(hinv, c, r, H, W)
    hit = np.zeros_like(inside)
    hit[inside] = mask[iy[inside], ix[inside]] != 0
    if not hit.any():
        return np.zeros(4, np.int64)
    rows, cols = np.flatnonzero(hit.any(1)), np.flatnonzero(hit.any(0))
    return np.array([x0 + cols[0], y0 + rows[0], x0 + cols[-1] + 1, y0 + rows[-1] + 1], np.int64)


def recentred_crop(rgb, mask, hinv, box, T=224):
    """rgb u8 [H,W,3], mask [H,W], the virtual box -> dict(images f64 [3,T,T], mask f64 [T,T], M f32 [3,3],
    tie bool [T,T] (pixels whose nearest frame pixel is decided within 1e-6 px))."""
    H, W = mask.shape
    x1, y1, x2, y2 = (int(v) for v in box)
    w, h = x2 - x1, y2 - y1
    # float32, as the images ATen crops: its nearest index arithmetic depends on the dtype (exact below 2^24 pixels)
    assert h * w < 1 << 24
    coords = (torch.arange(h * w, dtype=torch.float64) + 1).to(torch.float32).reshape(1, h, w)
    idx, M_local = crop_aten([0, 0, w, h], coords, T)
    shift = torch.eye(3)
    shift[:2, 2] = -torch.tensor([x1, y1], dtype=torch.float32)
    M = torch.matmul(M_local, shift)
    idx = idx[0].numpy().astype(np.int64) - 1                      # -1 = padding
    pad = idx < 0
    vr, vc = np.where(pad, 0, idx // max(w, 1)) + y1, np.where(pad, 0, idx % max(w, 1)) + x1
    x, y, ix, iy, inside = sample(hinv, vc, vr, H, W)
    inside &= ~pad
    m = np.zeros((T, T))
    m[inside] = (np.asarray(mask)[iy[inside], ix[inside]] != 0).astype(np.float64)
    out = np.zeros((3, T, T))
    xs, ys = x[inside], y[inside]
    fx, fy = np.floor(xs), np.floor(ys)
    ax, ay = xs - fx, ys - fy
    xa, xb = np.clip(fx, 0, W - 1).astype(np.int64), np.clip(fx + 1, 0, W - 1).astype(np.int64)
    ya, yb = np.clip(fy, 0, H - 1).astype(np.int64), np.clip(fy + 1, 0, H - 1).astype(np.int64)
    img = np.asarray(rgb, np.float64)
    v = ((1 - ay)[:, None] * ((1 - ax)[:, None] * img[ya, xa] + ax[:, None] * img[ya, xb]) +
         ay[:, None] * ((1 - ax)[:, None] * img[yb, xa] + ax[:, None] * img[yb, xb]))
    out[:, inside] = (v / 255.0 * m[inside][:, None]).T
    out = (out - CLIP_MEAN[:, None, None]) / CLIP_STD[:, None, None]
    tie = np.zeros((T, T), bool)
    tie[~pad] = near_tie(np.where(np.isfinite(x), x, 0.0), np.where(np.isfinite(y), y, 0.0))[~pad]
    return dict(images=out, mask=m, M=M.numpy(), tie=tie)
