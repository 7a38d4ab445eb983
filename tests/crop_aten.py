"""Row f3's crop restated in plain ATen, independently of `oracle.port` and of the kernel's hand-derived index maps.

`CropResizePad.__call__` (the reference's query and template crop) is a sequence of stock ATen calls on the CPU:

  1. `scale = T / sizes.max()`: an int64 tensor under `Tensor.__rtruediv__`, so a float32 reciprocal times T;
  2. the slice `image[:, y1:y2, x1:x2]` (python slicing: upper bounds clip to the image);
  3. `F.interpolate(crop, scale_factor=scale.item())`, nearest;
  4. when the resized crop is not square, `F.pad` centred: top / left take the floor of half the difference;
  5. `F.interpolate(..., size=(T, T))`, nearest, which restores a row or column lost to rounding;
  6. `M = M_resize_pad @ M_crop` in float32 with `torch.matmul`.

`crop_aten` runs exactly those calls.  `geometry` names the branch of ATen's nearest-index arithmetic each box reaches,
so that a sweep can prove it exercised every one.  `MUTATIONS` are one-rule-wrong variants of `crop_aten`: a sweep
that cannot tell each of them from `crop_aten` is too weak to pin the kernel.  Only numpy and torch are used.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

# one-rule-wrong variants of crop_aten
MUTATIONS = ("one_division",        # scale = float32(T / side), one rounding instead of reciprocal-then-multiply
             "double_index",        # first resize: source index floor(dst * (1 / scale)) in double, not float32
             "no_small_rules",      # first resize: float32 index arithmetic even when out_h + out_w <= 128
             "ceil_padding",        # the odd pixel of the padding goes to the top / left instead of the bottom / right
             "no_second_resize")    # the final resize to T x T is skipped

# ATen's CPU nearest resize hands outputs with out_h + out_w <= SMALL_OUTPUT to a kernel whose index function maps an
# unchanged size by the identity and an exactly doubled size by dst >> 1 instead of the float32 arithmetic
SMALL_OUTPUT = 128


def box_scale(box, T: int, mutation: str | None = None) -> torch.Tensor:
    """The reference's float32 scale of an xyxy box: `T / max(w, h)` on int64 sizes (two roundings)."""
    b = torch.as_tensor(box, dtype=torch.int64).reshape(4)
    sizes = torch.stack([b[2] - b[0], b[3] - b[1]])
    if mutation == "one_division":
        return torch.tensor(float(T), dtype=torch.float32) / sizes.max().to(torch.float32)
    return T / sizes.max()


def _index(out_size: int, in_size: int, scale: float, small: bool, in_double: bool) -> torch.Tensor:
    dst = torch.arange(out_size)
    if small and out_size == in_size:
        return dst
    if small and out_size == 2 * in_size:
        return dst >> 1
    if in_double:
        idx = torch.floor(dst.to(torch.float64) * (1.0 / scale))
    else:
        idx = torch.floor(dst.to(torch.float32) * torch.tensor(1.0 / scale, dtype=torch.float32))
    return idx.long().clamp(max=in_size - 1)


def _first_resize(crop: torch.Tensor, scale: float, mutation: str | None) -> torch.Tensor:
    if mutation not in ("double_index", "no_small_rules"):
        return F.interpolate(crop[None], scale_factor=scale)[0]
    # the mutated index maps, written out as a gather (the output size is ATen's: floor(in * scale) in double)
    h, w = crop.shape[-2:]
    rh, rw = math.floor(h * scale), math.floor(w * scale)
    small = rh + rw <= SMALL_OUTPUT and mutation != "no_small_rules"
    rows = _index(rh, h, scale, small, mutation == "double_index")
    cols = _index(rw, w, scale, small, mutation == "double_index")
    return crop[:, rows][:, :, cols]


def pads(rh: int, rw: int, T: int, mutation: str | None = None):
    """(pad_left, pad_right, pad_top, pad_bottom) of a resized crop rh x rw, None when it is square (no padding)."""
    if rw == rh:
        return None
    div = (lambda a: -(-a // 2)) if mutation == "ceil_padding" else (lambda a: a // 2)
    pad_top = div(T - rh)
    pad_bottom = max(T - rh - pad_top, 0)
    pad_left = max(div(T - rw), 0)
    pad_right = T - rw - pad_left
    return pad_left, pad_right, pad_top, pad_bottom


@torch.no_grad()
def crop_aten(box, image: torch.Tensor, T: int, mutation: str | None = None, clamp_origin: bool = False):
    """The reference's crop of one xyxy int box from image [C,H,W] (CPU) -> (crop [C,T,T], M [3,3] float32).

    Raises where the reference raises: a crop or resized crop with no rows or columns.  `clamp_origin` clamps the
    slice bounds to 0 instead of letting a negative one wrap to the far edge (the scale and M still come from the box
    as given): the kernel's documented reading of a box with a negative top-left corner."""
    assert mutation is None or mutation in MUTATIONS, mutation
    b = torch.as_tensor(box, dtype=torch.int64).reshape(4)
    x1, y1, x2, y2 = (int(v) for v in b)
    scale = box_scale(b, T, mutation)
    if clamp_origin:
        x1, y1, x2, y2 = max(x1, 0), max(y1, 0), max(x2, 0), max(y2, 0)
    x = _first_resize(image[:, y1:y2, x1:x2], scale.item(), mutation)
    M_crop, M_resize_pad = torch.eye(3), torch.eye(3)
    M_crop[:2, 2] = -b[:2]
    M_resize_pad[:2, :2] *= scale
    rh, rw = x.shape[-2:]
    p = pads(rh, rw, T, mutation) if rw / rh != 1 else None
    if p is not None:
        x = F.pad(x, list(p))
        M_resize_pad[:2, 2] = torch.tensor([p[0], p[2]])
    M = torch.matmul(M_resize_pad, M_crop)
    if mutation != "no_second_resize":
        x = F.interpolate(x[None], size=(T, T))[0]
    return x, M


def geometry(box, H: int, W: int, T: int, clamp_origin: bool = False) -> dict:
    """The branches one box reaches in the reference's crop of an H x W image, from the same steps in plain python:
    crop size (ch, cw) after slicing, resized size (rh, rw), padding `pads` (None when square), the first resize's
    index rule per axis (`rule_h`, `rule_w`: "identity", "double" or "float" in the small-output kernel, "plain"
    otherwise), and whether the second resize is the identity.  `empty` marks boxes where the reference raises (no
    rows or columns to resize).  `clamp_origin` as in `crop_aten`."""
    x1, y1, x2, y2 = (int(v) for v in box)
    scale = box_scale(box, T).item()
    if clamp_origin:
        x1, y1, x2, y2 = max(x1, 0), max(y1, 0), max(x2, 0), max(y2, 0)
    ch = len(range(*slice(y1, y2).indices(H)))
    cw = len(range(*slice(x1, x2).indices(W)))
    rh, rw = math.floor(ch * scale), math.floor(cw * scale)
    g = dict(ch=ch, cw=cw, rh=rh, rw=rw, scale=scale, empty=min(ch, cw, rh, rw) == 0)
    if g["empty"]:
        return g
    small = rh + rw <= SMALL_OUTPUT

    def rule(out_size, in_size):
        if not small:
            return "plain"
        return "identity" if out_size == in_size else "double" if out_size == 2 * in_size else "float"

    g["rule_h"], g["rule_w"] = rule(rh, ch), rule(rw, cw)
    g["pads"] = p = pads(rh, rw, T)
    ph, pw = (rh, rw) if p is None else (rh + p[2] + p[3], rw + p[0] + p[1])
    g["second_identity"] = (ph, pw) == (T, T)
    return g


def branches(g: dict) -> list:
    """The branch names one `geometry` counts towards (for coverage tallies)."""
    if g["empty"]:
        return ["empty"]
    out = ["small" if g["rule_h"] != "plain" else "plain"]
    out += sorted({f"small_{g['rule_h']}", f"small_{g['rule_w']}"} - {"small_plain"})
    if g["pads"] is None:
        out.append("square")
    else:
        out.append("padded")
        for name, v in zip(("left", "right", "top", "bottom"), g["pads"]):
            out.append(f"pad_{name}_{'odd' if v % 2 else 'even'}")
    out.append("second_identity" if g["second_identity"] else "second_resize")
    return out


ALL_BRANCHES = ("plain", "small", "small_identity", "small_double", "small_float", "square", "padded",
                "pad_left_odd", "pad_left_even", "pad_right_odd", "pad_right_even", "pad_top_odd", "pad_top_even",
                "pad_bottom_odd", "pad_bottom_even", "second_identity", "second_resize")

# image sizes (H, W) of the sweep
IMAGES = ((17, 23), (480, 640), (1080, 1920))


def planted(T: int):
    """Boxes placed on purpose in the small-output kernel's identity and doubling rules, with scales just above 1 and
    2 (where the float32 index arithmetic differs from both rules): (H, W, box)."""
    out = []
    for side in (T - 1, T, T // 2 - 1, T // 2):
        for keep_h, keep_w in ((10, 50), (50, 10), (1, 1), (20, 20), (5, 40), (30, 33)):
            for H, W in ((480, 640), (1080, 1920)):
                out.append((H, W, (W - keep_w, H - keep_h, W - keep_w + side, H - keep_h + side)))
    return out


def sweep(T: int):
    """(H, W, box, clamp) of the whole sweep at target size T; `clamp` marks boxes with a negative top-left corner,
    which the kernel reads with the corner clamped to 0 (`crop_aten(..., clamp_origin=True)`).  Boxes where the
    reference raises (`geometry(...)["empty"]`) are left out."""
    out = []
    for side in range(1, 2 * T + 1):                                    # every square side at a fixed origin
        out.append((480, 640, (5, 3, 5 + side, 3 + side)))
    for k, long in enumerate((T // 2 + 1, T - 1, T + 1, 2 * T - 1)):  # every short side, both orientations
        x0, y0 = 7 + 3 * k, 11 + k
        for short in range(1, long + 1):
            out.append((1080, 1920, (x0, y0, x0 + long, y0 + short)))
            out.append((1080, 1920, (x0, y0, x0 + short, y0 + long)))
    sizes = ((T // 3, T // 5), (T - 1, T - 1), (T // 2 - 1, T + 7), (2 * T + 9, 3 * T // 2))
    for H, W in IMAGES[:2]:                                             # overhanging each border and pair of borders
        for sides in range(1, 16):
            left, top, right, bottom = (bool(sides >> i & 1) for i in range(4))
            for d in range(41):
                w, h = sizes[(d + sides) % len(sizes)]
                x1 = -d if left else (W - w + d if right else (W - min(w, W)) // 2)
                y1 = -d if top else (H - h + d if bottom else (H - min(h, H)) // 2)
                x2 = W + d if right else x1 + w
                y2 = H + d if bottom else y1 + h
                out.append((H, W, (x1, y1, x2, y2)))
    for H, W, box in planted(T):
        out.append((H, W, box))
    res = []
    for H, W, box in out:
        clamp = box[0] < 0 or box[1] < 0
        if not geometry(box, H, W, T, clamp_origin=clamp)["empty"]:
            res.append((H, W, box, clamp))
    return res


def coordinate_image(C: int, H: int, W: int) -> torch.Tensor:
    """f32 [C,H,W] whose pixel (c, r, x) holds 1 + c * H * W + r * W + x (exact in float32 up to 1080 x 1920 x 4):
    cropping it yields each output pixel's source index, 0 where the output is padding."""
    return (torch.arange(C * H * W, dtype=torch.float64) + 1).to(torch.float32).reshape(C, H, W)


def ulp_distance(a, b) -> np.ndarray:
    """Units in the last place between float32 arrays a and b (same sign assumed away: ordered integer distance)."""
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)
