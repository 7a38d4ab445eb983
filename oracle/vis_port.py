"""TEST INFRASTRUCTURE ONLY -- not part of the product path.

Row f14: the four contracts of gigapose_b200/csrc/vis.cu restated in numpy (the header comment of vis.cu states them):
per-vertex ADD / ADD-S errors, heat-map colours, the grey overlay with contours, and the Kabsch retrieval panel with
cv2.warpAffine's fixed-point bilinear warp and PIL's paste blend.  tests/test_vis_cpu.py checks it against cv2 4.13,
PIL and scipy (live and through tests/golden/vis_reference.npz); tests/test_gpu_vis.py checks the kernels against it.
"""
import numpy as np

from oracle.add_port import F32, add_terms

CROP = 224                                               # GP_VIS_CROP
# the reference's inverse ImageNet normalisation (src/libVis/torch.py: inv_rgb_transform), each a double rounded to f32
INV_MEAN = np.array([-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225], F32)
INV_STD = np.array([1 / 0.229, 1 / 0.224, 1 / 0.225], F32)


# ---------------------------------------------------------------------------------------------- pixels
def gray(img):
    """cv2.cvtColor(img, COLOR_RGB2GRAY) on u8 [..., 3]: (9798 r + 19235 g + 3735 b + 2^14) >> 15."""
    x = np.asarray(img).astype(np.int64)
    return ((9798 * x[..., 0] + 19235 * x[..., 1] + 3735 * x[..., 2] + 16384) >> 15).astype(np.uint8)


def np_uint8(x):
    """np.uint8 of fp32 values on x86: truncation to int32 (INT_MIN outside its range and for NaN), low 8 bits."""
    x = np.asarray(x, F32)
    with np.errstate(invalid="ignore"):
        ok = np.abs(x) < F32(2147483648.0)
        t = np.trunc(np.where(ok, x, 0)).astype(np.int64)
    return (np.where(ok, t, 0) & 255).astype(np.uint8)


CLIP_MEAN = np.array([0.48145466, 0.4578275, 0.40821073], F32)
CLIP_STD = np.array([0.26862954, 0.26130258, 0.27577711], F32)


def crop_from_u8(rgb, mask):
    """Normalised crop f32 [..., 3, H, W] and mask f32 [..., H, W] from u8 planes: (rgb / 255 - mean) / std in fp32, as
    the fixtures store their crops."""
    x = (np.asarray(rgb, np.uint8).astype(F32) / F32(255)).astype(F32)
    x = ((x - CLIP_MEAN[:, None, None]).astype(F32) / CLIP_STD[:, None, None]).astype(F32)
    return x, (np.asarray(mask, np.uint8).astype(F32) / F32(255)).astype(F32)


def unnormalise(crop):
    """convert_tensor_to_image of f32 [3, H, W] -> u8 [H, W, 3]."""
    c = np.asarray(crop, F32)
    with np.errstate(all="ignore"):
        x = ((c - INV_MEAN[:, None, None]).astype(F32) / INV_STD[:, None, None]).astype(F32)
        x = (x * F32(255)).astype(F32)
    return np_uint8(x).transpose(1, 2, 0)


def mask_u8(mask):
    with np.errstate(all="ignore"):
        return np_uint8((np.asarray(mask, F32) * F32(255)).astype(F32))


def boundary_edge(mask):
    """Mask pixels with a 4-neighbour outside the mask or outside the image."""
    m = np.pad(np.asarray(mask, bool), 1)
    inner = m[:-2, 1:-1] & m[2:, 1:-1] & m[1:-1, :-2] & m[1:-1, 2:]
    return m[1:-1, 1:-1] & ~inner


def dilate2(edge):
    """scipy.ndimage.binary_dilation(edge, np.ones((2, 2))): (y, x) is set when an edge lies at (y..y+1, x..x+1)."""
    e = np.pad(np.asarray(edge, bool), ((0, 1), (0, 1)))
    return e[:-1, :-1] | e[1:, :-1] | e[:-1, 1:] | e[1:, 1:]


def dilate3(edge):
    """scipy.ndimage.binary_dilation(edge, np.ones((3, 3)))."""
    e = np.pad(np.asarray(edge, bool), 1)
    H, W = edge.shape
    out = np.zeros((H, W), bool)
    for dy in range(3):
        for dx in range(3):
            out |= e[dy:dy + H, dx:dx + W]
    return out


def div255(t):
    t = np.asarray(t, np.int64) + 128
    return ((t >> 8) + t) >> 8


def paste(dst, src_rgb, alpha):
    """PIL Image.paste(src, (0, 0), alpha) of RGB images (u8 [H, W, 3]) through an L mask u8 [H, W]."""
    a = np.asarray(alpha, np.int64)[..., None]
    return div255(np.asarray(dst, np.int64) * (255 - a) + np.asarray(src_rgb, np.int64) * a).astype(np.uint8)


def self_pasted(mask):
    """create_edge_from_mask's L image: the mask pasted onto black through itself, DIV255(a a)."""
    a = np.asarray(mask, np.int64)
    return div255(a * a).astype(np.uint8)


# ---------------------------------------------------------------------------------------------- warpAffine
def _inverse(M):
    M = np.asarray(M, np.float64).reshape(-1)[:6]
    a, b, c, d, e, f = (float(v) for v in M)
    D = a * e - b * d
    D = 1.0 / D if D != 0 else 0.0
    A11, A22, A12, A21 = e * D, a * D, b * -D, d * -D
    return np.array([A11, A12, -A11 * c - A12 * f, A21, A22, -A21 * c - A22 * f])


def warp_affine(src, M, size=(CROP, CROP)):
    """cv2.warpAffine(src, M[:2], (W, H)) with INTER_LINEAR and BORDER_CONSTANT 0 on u8 [h, w, C]."""
    src = np.asarray(src, np.uint8)
    if src.ndim == 2:
        return warp_affine(src[..., None], M, size)[..., 0]
    W, H = size
    h, wd, C = src.shape
    iM = _inverse(M)
    xs, ys = np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64)
    X0 = np.rint((iM[1] * ys + iM[2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((iM[4] * ys + iM[5]) * 1024).astype(np.int64) + 16
    ad = np.rint(iM[0] * xs * 1024).astype(np.int64)
    bd = np.rint(iM[3] * xs * 1024).astype(np.int64)
    X = (X0[:, None] + ad[None, :]).astype(np.int32).astype(np.int64) >> 5
    Y = (Y0[:, None] + bd[None, :]).astype(np.int32).astype(np.int64) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    w = [32 * (32 - fx) * (32 - fy), 32 * fx * (32 - fy), 32 * (32 - fx) * fy, 32 * fx * fy]
    acc = np.zeros((H, W, C), np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = sy + dy, sx + dx
        inside = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < wd)
        tap = src[np.clip(yy, 0, h - 1), np.clip(xx, 0, wd - 1)].astype(np.int64)
        acc += np.where(inside[..., None], w[k][..., None] * tap, 0)
    return np.minimum((acc + 16384) >> 15, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------- the four entry points
def vertex_errors(vertices, pose_est, pose_gt, symmetric):
    """gp_vis_vertex_errors of one pair -> f32 [V]: ADD distances, or ADD-S distances when `symmetric`."""
    add, adds, _ = add_terms(vertices, pose_est, pose_gt, np.eye(3, dtype=F32))
    return adds if symmetric else add


def heat_colors(values, symmetric, max_distance, turbo):
    """gp_vis_heat_colors of one pair -> (f32 [V, 3] colours, i64 [V] table indices, -1 for the bad colour)."""
    v = np.asarray(values, F32).astype(np.float64)
    md = np.float64(F32(max_distance))
    ext = np.concatenate([v, [0.0, md] if symmetric else [md]]) / md
    d = v / md
    with np.errstate(all="ignore"):
        lo, hi = ext.min(), ext.max()
        rng = hi - lo
        if np.isnan(rng) or not rng > 0:
            idx = np.full(len(v), -1, np.int64)
        else:
            idx = np.minimum(np.trunc(((d - lo) / rng) * 256.0).astype(np.int64), 255)
    table = np.asarray(turbo, np.uint8).reshape(256, 3)
    col = np.where(idx[:, None] >= 0, (table[np.maximum(idx, 0)].astype(F32) / F32(255)).astype(F32), F32(0))
    return col.astype(F32), idx


def overlay(image, renders, boxes, colors):
    """gp_vis_overlay: image u8 [H, W, 3] or None (black), renders f32 [n, 4, H, W], boxes [n, 4] (unused: the result
    does not depend on them), colors u8 [n, 3] or None -> u8 [H, W, 3]."""
    renders = np.asarray(renders, F32)
    H, W = renders.shape[-2:] if image is None else np.asarray(image).shape[:2]
    out = np.zeros((H, W, 3), np.uint8) if image is None else np.repeat(gray(image)[..., None], 3, 2)
    for l in range(len(renders)):
        m = renders[l, 3] > 0
        rgb = np.clip(np.rint((renders[l, :3] * F32(255)).astype(F32)), 0, 255).astype(np.uint8).transpose(1, 2, 0)
        out[m] = rgb[m]
        if colors is not None:
            out[dilate2(boundary_edge(m))] = np.asarray(colors, np.uint8)[l]
    return out


def contour(mask):
    """The pixels gp_vis_overlay paints in a layer's outline colour."""
    return dilate2(boundary_edge(mask))


def kabsch_panel(query, query_mask, tmpl, tmpl_mask, M):
    """gp_vis_kabsch of one triple -> u8 [224, 224, 3] (plot_Kabsch without the keypoint panel)."""
    q = unnormalise(query)
    g = np.repeat(gray(q)[..., None], 3, 2)
    rgba = np.concatenate([unnormalise(tmpl), mask_u8(tmpl_mask)[..., None]], 2)
    warped = warp_affine(rgba, np.asarray(M, np.float64).reshape(3, 3)[:2])
    a = warped[..., 3]
    out = paste(g, warped[..., :3], a)
    out[dilate3(boundary_edge(self_pasted(a) > 0))] = (255, 0, 0)
    out[dilate3(boundary_edge(self_pasted(mask_u8(query_mask)) > 0))] = (0, 255, 0)
    return out
