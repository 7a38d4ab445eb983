"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/vis_reference.npz (row f14).

Runs the libraries the reference's visualisations call (cv2 4.13, PIL, scipy) on seeded inputs, so that tests that run
where those libraries are missing (the GPU tests never import cv2) can compare against them:
  gray_*       cv2.cvtColor(RGB2GRAY) on random and extreme images
  warp_*       cv2.warpAffine of a 224 x 224 RGBA image under 20 similarity transforms (identity, scales 0.25-4,
               rotations up to 180 degrees, sub-pixel and off-crop translations, coefficients next to the fixed-point
               rounding boundaries), as SHA-256 digests of the outputs and the first three outputs in full
  paste_*      PIL Image.paste(rgb, (0, 0), alpha) with partial alpha, and an L mask pasted through itself
  dil_*        scipy.ndimage.binary_dilation with np.ones((2, 2)) and np.ones((3, 3))
  turbo        cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_TURBO) in RGB order
  kabsch_*     plot_Kabsch's pipeline (src/libVis/torch.py) on normalised crops (vis_port.crop_from_u8 of the
               stored u8 planes) with cv2, PIL and scipy, with the
               boundary edge of vis.cu in place of skimage's canny (skimage is not installed)
Nothing under the reference checkout is read.

    python -m oracle.make_golden_vis
"""
import hashlib
import os

import cv2
import numpy as np
from PIL import Image
from scipy.ndimage import binary_dilation

from oracle import vis_port as P

WARP_FULL = 3
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "vis_reference.npz")


def similarity(scale, deg, tx, ty, cx=112.0, cy=112.0):
    a = np.deg2rad(deg)
    R = scale * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = np.array([cx, cy]) + np.array([tx, ty]) - R @ np.array([cx, cy])
    M = np.eye(3)
    M[:2, :2], M[:2, 2] = R, t
    return M.astype(np.float32)


def warp_matrices():
    Ms = [np.eye(3, dtype=np.float32)]
    for s in (0.25, 0.5, 0.9, 1.37, 2.0, 4.0):
        Ms.append(similarity(s, 0.0, 0.0, 0.0))
    for deg in (7.5, 45.0, 90.0, -120.0, 180.0):
        Ms.append(similarity(1.0, deg, 0.0, 0.0))
    Ms += [similarity(1.0, 0.0, 0.25, -0.75), similarity(0.8, 30.0, 3.3, 1.1), similarity(1.0, 0.0, 200.0, -150.0),
           similarity(1.5, -60.0, -300.0, 50.0)]
    # coefficients that put destination coordinates exactly on (and one ulp off) the 1/1024 and 1/32 grids
    for d in (1 / 2048, 1 / 64, 1 / 64 + 2 ** -30, 1 / 2048 - 2 ** -30):
        M = np.eye(3, dtype=np.float32)
        M[0, 2], M[1, 2] = d, -d
        Ms.append(M)
    return np.stack(Ms)


def crops(rng, n):
    """u8 crops [n,3,224,224] and masks [n,224,224] (rings of colour on a gradient, soft mask rims); the normalised f32
    crops are vis_port.crop_from_u8 of them."""
    yy, xx = np.mgrid[0:224, 0:224].astype(np.float32)
    imgs, masks = [], []
    for _ in range(n):
        cx, cy, r = rng.uniform(60, 164), rng.uniform(60, 164), rng.uniform(30, 90)
        d = np.sqrt((xx - cx) ** 2 + (yy - cy) ** 2)
        m = np.clip((r - d) / 3.0, 0, 1)
        rgb = np.stack([(xx / 223) * rng.uniform(0.3, 1), (yy / 223) * rng.uniform(0.3, 1),
                        0.5 + 0.5 * np.sin(d / rng.uniform(5, 20))])
        imgs.append(np.clip(np.rint(rgb * 255), 0, 255).astype(np.uint8))
        masks.append(np.rint(m * 255).astype(np.uint8))
    return np.stack(imgs), np.stack(masks)


def kabsch_reference(query, qmask, tmpl, tmask, M):
    """plot_Kabsch for one triple with cv2 / PIL / scipy, the boundary edge in place of canny."""
    def edge_from_mask(mask_pil):
        tmp = Image.new("L", mask_pil.size, 0)
        tmp.paste(mask_pil, (0, 0), mask_pil)
        return binary_dilation(P.boundary_edge(np.array(tmp) > 0), np.ones((3, 3)))

    src_img, tar_img = P.unnormalise(tmpl), P.unnormalise(query)
    src_mask, tar_mask = P.mask_u8(tmask), Image.fromarray(P.mask_u8(qmask))
    src_rgba = np.concatenate([src_img, src_mask[:, :, None]], axis=2)
    tar = cv2.cvtColor(cv2.cvtColor(tar_img, cv2.COLOR_RGB2GRAY), cv2.COLOR_GRAY2RGB)
    tar = Image.fromarray(tar)
    wrap = Image.fromarray(cv2.warpAffine(src_rgba, M[:2].astype(np.float64), (224, 224)))
    alpha = wrap.getchannel("A")
    tar.paste(wrap.convert("RGB"), (0, 0), alpha)
    e_src, e_tar = edge_from_mask(alpha), edge_from_mask(tar_mask)
    out = np.array(tar.convert("RGB"))
    out[e_src] = (255, 0, 0)
    out[e_tar] = (0, 255, 0)
    return out


def main():
    rng = np.random.default_rng(14)
    out = {}
    g = [rng.integers(0, 256, (61, 97, 3), dtype=np.uint8)]
    ext = np.array(np.meshgrid([0, 1, 127, 128, 254, 255], [0, 1, 127, 128, 254, 255], [0, 1, 127, 128, 254, 255],
                               indexing="ij")).reshape(3, -1).T.astype(np.uint8)
    g.append(ext.reshape(6, 36, 3))
    out["gray_in_random"], out["gray_in_extreme"] = g
    out["gray_out_random"] = cv2.cvtColor(g[0], cv2.COLOR_RGB2GRAY)
    out["gray_out_extreme"] = cv2.cvtColor(g[1], cv2.COLOR_RGB2GRAY)

    yy, xx = np.mgrid[0:224, 0:224]
    src = np.stack([(xx * 5 + yy) % 256, (yy * 3) % 256, ((xx // 8 + yy // 8) % 2) * 255,
                    np.clip(255 - 2 * np.abs(xx - 112), 0, 255)], -1).astype(np.uint8)
    src[::23, ::19] = rng.integers(0, 256, src[::23, ::19].shape, dtype=np.uint8)
    Ms = warp_matrices()
    out["warp_src"], out["warp_M"] = src, Ms
    warped = [cv2.warpAffine(src, M[:2].astype(np.float64), (224, 224)) for M in Ms]
    # every output as a SHA-256 of its bytes (a bit-exact comparison), the first WARP_FULL also in full
    out["warp_sha256"] = np.array([hashlib.sha256(np.ascontiguousarray(w).tobytes()).hexdigest() for w in warped])
    out["warp_out"] = np.stack(warped[:WARP_FULL])

    dst = rng.integers(0, 256, (40, 50, 3), dtype=np.uint8)
    prgb = rng.integers(0, 256, (40, 50, 3), dtype=np.uint8)
    alpha = rng.integers(0, 256, (40, 50), dtype=np.uint8)
    alpha[:5] = 0
    alpha[5:10] = 255
    im = Image.fromarray(dst.copy())
    im.paste(Image.fromarray(prgb), (0, 0), Image.fromarray(alpha))
    tmp = Image.new("L", (50, 40), 0)
    tmp.paste(Image.fromarray(alpha), (0, 0), Image.fromarray(alpha))
    out.update(paste_dst=dst, paste_rgb=prgb, paste_alpha=alpha, paste_out=np.array(im), paste_self=np.array(tmp))

    edge = rng.random((37, 41)) < 0.08
    edge[0, 0] = edge[-1, -1] = edge[0, -1] = edge[-1, 0] = True
    out["dil_in"] = edge
    out["dil_2"] = binary_dilation(edge, np.ones((2, 2)))
    out["dil_3"] = binary_dilation(edge, np.ones((3, 3)))

    out["turbo"] = cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_TURBO).reshape(256, 3)[:, ::-1].copy()

    n = 6
    q8, qm8 = crops(rng, n)
    t8, tm8 = crops(rng, n)
    (q, qm), (t, tm) = P.crop_from_u8(q8, qm8), P.crop_from_u8(t8, tm8)
    KM = np.stack([np.eye(3, dtype=np.float32), similarity(1.2, 20.0, 4.5, -3.25), similarity(0.6, -75.0, 10.0, 2.0),
                   similarity(1.0, 180.0, 0.5, 0.5), similarity(2.5, 10.0, -40.0, 30.0), similarity(0.9, 0.0, 150.0, 0.0)])
    out.update(kabsch_query_u8=q8, kabsch_query_mask_u8=qm8, kabsch_tmpl_u8=t8, kabsch_tmpl_mask_u8=tm8, kabsch_M=KM)
    out["kabsch_out"] = np.stack([kabsch_reference(q[i], qm[i], t[i], tm[i], KM[i]) for i in range(n)])
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
