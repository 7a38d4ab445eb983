"""Row f3 on the GPU: `crop_resize_pad_kernel` (csrc/preprocess.cu) and its run-length form pinned to the reference's
crop in plain ATen (`tests/crop_aten.py`), bit for bit, over the crop sweep at T = 224, 160 and 128: the dense query
path with 1 to 4 channels, the fused /255, x mask, CLIP path, the run-length path on masks decoded from their runs, and
the template path of `GigaPose.template_crops`.  ATen runs once per distinct geometry, on a coordinate image whose crop
is each output pixel's source index; the expected crops of random images are gathers through that index map.  Also
pins M, and the boxes where the reference has no crop and the kernel writes zeros (DESIGN.md row f3).  Each test
prints the boxes it compared and the worst ulp distance of the kernel's M translations to ATen's float32 matmul."""
import collections
import types

import numpy as np
import pytest
import torch

from crop_aten import IMAGES, box_scale, coordinate_image, crop_aten, geometry, pads, sweep, ulp_distance
from gigapose_b200 import preprocess

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TARGETS = (224, 160, 128)
MEAN = torch.tensor(preprocess.CLIP_MEAN, dtype=torch.float32).view(3, 1, 1)
STD = torch.tensor(preprocess.CLIP_STD, dtype=torch.float32).view(3, 1, 1)


def _maps(T, H, W, boxes, clamps):
    """ATen's source index of every output pixel, int64 [n,T,T] (-1 where padding), and its M [n,3,3], per box.  The
    map comes from a one-channel image; each test also crops one box per batch straight from its C-channel image."""
    coords = coordinate_image(1, H, W)
    idx, Ms = [], []
    for box, clamp in zip(boxes, clamps):
        x, M = crop_aten(box, coords, T, clamp_origin=clamp)
        idx.append(x[0].to(torch.int64) - 1)
        Ms.append(M)
    return torch.stack(idx), torch.stack(Ms)


def _gather(planes, image_index, idx):
    """planes f32 [m,C,H*W], image_index [n], idx [n,T,T] -> [n,C,T,T]: the pixel each index names, 0 on padding."""
    m, C, HW = planes.shape
    n, T, _ = idx.shape
    lin = (image_index.view(n, 1, 1) * C + torch.arange(C).view(1, C, 1)) * HW + idx.clamp(min=0).view(n, 1, T * T)
    v = torch.take(planes, lin).view(n, C, T, T)
    return torch.where(idx[:, None] >= 0, v, torch.zeros((), dtype=planes.dtype))


def _mask_values(det, pix):
    """A fixed {0,1} mask per detection, computable at any pixel without building it: det [n,1,1], pix [..] int64."""
    return (((pix * 2654435761 + det * 40503) >> 7) % 5 != 0).to(torch.float32)


def _check_M(T, H, W, boxes, clamps, got, want):
    """Scale and constant entries equal to ATen's; translations equal to s * (-x1) + pad rounded once from fp64 (the
    kernel's fmaf), and within one ulp (at the larger of the product and the result) of ATen's float32 matmul, which
    may round the product before adding the padding.  Returns the largest ulp distance to ATen's translations."""
    got, want = got.cpu(), want.cpu()
    worst = 0
    rows, cols = [0, 0, 1, 1, 2, 2, 2], [0, 1, 0, 1, 0, 1, 2]
    assert torch.equal(got[:, rows, cols], want[:, rows, cols]), "M's scale or constant entries differ from ATen's"
    for i, (box, clamp) in enumerate(zip(boxes, clamps)):
        g = geometry(box, H, W, T, clamp_origin=clamp)
        s = float(box_scale(box, T))
        p = g["pads"] or (0, 0, 0, 0)
        exact = np.array([s * -box[0] + p[0], s * -box[1] + p[2]])                # exact in fp64
        assert np.array_equal(got[i, :2, 2].numpy(), exact.astype(np.float32)), (box, got[i].tolist(), exact)
        worst = max(worst, int(ulp_distance(got[i, :2, 2], want[i, :2, 2]).max()))
        bar = float(np.spacing(np.float32(max(abs(s * box[0]), abs(s * box[1]), np.abs(exact).max(), T))))
        assert float((got[i, :2, 2] - want[i, :2, 2]).abs().max()) <= bar, (box, got[i].tolist(), want[i].tolist())
    return worst


def _report(path, T, n, worst):
    print(f"{path} T={T}: {n} boxes equal to ATen's crop; M translations == fp64 s * (-x1) + pad rounded once, worst "
          f"distance to ATen's float32 matmul {worst} ulp")


def _groups(T):
    by = collections.defaultdict(list)
    for H, W, box, clamp in sweep(T):
        by[(H, W)].append((box, clamp))
    return by


@pytest.mark.parametrize("T", TARGETS)
def test_dense_and_fused_query_crops_equal_aten(T):
    gen = torch.Generator().manual_seed(T)
    chunk_no = n_dense = n_clamped = worst = 0
    for (H, W), entries in sorted(_groups(T).items()):
        chunk = int(min(128, max(16, 2 ** 26 // (H * W))))
        rgb_u8 = torch.randint(0, 256, (3, 3, H, W), generator=gen, dtype=torch.uint8)
        rgb_planes = rgb_u8.to(torch.float32).view(3, 3, H * W)
        rgb_dev = rgb_u8.to(DEV)
        pix = torch.arange(H * W, device=DEV).view(1, H, W)
        for c0 in range(0, len(entries), chunk):
            part = entries[c0:c0 + chunk]
            boxes = [b for b, _ in part]
            clamps = [c for _, c in part]
            n = len(boxes)
            idx, M_aten = _maps(T, H, W, boxes, clamps)
            boxes_t = torch.tensor(boxes, dtype=torch.int64)
            image_index = torch.randint(0, 3, (n,), generator=gen)
            # dense: 1 to 4 channels, several detections per image
            C = 1 + chunk_no % 4
            chunk_no += 1
            images = torch.rand(3, C, H, W, generator=gen)
            got = preprocess.crop_resize_pad(boxes_t.to(DEV), images.to(DEV), T, image_index=image_index.to(DEV))
            got = {k: v.cpu() for k, v in got.items()}
            want = _gather(images.view(3, C, H * W), image_index, idx)
            bad = [i for i in range(n) if not torch.equal(got["images"][i], want[i])]
            assert not bad, f"T={T} image {H}x{W}: dense crop differs from ATen for boxes {[boxes[i] for i in bad[:8]]}"
            # ATen straight on the C-channel image, for one box per chunk
            direct, _ = crop_aten(boxes[0], images[image_index[0]], T, clamp_origin=clamps[0])
            assert torch.equal(got["images"][0], direct), boxes[0]
            worst = max(worst, _check_M(T, H, W, boxes, clamps, got["M"], M_aten))
            n_dense += n
            n_clamped += sum(clamps)
            # fused: rgb / 255, x mask, crop of the 4 channels, CLIP on the rgb ones
            det = torch.arange(n, device=DEV).view(n, 1, 1) + c0
            masks = _mask_values(det, pix)
            got = preprocess.preprocess_queries(rgb_dev, masks, boxes_t.to(DEV), image_index.to(DEV), T)
            got = {k: v.cpu() for k, v in got.items()}
            m = torch.where(idx >= 0, _mask_values(det.cpu(), idx.clamp(min=0)), torch.zeros(()))
            rgb = _gather(rgb_planes, image_index, idx) / 255.0 * m[:, None]
            want_img = (rgb - MEAN) / STD
            assert torch.equal(got["tar_mask"], m), f"T={T} image {H}x{W}: fused mask differs"
            bad = [i for i in range(n) if not torch.equal(got["tar_img"][i], want_img[i])]
            assert not bad, f"T={T} image {H}x{W}: fused crop differs for boxes {[boxes[i] for i in bad[:8]]}"
            worst = max(worst, _check_M(T, H, W, boxes, clamps, got["tar_M"], M_aten))
    _report(f"dense and fused ({n_clamped} with a negative corner, read clamped to 0)", T, n_dense, worst)


def _rle_encode(mask):
    """COCO run-length counts of a {0,1} mask [H,W]: column-major runs, the first one counting zeros."""
    flat = np.asarray(mask, bool).flatten(order="F")
    bounds = np.concatenate([[0], np.flatnonzero(flat[1:] != flat[:-1]) + 1, [flat.size]])
    counts = np.diff(bounds)
    return (np.concatenate([[0], counts]) if flat[0] else counts).astype(np.int32)


def _rle_decode(counts, H, W):
    return np.repeat(np.arange(len(counts)) % 2, counts).astype(bool).reshape(W, H).T


def _rle_boxes(T, H, W):
    """Mask boxes for the run-length path: the sweep's boxes inside the image, masks touching each border of it, a
    one-pixel mask and single-row / single-column masks."""
    out = [box for h, w, box, clamp in sweep(T) if (h, w) == (H, W) and not clamp and box[2] <= W and box[3] <= H]
    out += [(0, 0, 1, 1), (W - 1, H - 1, W, H), (0, 0, W, H), (0, 3, 7, H - 2), (W - 9, 2, W, 11), (3, 0, W - 5, 4),
            (1, H - 6, 9, H), (0, H // 2, min(W, T), H // 2 + 1), (W // 3, 0, W // 3 + 1, min(H, T))]
    return [box for box in out if not geometry(box, H, W, T)["empty"]]


@pytest.mark.parametrize("T", TARGETS)
def test_run_length_crops_equal_aten(T):
    """crop_detections_rle (gp_crop_resize_pad_rle) against rgb / 255, x the mask decoded from its runs, ATen's crop,
    CLIP; each box computed from the decoded runs."""
    rng = np.random.default_rng(T)
    n_rle = worst = 0
    for H, W in IMAGES[:2]:
        boxes = _rle_boxes(T, H, W)
        counts, got_boxes, masks = [], [], []
        for x1, y1, x2, y2 in boxes:
            m = np.zeros((H, W), bool)
            m[y1:y2, x1:x2] = rng.random((y2 - y1, x2 - x1)) < 0.6
            m[y1, rng.integers(x1, x2)] = m[y2 - 1, rng.integers(x1, x2)] = True      # the box touches every side
            m[rng.integers(y1, y2), x1] = m[rng.integers(y1, y2), x2 - 1] = True
            c = _rle_encode(m)
            d = _rle_decode(c, H, W)
            rows, cols = np.flatnonzero(d.any(1)), np.flatnonzero(d.any(0))
            got_boxes.append((int(cols[0]), int(rows[0]), int(cols[-1]) + 1, int(rows[-1]) + 1))
            counts.append(c)
            masks.append(torch.from_numpy(d.reshape(-1)).to(torch.float32))
        assert got_boxes == [tuple(b) for b in boxes]
        n = len(boxes)
        rgb = torch.randint(0, 256, (2, H, W, 3), generator=torch.Generator().manual_seed(T + H), dtype=torch.uint8)
        image_index = torch.arange(n) % 2
        off = np.concatenate([[0], np.cumsum([len(c) for c in counts])])
        got = preprocess.crop_detections_rle(rgb.to(DEV), np.concatenate(counts), off, got_boxes, image_index, T)
        got = {k: v.cpu() for k, v in got.items()}
        idx, M_aten = _maps(T, H, W, got_boxes, [False] * n)
        m = _gather(torch.stack(masks)[:, None], torch.arange(n), idx)[:, 0]
        want = (_gather(rgb.permute(0, 3, 1, 2).reshape(2, 3, H * W).to(torch.float32), image_index, idx) / 255.0
                * m[:, None] - MEAN) / STD
        assert torch.equal(got["tar_mask"], m), f"T={T} image {H}x{W}: run-length mask differs"
        bad = [i for i in range(n) if not torch.equal(got["tar_img"][i], want[i])]
        assert not bad, f"T={T} image {H}x{W}: run-length crop differs for boxes {[got_boxes[i] for i in bad[:8]]}"
        worst = max(worst, _check_M(T, H, W, got_boxes, [False] * n, got["tar_M"], M_aten))
        n_rle += n
    _report("run-length", T, n_rle, worst)


def test_template_crops_equal_aten():
    """GigaPose.template_crops (the crop of GigaPose._onboard) on 640 x 480 RGBA renders with PIL boxes: ATen's crop,
    then CLIP on the rgb channels and mean 0, std 1 on the alpha channel."""
    from PIL import Image
    from src.models.gigaPose import GigaPose
    H, W, n = 480, 640, 48
    gen = torch.Generator().manual_seed(4)
    rgba = torch.randint(0, 256, (n, 4, H, W), generator=gen, dtype=torch.uint8).to(torch.float32) / 255.0
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    for i in range(n):                                   # silhouettes from one pixel to the whole frame, some at edges
        ry, rx = (0.5 + (i * 37 % 97) / 96 * (H / 1.8), 0.5 + (i * 53 % 89) / 88 * (W / 1.8))
        cy, cx = (i * 71 % H, i * 113 % W) if i % 3 else (H / 2, W / 2)
        rgba[i, 3] = (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).to(torch.float32)
    rgba[0, 3] = 0
    rgba[0, 3, 200, 300] = 1                             # one pixel
    rgba[1, 3] = 1                                       # the whole frame
    boxes = torch.tensor([Image.fromarray((rgba[i, 3] * 255).to(torch.uint8).numpy()).getbbox() for i in range(n)])
    model = types.SimpleNamespace(template_views={"t": lambda o, ids: (rgba[ids].to(DEV), boxes[ids])}, device=DEV)
    ids = list(range(n))
    rgb, mask = (t.cpu() for t in GigaPose.template_crops(model, "t", 0, ids))
    for i in ids:
        x, _ = crop_aten(boxes[i].tolist(), rgba[i], 224)
        assert torch.equal(rgb[i], (x[:3] - MEAN) / STD), boxes[i].tolist()
        assert torch.equal(mask[i], (x[3] - 0.0) / 1.0), boxes[i].tolist()
    print(f"template T=224: {n} renders equal to ATen's crop")


def _kernel_M(box, H, W, T):
    """The M the kernel writes, from its documented reading of the box (corner clamped to 0, crop clipped to the
    image, empty crops allowed), with the translation s * (-x1) + pad rounded once."""
    x1, y1, x2, y2 = box
    s = float(box_scale(box, T))
    cx, cy = min(max(x1, 0), W), min(max(y1, 0), H)
    rw, rh = int(np.floor(max(min(x2, W) - cx, 0) * s)), int(np.floor(max(min(y2, H) - cy, 0) * s))
    p = pads(rh, rw, T) or (0, 0, 0, 0)
    return torch.tensor([[s, 0, s * -x1 + p[0]], [0, s, s * -y1 + p[2]], [0, 0, 1]], dtype=torch.float64).float()


EDGE_BOXES = ((10, 10, 310, 11),        # 300 x 1: the resized crop has no rows (the reference raises in interpolate)
              (10, 10, 11, 310),        # no columns
              (650, 10, 700, 60),       # entirely right of the image
              (10, 490, 60, 540),       # entirely below it
              (700, 500, 900, 700),     # beyond the bottom-right corner
              (-100, 10, -40, 60),      # entirely left of it: a negative corner
              (-80, -60, -20, -10))     # above and left


def test_boxes_without_a_crop_give_zeros_and_M():
    """DESIGN.md row f3: where the reference raises (or would wrap a negative corner), the kernel writes zeros, a mask
    of zeros, the normalised zero on the fused path, and M.  (A run of a BOP test split refuses such boxes before they
    reach the kernel: `bop_run.image_inputs`, tests/test_crop_aten_cpu.py.)"""
    H, W, T = 480, 640, 224
    boxes = torch.tensor(EDGE_BOXES)
    n = len(EDGE_BOXES)
    want_M = torch.stack([_kernel_M(b, H, W, T) for b in EDGE_BOXES])
    for x1, y1, x2, y2 in EDGE_BOXES:
        assert geometry((x1, y1, x2, y2), H, W, T, clamp_origin=True)["empty"] or x2 <= 0 or y2 <= 0
    images = torch.rand(1, 2, H, W, device=DEV) + 1
    got = preprocess.crop_resize_pad(boxes.to(DEV), images, T, image_index=torch.zeros(n, device=DEV))
    assert not got["images"].any()
    assert torch.equal(got["M"].cpu(), want_M)
    rgb = torch.full((1, 3, H, W), 200, dtype=torch.uint8, device=DEV)
    got = preprocess.preprocess_queries(rgb, torch.ones(n, H, W, device=DEV), boxes.to(DEV), torch.zeros(n, device=DEV))
    assert not got["tar_mask"].any()
    assert torch.equal(got["tar_img"].cpu(), ((torch.zeros(n, 3, T, T) - MEAN) / STD))
    assert torch.equal(got["tar_M"].cpu(), want_M)


def test_target_sizes_below_128_are_refused():
    """Outputs of T + T <= 128 take ATen's small-output kernel in the second resize, which the kernel does not
    restate: both entry points refuse them."""
    with pytest.raises(Exception, match="target_size"):
        preprocess.crop_resize_pad(torch.tensor([[0, 0, 8, 8]], device=DEV), torch.zeros(1, 1, 16, 16, device=DEV), 127)
    c = _rle_encode(np.ones((16, 16), bool))
    with pytest.raises(Exception, match="target_size"):
        preprocess.crop_detections_rle(torch.zeros(1, 16, 16, 3, dtype=torch.uint8, device=DEV), c, [0, len(c)],
                                       [[0, 0, 16, 16]], [0], 127)
