"""Row f3's CPU restatement `oracle.port.crop_resize_pad` against the reference's crop in plain ATen
(`tests/crop_aten.py`) over the whole crop sweep, bit for bit, with proof that the sweep reaches every branch of ATen's
nearest-index arithmetic and tells apart every one-rule-wrong variant of the crop."""
import collections

import numpy as np

import pytest
import torch

from crop_aten import (ALL_BRANCHES, IMAGES, MUTATIONS, branches, coordinate_image, crop_aten, geometry, pads,
                       sweep)
from oracle import port

TARGETS = (224, 160, 128)
# fewest boxes of the sweep (all target sizes together) that must reach each branch
MIN_PER_BRANCH = 40


@pytest.fixture(scope="module")
def images():
    return {hw: coordinate_image(4, *hw) for hw in IMAGES}


def test_sweep_reaches_every_branch():
    count = collections.Counter()
    for T in TARGETS:
        for H, W, box, clamp in sweep(T):
            count.update(branches(geometry(box, H, W, T, clamp_origin=clamp)))
    print("boxes per branch:", {b: count[b] for b in ALL_BRANCHES})
    thin = [b for b in ALL_BRANCHES if count[b] < MIN_PER_BRANCH]
    assert not thin, f"branches reached by fewer than {MIN_PER_BRANCH} boxes: {thin}"
    assert count["empty"] == 0


@pytest.mark.parametrize("T", TARGETS)
def test_port_equals_aten_over_the_sweep(T, images):
    """Every box of the sweep inside the port's domain (a non-negative top-left corner), with 1 to 4 channels: the
    crop of a coordinate image is each output pixel's source index, so equal crops are equal index maps."""
    n = 0
    for i, (H, W, box, clamp) in enumerate(sweep(T)):
        if clamp:
            continue
        img = images[(H, W)][: 1 + i % 4]
        want, want_M = crop_aten(box, img, T)
        got = port.crop_resize_pad(torch.tensor([box]), img[None], target_size=T)
        assert torch.equal(got["images"][0], want), f"T={T} image {H}x{W} box {box}: {geometry(box, H, W, T)}"
        assert torch.equal(got["M"][0], want_M), f"T={T} box {box}: M {got['M'][0].tolist()} != {want_M.tolist()}"
        n += 1
    print(f"T={T}: port == ATen on {n} boxes")
    assert n > 1500


def _differs(a, b):
    return a[0].shape != b[0].shape or not torch.equal(a[0], b[0]) or not torch.equal(a[1], b[1])


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_sweep_tells_every_mutation_apart(mutation, images):
    for T in TARGETS:
        for H, W, box, clamp in sweep(T):
            img = images[(H, W)][:1]
            if _differs(crop_aten(box, img, T, clamp_origin=clamp),
                        crop_aten(box, img, T, mutation=mutation, clamp_origin=clamp)):
                print(f"{mutation}: first differing box T={T} image {H}x{W} box {box}")
                return
    pytest.fail(f"no box of the sweep tells `{mutation}` from the reference's crop")


def test_geometry_agrees_with_aten_shapes(images):
    """`geometry`'s resized size and padding are those of the ATen calls (checked through the unpadded crop)."""
    import torch.nn.functional as F
    for T in TARGETS:
        for H, W, box, clamp in sweep(T)[::7]:
            g = geometry(box, H, W, T, clamp_origin=clamp)
            x1, y1 = (max(box[0], 0), max(box[1], 0)) if clamp else box[:2]
            r = F.interpolate(images[(H, W)][None, :1, y1:box[3], x1:box[2]], scale_factor=g["scale"])
            assert tuple(r.shape[-2:]) == (g["rh"], g["rw"]), (T, H, W, box)
            assert g["pads"] == pads(g["rh"], g["rw"], T)


def test_the_reference_raises_where_the_crop_is_empty(images):
    """The contract edges of row f3 (DESIGN.md): the reference has no crop for them; the kernel writes zeros."""
    img = images[(480, 640)][:1]
    for box in ((10, 10, 310, 11),          # 300 x 1: the resized crop has no rows at T = 224
                (10, 10, 11, 310),          # no columns
                (650, 10, 700, 60),         # entirely right of the image
                (10, 490, 60, 540)):        # entirely below it
        assert geometry(box, 480, 640, 224)["empty"]
        with pytest.raises((RuntimeError, ValueError, ZeroDivisionError)):
            crop_aten(box, img, 224)


def test_a_negative_corner_wraps_in_the_reference():
    """Python slicing reads a negative corner from the far edge: the reference's crop of (-5, 0, 45, 50) is empty
    (columns 635 to 45) and that of (-5, 0, 700, 50) keeps the last 5 columns; the kernel clamps the corner to 0."""
    assert geometry((-5, 0, 45, 50), 480, 640, 224)["empty"]
    g = geometry((-5, 0, 45, 50), 480, 640, 224, clamp_origin=True)
    assert (g["ch"], g["cw"]) == (50, 45)
    g = geometry((-5, 0, 700, 50), 480, 640, 224)
    assert (g["ch"], g["cw"]) == (50, 5)
    g = geometry((-5, 0, 700, 50), 480, 640, 224, clamp_origin=True)
    assert (g["ch"], g["cw"]) == (50, 640)


def test_empty_crops_finds_exactly_the_boxes_without_a_resized_crop():
    """`preprocess.empty_crops` (the host check that keeps such boxes from the kernel) against ATen's scale and the
    clamped slice of `geometry`: no sweep box is empty, and on random boxes, many of them thin or outside the image,
    it names exactly those with no rows or columns once resized."""
    from gigapose_b200.preprocess import empty_crops
    for T in TARGETS:
        for (H, W) in IMAGES:
            boxes = [box for h, w, box, _ in sweep(T) if (h, w) == (H, W)]
            assert len(empty_crops(boxes, H, W, T)) == 0
    g = torch.Generator().manual_seed(11)
    H, W, n = 480, 640, 4000
    x1 = torch.randint(-200, W + 50, (n,), generator=g)
    y1 = torch.randint(-200, H + 50, (n,), generator=g)
    long, short = torch.randint(1, 900, (n,), generator=g), torch.randint(1, 6, (n,), generator=g)
    wide = torch.rand(n, generator=g) < 0.5
    boxes = torch.stack([x1, y1, x1 + torch.where(wide, long, short), y1 + torch.where(wide, short, long)], 1).tolist()
    for T in TARGETS:
        want = [i for i, b in enumerate(boxes) if geometry(b, H, W, T, clamp_origin=True)["empty"]]
        assert empty_crops(boxes, H, W, T).tolist() == want
        assert 200 < len(want) < n - 200
    assert empty_crops([[5, 5, 5, 9], [5, 5, 9, 5], [9, 9, 5, 5]], H, W).tolist() == [0, 1, 2]


def test_a_bop_run_refuses_a_detection_that_cannot_be_cropped():
    """A CNOS mask one row high and more than 224 px long has no rows once resized: the reference's F.interpolate
    raises, and the kernel would crop it to zeros.  `bop_run.image_inputs` refuses it, naming the image and the
    detection; one 224 px long still has one row and is kept."""
    from gigapose_b200 import bop_run
    from oracle.bop_run_port import binary_mask_to_rle

    def det(x, y, w, h):
        m = np.zeros((480, 640), bool)
        m[y:y + h, x:x + w] = True
        return dict(category_id=1, bbox=[x, y, w, h], score=0.9, time=0.1,
                    segmentation=dict(size=[480, 640], counts=binary_mask_to_rle(m)["counts"]))

    ok = [det(10, 20, 30, 40), det(100, 40, 224, 1), det(300, 10, 1, 224)]
    x = bop_run.image_inputs(ok, [], "ycbv", (480, 640), "000048_000001")
    assert x["boxes"].tolist() == [[10, 20, 40, 60], [100, 40, 324, 41], [300, 10, 301, 234]]
    for thin in (det(100, 40, 225, 1), det(300, 10, 1, 300)):
        with pytest.raises(bop_run.BopRunError, match=r"image 000048_000001, detection 1: .*no rows or columns"):
            bop_run.image_inputs([ok[0], thin], [], "ycbv", (480, 640), "000048_000001")
