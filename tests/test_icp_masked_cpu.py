"""Row f11 on the CPU: the masked-normal mode's restatement (tests/icp_masked_port.py) against the frame-smoothed port,
the box restriction against the full-frame definition, the run-length boxes, and the accuracy the mode is for, on a
noisy, occluded scene rendered with oracle/bop_port.render_depth."""
import numpy as np
import pytest

import icp_masked_port as mp
from gigapose_b200 import icp
from oracle import bop_port, bop_run_port, icp_port

K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]], np.float32)


def _depth(H, W, seed):
    rng = np.random.default_rng(seed)
    d = (700 + 40 * np.sin(np.arange(W) / 7.0)[None] + 30 * np.cos(np.arange(H) / 5.0)[:, None]
         + rng.normal(0, 2, (H, W))).astype(np.float32)
    d[rng.random((H, W)) < 0.1] = 0
    return d


def test_all_ones_mask_is_the_frame_map_bit_for_bit():
    d = _depth(40, 52, 0)
    ones = np.ones(d.shape, bool)
    assert np.array_equal(mp.scene_masked(d, ones, K), icp_port.scene(d, K))
    box, m = mp.scene_masked_box(d, ones, K)
    assert box == (0, 0, 52, 40) and np.array_equal(m, icp_port.scene(d, K))


def _masks(H, W, rng):
    out = []
    m = np.zeros((H, W), bool); m[5:20, 8:30] = True; m[10:14, 15:22] = False; out.append(m)    # a hole
    for sl in [(slice(0, 6), slice(10, 20)), (slice(H - 4, H), slice(3, 30)), (slice(8, 30), slice(0, 3)),
               (slice(2, 25), slice(W - 1, W)), (slice(0, H), slice(0, 2))]:                 # each border
        m = np.zeros((H, W), bool); m[sl] = True; out.append(m)
    for y, x in [(0, 0), (H - 1, W - 1), (H // 2, W // 2), (0, W - 1), (1, 1)]:                       # one pixel
        m = np.zeros((H, W), bool); m[y, x] = True; out.append(m)
    out.append(rng.random((H, W)) < 0.3)                                                        # scattered
    return out


@pytest.mark.parametrize("shape", [(17, 17), (40, 52), (33, 19)])
def test_box_restriction_equals_the_full_frame_map_inside_the_box(shape):
    H, W = shape
    rng = np.random.default_rng(H * W)
    d = _depth(H, W, H)
    for m in _masks(H, W, rng):
        full = mp.scene_masked(d, m, K)
        garbage = rng.normal(0, 1e4, d.shape).astype(np.float32)
        (x0, y0, x1, y1), box_map = mp.scene_masked_box(d, m, K)
        outside = np.ones(d.shape, bool); outside[y0:y1, x0:x1] = False
        _, box_map_g = mp.scene_masked_box(np.where(outside, garbage, d), m, K)
        assert np.array_equal(box_map, full[y0:y1, x0:x1]), (shape, (x0, y0, x1, y1))
        assert np.array_equal(box_map_g, box_map)


def test_rle_boxes_match_the_decoded_masks():
    rng = np.random.default_rng(3)
    H, W = 23, 31
    masks = _masks(H, W, rng) + [np.zeros((H, W), bool)]
    m = np.zeros((H, W), bool); m[H - 2:, 4] = True; m[:3, 5] = True; masks.append(m)     # one run over two columns
    counts = [bop_run_port.binary_mask_to_rle(m)["counts"] for m in masks]
    off = np.concatenate([[0], np.cumsum([len(c) for c in counts])])
    got = icp.rle_boxes(np.concatenate(counts), off, H, W)
    for b, m, c in zip(got, masks, counts):
        assert np.array_equal(bop_run_port.rle_to_binary_mask(dict(size=[H, W], counts=c)), m)
        assert tuple(b) == mp.mask_box(m)


def _plane(z, Km, H, W):
    v = np.array([[-2e3, -2e3, z], [2e3, -2e3, z], [2e3, 2e3, z], [-2e3, 2e3, z]], np.float32)
    return bop_port.render_depth(v, np.array([[0, 1, 2], [0, 2, 3]], np.int32), np.eye(4, dtype=np.float32), Km, H, W,
                                 100.0)["depth"]


def occluded_scene_cpu():
    """noisy_occluded_scene's recipe on the CPU (one sample per pixel, numpy noise), with test_gpu_icp's start pose
    T0 and the render of the ellipsoid at T0 -> (depth, mask, T0, render, render box)."""
    from icp_scenes import T_ELL, ellipsoid, perturb
    H, W = 480, 640
    mesh = ellipsoid()
    obj = bop_port.render_depth(mesh["vertices"], mesh["faces"], T_ELL, K, H, W, 100.0)["depth"]
    mask = obj > 0
    d = np.where(mask, obj, _plane(float(T_ELL[2, 3]) + 150.0, K, H, W)).astype(np.float32)
    rng = np.random.default_rng(3)
    d = (d + rng.normal(size=d.shape)).astype(np.float32)
    d[rng.random(d.shape) < 0.1] = 0
    ys, xs = np.nonzero(mask)
    x_cut = int(np.sort(xs)[int(0.3 * len(xs))])
    d[ys.min():ys.max() + 1, xs.min():x_cut] = float(T_ELL[2, 3]) - 120.0
    mask[ys.min():ys.max() + 1, xs.min():x_cut] = False
    T0 = perturb(T_ELL, [0.2, 1, 0.4], 8.0, [9.0, -8.0, 9.0])
    r = bop_port.render_depth(mesh["vertices"], mesh["faces"], T0, K, H, W, 100.0)
    return d, mask, T0, r["depth"], r["box"]


def test_masked_mode_reaches_the_aim_on_the_noisy_occluded_scene():
    """On occluded_scene_cpu the frame-smoothed port stays above 2 mm / 1 degree, the masked mode gets below."""
    from icp_scenes import T_ELL
    d, mask, T0, R, box = occluded_scene_cpu()

    def err(T):
        dR = T[:3, :3].astype(np.float64) @ T_ELL[:3, :3].astype(np.float64).T
        return (float(np.linalg.norm(T[:3, 3].astype(np.float64) - T_ELL[:3, 3])),
                float(np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))))
    frame = icp_port.refine(icp_port.scene(d, K), R, box, K, T0, mask=mask)
    masked = mp.refine_masked(d, mask, R, box, K, T0)
    ef, em = err(frame[0]), err(masked[0])
    print(f"frame-smoothed {ef[0]:.2f} mm {ef[1]:.2f} deg, masked {em[0]:.2f} mm {em[1]:.2f} deg")
    assert masked[1] == icp_port.OK and em[0] <= 2.0 and em[1] <= 1.0
    assert ef[0] > em[0] and ef[1] > em[1]


def test_bop_run_selects_the_kept_masks_and_parses_the_flag():
    from gigapose_b200 import bop_run
    counts = np.array([5, 2, 3, 1, 0, 4, 6, 7, 8], np.int32)
    off = np.array([0, 3, 6, 9])
    c, o = bop_run.select_rle((counts, off), [2, 0])
    assert c.tolist() == [6, 7, 8, 5, 2, 3] and o.tolist() == [0, 3, 6]
    c, o = bop_run.select_rle((counts, off), [])
    assert len(c) == 0 and o.tolist() == [0]
    a = bop_run.parser().parse_args(["--dataset-dir", "d", "--checkpoint", "c", "--template-poses", "p",
                                     "--refine-depth", "2", "--refine-masks"])
    assert a.refine_masks and a.refine_depth == 2
    with pytest.raises(SystemExit):
        bop_run.main(["--dataset-dir", "d", "--checkpoint", "c", "--template-poses", "p", "--refine-masks"])
