"""`template_poses` against the reference's predefined template poses (tests/golden/template_poses.npz, copied from its
src/lib3d/predefined_poses by `python -m oracle.make_golden_template_poses`), for every level and both distributions.

Blender computed the reference's vertices in fp32, so the poses agree to a tolerance, not bit for bit.  The order is
the reference's wherever its elevations differ by more than the angular tolerance.  Where they differ by less (a ring
of views at one elevation, whose fp32 elevations differ by noise alone), the reference's sort followed that noise and
this one the fp64 elevation and then the azimuth: within such a ring the poses must be the same set, and the
generated ring must be in (elevation, azimuth) order."""
import os

import numpy as np
import pytest

from gigapose_b200 import template_poses as tp

MM = 1e-4           # translation tolerance, mm
RAD = 1e-7          # rotation and elevation tolerance, rad
COUNTS = {"all": {0: 42, 1: 162, 2: 642}, "upper": {0: 26, 1: 91, 2: 341}}


def _angle(A, B):
    """Largest entry of |A - B| for rotation stacks: for small differences each entry is an angle in rad.  (The
    geodesic angle reaches 1.07e-7 rad at level 2, on views near the poles, where `look_at`'s right vector magnifies
    the fp32 noise of the reference's camera direction.)"""
    return np.abs(A - B).max((-2, -1))


def _elevation(cam):
    p = cam[:, :3, 3]
    return np.arctan2(p[:, 2], np.hypot(p[:, 0], p[:, 1]))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "template_poses.npz")))


@pytest.mark.parametrize("distribution", tp.DISTRIBUTIONS)
@pytest.mark.parametrize("level", tp.LEVELS)
def test_template_poses_match_the_reference_files(golden, level, distribution):
    cam, obj = golden[f"cam_poses_level{level}"], golden[f"obj_poses_level{level}"]
    keep = cam[:, 2, 3] >= 0 if distribution == "upper" else np.ones(len(cam), bool)
    cam, obj = cam[keep], obj[keep]
    got = tp.template_poses(level, distribution, zoom=1.0)
    got_cam = tp.camera_poses(level)
    got_cam = got_cam[got_cam[:, 2, 3] >= 0] if distribution == "upper" else got_cam
    assert len(obj) == COUNTS[distribution][level]
    assert got.shape == obj.shape and got.dtype == np.float64
    assert np.array_equal(got[:, 3], np.tile([0.0, 0.0, 0.0, 1.0], (len(got), 1)))

    el = _elevation(cam)
    ring = np.concatenate([[0], np.cumsum(np.diff(el) > RAD)])
    got_el = _elevation(got_cam)
    got_az = np.arctan2(got_cam[:, 0, 3], got_cam[:, 1, 3])
    worst_t = worst_r = 0.0
    for r in np.unique(ring):
        ii = np.flatnonzero(ring == r)
        # within the ring: the generated views in (elevation, azimuth) order, each matching one reference view
        assert np.array_equal(np.lexsort((got_az[ii], got_el[ii])), np.arange(len(ii))), f"ring {r} out of order"
        ang = _angle(obj[ii][None, :, :3, :3], got[ii][:, None, :3, :3])
        match = ang.argmin(1)
        assert sorted(match) == list(range(len(ii))), f"ring {r} is not the reference's set of views"
        worst_r = max(worst_r, float(ang[np.arange(len(ii)), match].max()))
        worst_t = max(worst_t, float(np.abs(got[ii, :3, 3] - obj[ii][match, :3, 3]).max()))
        worst_t = max(worst_t, float(np.abs(got_cam[ii, :3, 3] - cam[ii][match, :3, 3]).max()))
        worst_r = max(worst_r, float(_angle(got_cam[ii, :3, :3], cam[ii][match, :3, :3]).max()))
    print(f"template_poses level {level} {distribution}: {len(got)} views, largest difference {worst_t:.2e} mm, "
          f"{worst_r:.2e} rad")
    assert worst_t < MM and worst_r < RAD


def test_the_test_templates_are_the_level_1_poses_zoomed_to_0_4(golden):
    want = golden["obj_poses_level1"].copy()
    want[:, :3, 3] *= 0.4
    got = tp.template_poses()
    assert got.shape == (162, 4, 4)
    assert np.abs(got[:, :3, 3] - want[:, :3, 3]).max() < 0.4 * MM
    assert np.allclose(got[:, :3, 3], [0.0, 0.0, 400.0], atol=0.4 * MM)


def test_object_pose_is_the_inverse_of_the_camera_pose():
    cam = tp.camera_poses(1)
    obj = tp.template_poses(1, zoom=1.0)
    assert np.abs(np.einsum("nij,njk->nik", obj, cam) - np.eye(4)).max() < 1e-12
    assert np.abs(np.einsum("nji,njk->nik", cam[:, :3, :3], cam[:, :3, :3]) - np.eye(3)).max() < 1e-12
    assert np.allclose(np.linalg.det(cam[:, :3, :3]), 1.0)


@pytest.mark.parametrize("level,distribution", [(3, "all"), (1, "lower"), (-1, "all")])
def test_unknown_level_or_distribution_is_refused(level, distribution):
    with pytest.raises(ValueError):
        tp.template_poses(level, distribution)
