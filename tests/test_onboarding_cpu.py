"""Row f16 on the CPU: the re-centring geometry of `onboarding.recentre` against independent fp64 constructions, the
view selection against a brute force, the onboarding_static reader on a synthetic tree with every refusal naming its
file or scene, and the runner's refusal of depth refinement in model-free runs."""
import json
import os

import numpy as np
import pytest

from gigapose_b200 import bop_run, onboarding
from gigapose_b200.onboarding import OnboardingError
from gigapose_b200.render import TEMPLATE_K


def _rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _pose(rng, max_off_deg=25.0, dist=(300.0, 900.0)):
    """Object -> camera pose whose origin is seen up to max_off_deg off the optical axis."""
    off, az = np.radians(rng.uniform(0, max_off_deg)), rng.uniform(0, 2 * np.pi)
    d = np.array([np.sin(off) * np.cos(az), np.sin(off) * np.sin(az), np.cos(off)])
    P = np.eye(4)
    P[:3, :3] = _rotation(rng)
    P[:3, 3] = d * rng.uniform(*dist)
    return P


def _K(rng):
    return np.array([[rng.uniform(500, 1600), 0, rng.uniform(300, 980)], [0, rng.uniform(500, 1600), rng.uniform(220, 560)],
                     [0, 0, 1.0]])


def _look_at_rotation(t):
    """Independent construction of a rotation taking t / |t| to +z: the axis-angle form with an explicit angle."""
    d = t / np.linalg.norm(t)
    axis = np.cross(d, [0.0, 0.0, 1.0])
    s = np.linalg.norm(axis)
    if s == 0:
        return np.eye(3)
    k = axis / s
    ang = np.arctan2(s, d[2])
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx


def test_recentre_rotation_is_proper_minimal_and_looks_at_the_origin():
    rng = np.random.default_rng(0)
    Kt = np.asarray(TEMPLATE_K)
    for _ in range(200):
        K, P = _K(rng), _pose(rng)
        Rv, V, Hinv = onboarding.recentre(K, P)
        np.testing.assert_allclose(Rv @ Rv.T, np.eye(3), atol=1e-14)
        assert abs(np.linalg.det(Rv) - 1) < 1e-14
        np.testing.assert_allclose(Rv, _look_at_rotation(P[:3, 3]), atol=1e-14)
        # the rotation axis is perpendicular to both the ray and the optical axis: minimal rotation
        t = P[:3, 3]
        np.testing.assert_allclose(Rv @ np.cross(t, [0, 0, 1.0]), np.cross(t, [0, 0, 1.0]), atol=1e-12)
        np.testing.assert_allclose(V[:3, :3], Rv @ P[:3, :3], atol=1e-14)
        np.testing.assert_allclose(V[:3, 3], [0, 0, np.linalg.norm(t)], rtol=1e-15)
        # the virtual pose projects the object origin to the template principal point
        p = Kt @ V[:3, 3]
        np.testing.assert_allclose(p[:2] / p[2], Kt[:2, 2], atol=1e-12)
        # the pose's rotation differs from the frame's by R_v: the camera direction in the object frame is unchanged
        np.testing.assert_allclose(onboarding.view_directions(V[None]), onboarding.view_directions(P[None]), atol=1e-14)


def test_recentre_is_the_identity_on_the_axis():
    rng = np.random.default_rng(1)
    for _ in range(20):
        P = _pose(rng)
        P[:3, 3] = [0.0, 0.0, rng.uniform(100, 1000)]
        Rv, V, Hinv = onboarding.recentre(_K(rng), P)
        assert np.array_equal(Rv, np.eye(3))
        assert np.array_equal(V[:3, :3], P[:3, :3]) and np.array_equal(V[:3, 3], P[:3, 3])
    _, _, Hinv = onboarding.recentre(TEMPLATE_K, P)
    np.testing.assert_allclose(Hinv, np.eye(3), atol=1e-12)          # K_f K_t^-1 rounds: sources land near, not on, integers


def test_homography_maps_frame_projections_to_virtual_projections():
    """H^-1 sends the virtual projection of a 3-D point to its frame projection, within 1e-9 px, for points spread
    over the whole view; both projections are computed here from the poses alone."""
    rng = np.random.default_rng(2)
    Kt = np.asarray(TEMPLATE_K)
    worst = 0.0
    for _ in range(100):
        K, P = _K(rng), _pose(rng)
        _, V, Hinv = onboarding.recentre(K, P)
        X = rng.uniform(-150, 150, size=(50, 3))                 # object points
        cf = X @ P[:3, :3].T + P[:3, 3]
        cv = X @ V[:3, :3].T + V[:3, 3]
        pf = cf @ K.T
        pf = pf[:, :2] / pf[:, 2:]
        pv = cv @ Kt.T
        pv = pv[:, :2] / pv[:, 2:]
        s = np.c_[pv, np.ones(len(pv))] @ Hinv.T
        back = s[:, :2] / s[:, 2:]
        worst = max(worst, float(np.abs(back - pf).max()))
        H = np.linalg.inv(Hinv)
        s = np.c_[pf, np.ones(len(pf))] @ H.T
        worst = max(worst, float(np.abs(s[:, :2] / s[:, 2:] - pv).max()))
    assert worst < 1e-9, worst


def test_recentre_refuses_objects_behind_the_camera():
    P = np.eye(4)
    for tz in (0.0, -5.0):
        P[:3, 3] = [10.0, 0.0, tz]
        with pytest.raises(OnboardingError, match="t_z"):
            onboarding.recentre(TEMPLATE_K, P)


def _brute(frame_poses, template_poses, valid):
    def direction(P):
        c = -P[:3, :3].T @ P[:3, 3]
        return c / np.linalg.norm(c)
    ids, gaps = [], []
    for tp in template_poses:
        best, arg = -2.0, -1
        for i, fp in enumerate(frame_poses):
            if not valid[i]:
                continue
            c = float(np.dot(direction(tp), direction(fp)))
            if c > best:                                           # strict: the first of equal cosines stays
                best, arg = c, i
        ids.append(arg)
        gaps.append(np.degrees(np.arccos(min(1.0, max(-1.0, best)))))
    return np.array(ids), np.array(gaps)


def test_select_views_equals_a_brute_force_with_planted_ties():
    from gigapose_b200.template_poses import template_poses
    rng = np.random.default_rng(3)
    tpl = template_poses(1, "all")
    frames = np.stack([_pose(rng, 25.0) for _ in range(60)])
    frames[10] = frames[4]                                     # exact duplicates: the lower index must win
    frames[30] = frames[4]
    frames[20] = tpl[7]                                        # exactly on a template view
    frames[25] = tpl[7]
    valid = np.ones(60, bool)
    valid[[5, 6, 40]] = False
    for v in (None, valid):
        ids, gaps = onboarding.select_views(frames, tpl, v)
        want_ids, want_gaps = _brute(frames, tpl, np.ones(60, bool) if v is None else v)
        assert np.array_equal(ids, want_ids)
        np.testing.assert_allclose(gaps, want_gaps, atol=1e-9)
        assert not np.isin(ids, [10, 30, 25]).any()
        assert ids[7] == 20 and gaps[7] < 1e-5
    assert not np.isin(onboarding.select_views(frames, tpl, valid)[0], [5, 6, 40]).any()
    with pytest.raises(OnboardingError, match="non-empty"):
        onboarding.select_views(frames, tpl, np.zeros(60, bool))


# ---------------------------------------------------------------------------------------------------- the reader
def _write_scene(root, name, obj, n=3, H=24, W=32, objects=None, skip_mask=None, skip_rgb=None):
    from PIL import Image
    d = os.path.join(root, "onboarding_static", name)
    os.makedirs(os.path.join(d, "rgb"))
    os.makedirs(os.path.join(d, "mask_visib"))
    gt, cam = {}, {}
    for im in range(n):
        P = np.eye(4)
        P[:3, 3] = [im, 0, 500.0]
        ids = objects if objects is not None and im == n - 1 else [obj]
        gt[str(im)] = [dict(obj_id=o, cam_R_m2c=P[:3, :3].reshape(-1).tolist(), cam_t_m2c=P[:3, 3].tolist()) for o in ids]
        cam[str(im)] = dict(cam_K=np.asarray(TEMPLATE_K).reshape(-1).tolist(), depth_scale=1.0)
        if im != skip_rgb:
            Image.fromarray(np.full((H, W, 3), 10 * im, np.uint8)).save(os.path.join(d, "rgb", f"{im:06d}.jpg"))
        if im != skip_mask:
            m = np.zeros((H, W), np.uint8)
            m[4:12, 5:20] = 255
            Image.fromarray(m).save(os.path.join(d, "mask_visib", f"{im:06d}_000000.png"))
    for fname, obj_ in (("scene_gt.json", gt), ("scene_camera.json", cam)):
        with open(os.path.join(d, fname), "w") as f:
            json.dump(obj_, f)
    return d


def _tree(root, objs=(1, 2)):
    for o in objs:
        _write_scene(root, f"obj_{o:06d}_up", o, n=3)
        _write_scene(root, f"obj_{o:06d}_down", o, n=2)


def test_reader_groups_up_and_down_scenes_by_object(tmp_path):
    root = str(tmp_path)
    _tree(root)
    frames = onboarding.read_onboarding_static(root)
    assert sorted(frames) == [1, 2]
    for o, fr in frames.items():
        assert len(fr) == 5
        assert [os.path.basename(os.path.dirname(os.path.dirname(p))) for p in fr.images] == \
            [f"obj_{o:06d}_down"] * 2 + [f"obj_{o:06d}_up"] * 3
        assert fr.K.shape == (5, 3, 3) and fr.poses.shape == (5, 4, 4)
        rgb, m = fr.load(0)
        assert rgb.shape == (24, 32, 3) and m.dtype == np.uint8 and m.sum() == 8 * 15
        assert fr.boxes[0].tolist() == [5, 4, 20, 12]


def test_reader_refusals_name_the_file_or_scene(tmp_path):
    cases = {
        "two_objects": (lambda r: (_tree(r, (1,)), _write_scene(r, "obj_000002_up", 2, objects=[2, 3])), "obj_000002_up"),
        "no_mask": (lambda r: (_tree(r, (1,)), _write_scene(r, "obj_000002_up", 2, skip_mask=1)),
                    "obj_000002_up/mask_visib/000001_000000.png"),
        "no_rgb": (lambda r: (_tree(r, (1,)), _write_scene(r, "obj_000002_up", 2, skip_rgb=2)),
                   "obj_000002_up/rgb/000002.jpg"),
        "ids": (lambda r: _tree(r, (1, 3)), r"\[1, 3\]"),
    }
    for name, (make, word) in cases.items():
        root = str(tmp_path / name)
        make(root)
        with pytest.raises(OnboardingError, match=word):
            onboarding.read_onboarding_static(root)
    root = str(tmp_path / "info")
    _tree(root)
    os.makedirs(os.path.join(root, "models"))
    with open(os.path.join(root, "models", "models_info.json"), "w") as f:
        json.dump({"1": {}, "2": {}, "3": {}}, f)
    with pytest.raises(OnboardingError, match="models_info.json"):
        onboarding.read_onboarding_static(root)
    with pytest.raises(OnboardingError, match="onboarding_static"):
        onboarding.read_onboarding_static(str(tmp_path / "nothing"))


def test_select_frames_skips_frames_with_empty_masks(tmp_path):
    """A frame that wins a view but has an empty mask leaves the candidates; only winning frames' masks are read."""
    rng = np.random.default_rng(4)
    poses = np.stack([_pose(rng) for _ in range(8)])
    masks = [np.ones((4, 4), np.uint8) for _ in range(8)]
    tpl = poses[[2, 5]].copy()
    masks[2][:] = 0
    fr = onboarding.Frames([np.zeros((4, 4, 3), np.uint8)] * 8, masks, np.stack([np.eye(3)] * 8), poses)
    ids, _ = onboarding.select_frames(fr, tpl)
    want, _ = _brute(poses, tpl, np.arange(8) != 2)
    assert np.array_equal(ids, want) and ids[1] == 5 and ids[0] != 2
    assert set(fr.boxes) <= {2} | set(ids.tolist())


def test_static_onboarding_refuses_depth_refinement(capsys):
    with pytest.raises(SystemExit):
        bop_run.main(["--dataset-dir", "x", "--checkpoint", "y", "--onboarding", "static", "--refine-depth", "1"])
    assert "depth refiners render the CAD model" in capsys.readouterr().err
    with pytest.raises(bop_run.BopRunError, match="refine-depth"):
        bop_run.check_onboarding("static", 1)
    with pytest.raises(bop_run.BopRunError, match="onboarding"):
        bop_run.check_onboarding("mesh", 0)
    assert bop_run.default_run_id("static") == "bop_run_static" and bop_run.default_run_id() == "bop_run"
