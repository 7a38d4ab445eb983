"""Row f14 without a GPU: oracle/vis_port.py against the cv2 4.13 / PIL / scipy fixture (tests/golden/vis_reference.npz)
and against those libraries live where they import, the heat-map normalisation on hand-made values, the wrappers'
argument checks, and render_results' image selection and pairing on a synthetic BOP tree."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import add_port
from oracle import vis_port as P
import bop_tree

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vis_reference.npz")


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def test_port_gray_equals_fixture(z):
    for k in ("random", "extreme"):
        assert np.array_equal(P.gray(z[f"gray_in_{k}"]), z[f"gray_out_{k}"])


def test_port_warp_equals_fixture(z):
    for i, M in enumerate(z["warp_M"]):
        w = P.warp_affine(z["warp_src"], M[:2])
        assert hashlib.sha256(np.ascontiguousarray(w).tobytes()).hexdigest() == str(z["warp_sha256"][i]), i
        if i < len(z["warp_out"]):
            assert np.array_equal(w, z["warp_out"][i])


def test_port_paste_dilation_turbo_equal_fixture(z):
    assert np.array_equal(P.paste(z["paste_dst"], z["paste_rgb"], z["paste_alpha"]), z["paste_out"])
    assert np.array_equal(P.self_pasted(z["paste_alpha"]), z["paste_self"])
    assert np.array_equal(P.dilate2(z["dil_in"]), z["dil_2"])
    assert np.array_equal(P.dilate3(z["dil_in"]), z["dil_3"])
    assert tuple(z["turbo"][0]) == (48, 18, 59) and tuple(z["turbo"][255]) == (122, 4, 3)


def test_port_kabsch_equals_fixture(z):
    q, qm = P.crop_from_u8(z["kabsch_query_u8"], z["kabsch_query_mask_u8"])
    t, tm = P.crop_from_u8(z["kabsch_tmpl_u8"], z["kabsch_tmpl_mask_u8"])
    for i in range(len(q)):
        assert np.array_equal(P.kabsch_panel(q[i], qm[i], t[i], tm[i], z["kabsch_M"][i]), z["kabsch_out"][i]), i


def test_kernel_turbo_table_is_the_fixture(z):
    """The constant table compiled into csrc/vis.cu is cv2's turbo map in RGB order."""
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gigapose_b200", "csrc",
                            "vis.cu")).read()
    body = src[src.index("kTurbo[256 * 3] = {") + len("kTurbo[256 * 3] = {"):]
    body = body[:body.index("}")]
    table = np.array([int(v) for v in body.replace("\n", " ").split(",") if v.strip()], np.uint8).reshape(256, 3)
    assert np.array_equal(table, z["turbo"])


def test_port_equals_live_libraries():
    cv2 = pytest.importorskip("cv2")
    from PIL import Image
    from scipy.ndimage import binary_dilation
    rng = np.random.default_rng(3)
    allc = np.stack(np.meshgrid(np.arange(0, 256, 3), np.arange(256), np.arange(0, 256, 5), indexing="ij"),
                    -1).reshape(-1, 1, 3).astype(np.uint8)
    assert np.array_equal(P.gray(allc), cv2.cvtColor(allc, cv2.COLOR_RGB2GRAY))
    src = rng.integers(0, 256, (224, 224, 4), dtype=np.uint8)
    for _ in range(5):
        a, s = rng.uniform(-np.pi, np.pi), rng.uniform(0.3, 3)
        M = np.array([[s * np.cos(a), -s * np.sin(a), rng.uniform(-80, 80)],
                      [s * np.sin(a), s * np.cos(a), rng.uniform(-80, 80)]], np.float32)
        assert np.array_equal(P.warp_affine(src, M), cv2.warpAffine(src, M.astype(np.float64), (224, 224)))
    dst, rgb = rng.integers(0, 256, (30, 20, 3), dtype=np.uint8), rng.integers(0, 256, (30, 20, 3), dtype=np.uint8)
    alpha = rng.integers(0, 256, (30, 20), dtype=np.uint8)
    im = Image.fromarray(dst.copy())
    im.paste(Image.fromarray(rgb), (0, 0), Image.fromarray(alpha))
    assert np.array_equal(P.paste(dst, rgb, alpha), np.array(im))
    e = rng.random((25, 31)) < 0.1
    assert np.array_equal(P.dilate2(e), binary_dilation(e, np.ones((2, 2))))
    assert np.array_equal(P.dilate3(e), binary_dilation(e, np.ones((3, 3))))


def test_np_uint8_rule():
    x = np.array([-1.5, -0.5, 255.9, 256.7, 300, -300, 1e10, -1e10, np.nan], np.float32)
    with np.errstate(invalid="ignore"):
        assert np.array_equal(P.np_uint8(x), x.astype(np.uint8))


# ---------------------------------------------------------------------------------------------- heat-map normalisation
def test_heat_normalisation_non_symmetric_starts_at_smallest_value():
    turbo = np.arange(768).reshape(256, 3) % 256
    v = np.array([16.0, 28.0, 40.0], np.float32)
    col, idx = P.heat_colors(v, False, 64.0, turbo)
    # range [16, 64] (not [0, 64]): x = 0, 1/4, 1/2
    assert idx.tolist() == [0, 64, 128]
    assert np.array_equal(col[1], np.asarray(turbo[64], np.float32) / np.float32(255))
    _, idx = P.heat_colors(np.array([20.0, 200.0], np.float32), False, 100.0, turbo)
    assert idx.tolist() == [0, 255]                      # x = 1 -> 256 -> 255


def test_heat_normalisation_symmetric_starts_at_zero():
    turbo = np.zeros((256, 3))
    _, idx = P.heat_colors(np.array([16.0, 24.0, 40.0], np.float32), True, 64.0, turbo)
    assert idx.tolist() == [64, 96, 160]                  # range [0, 64]: floor(256 * v / 64)
    _, idx = P.heat_colors(np.zeros(4, np.float32), True, 100.0, turbo)
    assert idx.tolist() == [0, 0, 0, 0]
    _, idx = P.heat_colors(np.array([1.0, np.nan], np.float32), True, 100.0, turbo)
    assert idx.tolist() == [-1, -1]


# ---------------------------------------------------------------------------------------------- argument checks
def test_wrapper_validation():
    from gigapose_b200 import vis
    from gigapose_b200._lib import GigaPoseNativeError
    V = torch.zeros(4, 3)
    P4 = torch.zeros(1, 4, 4)
    with pytest.raises(GigaPoseNativeError, match="CUDA"):
        vis.vertex_errors([0], [0, 4], V, P4, P4, [False])
    with pytest.raises(GigaPoseNativeError, match="symmetric"):
        vis.vertex_errors([0], [0, 4], V, P4, P4, [False, True])
    with pytest.raises(GigaPoseNativeError, match="obj_idx"):
        vis.vertex_errors([1], [0, 4], V, P4, P4, [False])
    with pytest.raises(GigaPoseNativeError, match="max_distance"):
        vis.heat_colors(torch.zeros(4), [0, 4], [False], max_distance=0.0)
    with pytest.raises(GigaPoseNativeError, match="CUDA"):
        vis.heat_colors(torch.zeros(4), [0, 4], [False])
    with pytest.raises(GigaPoseNativeError, match="CUDA"):
        vis.overlay(torch.zeros(4, 4, 3, dtype=torch.uint8), None, None)
    with pytest.raises(GigaPoseNativeError, match="size"):
        vis.overlay(None, None, None)
    with pytest.raises(GigaPoseNativeError, match="CUDA"):
        vis.kabsch(*(torch.zeros(1, 3, 224, 224), torch.zeros(1, 224, 224)) * 2, torch.zeros(1, 3, 3))


def test_cli_parses():
    from gigapose_b200 import vis
    a = vis.parser().parse_args(["--results", "a.csv", "b_icp.csv", "--dataset-dir", "D", "--max-images", "3"])
    assert a.results == ["a.csv", "b_icp.csv"] and a.max_images == 3 and a.max_distance_mm == 100.0 and a.split == "test"


# ---------------------------------------------------------------------------------------------- selection and pairing
def synthetic_tree(root):
    """Two images; object 1 (a tetrahedron, not symmetric) with two instances in image (1, 0), object 2 (a spheroid,
    symmetric about z) once per image; ground truths at several distances."""
    models = {1: bop_tree.tetra(), 2: bop_tree.spheroid(n_lat=8, n_lon=16)}
    info = {1: dict(diameter=70.7), 2: dict(diameter=80.0, symmetries_continuous=[dict(axis=[0, 0, 1], offset=[0, 0, 0])])}
    K = np.array([[500.0, 0, 80], [0, 500.0, 60], [0, 0, 1]])
    png = np.zeros((120, 160), np.uint16)
    scenes = {1: {0: dict(gt=[(1, np.eye(3), [-30.0, 0.0, 600.0]), (2, bop_tree.rot([1, 0, 0], 30), [40.0, 10.0, 800.0]),
                              (1, bop_tree.rot([0, 1, 0], 40), [10.0, -30.0, 700.0])],
                          visib=[1.0, 1.0, 1.0], K=K, depth_scale=1.0, png=png),
                      3: dict(gt=[(2, np.eye(3), [0.0, 0.0, 500.0]), (1, np.eye(3), [0.0, 20.0, 900.0])],
                              visib=[1.0, 1.0], K=K, depth_scale=1.0, png=png)}}
    targets = [(1, 0, 1, 2), (1, 0, 2, 1), (1, 3, 2, 1)]
    bop_tree.write_tree(str(root), models, info, scenes, targets)
    from PIL import Image
    for im in (0, 3):
        d = os.path.join(str(root), "test", "000001", "rgb")
        os.makedirs(d, exist_ok=True)
        Image.fromarray(np.random.default_rng(im).integers(0, 256, (120, 160, 3), dtype=np.uint8)).save(
            os.path.join(d, f"{im:06d}.png"))
    return models, info, scenes


def _res(s, im, o, score, R, t):
    return dict(scene_id=s, im_id=im, obj_id=o, score=score, R=np.asarray(R, float).reshape(3, 3),
                t=np.asarray(t, float).reshape(3), time=1.0)


def synthetic_results(scenes):
    gt = scenes[1][0]["gt"]
    return [
        _res(1, 0, 1, 0.9, gt[2][1], np.add(gt[2][2], [2.0, 0, 0])),     # near instance 2 (gt index in file: 2)
        _res(1, 0, 1, 0.8, gt[0][1], np.add(gt[0][2], [0, 3.0, 0])),     # near instance 0
        _res(1, 0, 1, 0.1, np.eye(3), [0, 0, 650.0]),                    # third by score: dropped (inst_count 2)
        _res(1, 0, 2, 0.5, gt[1][1], gt[1][2]),
        _res(1, 0, 3, 0.5, np.eye(3), [0, 0, 500.0]),                    # not a target object
        _res(1, 3, 2, 0.7, np.eye(3), [0, 0, 510.0]),
    ]


def test_plan_selection_and_pairing(tmp_path):
    from gigapose_b200 import vis
    models, info, scenes = synthetic_tree(tmp_path)
    results = synthetic_results(scenes)
    p = vis.plan([results, results[:2]], str(tmp_path), max_images=None)
    assert [(i["scene_id"], i["im_id"]) for i in p["images"]] == [(1, 0), (1, 3)]
    im0 = p["images"][0]
    # ground truths far to near: |t| 800 (obj 2), 700, 600
    assert [round(float(np.linalg.norm(g["t"]))) for g in im0["gt"]] == [801, 701, 601]
    assert im0["est"][0] == [0, 1, 3] and im0["est"][1] == [0, 1]
    assert p["images"][1]["est"][0] == [5] and p["images"][1]["gt"][0]["obj_id"] == 2
    # pairing by the minimum ADD(-S) error, with errors from the fp32 port of gp_bop_add
    err = {}
    for e in im0["est"][0]:
        r = results[e]
        for k, g in enumerate(im0["gt"]):
            if g["obj_id"] == r["obj_id"]:
                add, adds, _ = add_port.add_errors(models[r["obj_id"]][0], vis._pose(r["R"], r["t"]),
                                                   vis._pose(g["R"], g["t"]), np.eye(3, dtype=np.float32))
                err[(e, k)] = adds if r["obj_id"] == 2 else add
    match = vis.pair_estimates(im0, results, im0["est"][0], err)
    assert match == {0: 1, 1: 2, 3: 0}
    assert len(vis.plan([results], str(tmp_path), max_images=1)["images"]) == 1


def test_result_lists_and_display_models(tmp_path):
    from gigapose_b200 import vis
    one = [dict(scene_id=1, im_id=0, obj_id=1, score=1.0, R=np.eye(3), t=np.zeros(3), time=1.0)]
    assert vis.result_lists(one) == [one]                          # one result list, not one csv per result
    assert vis.result_lists([one, one]) == [one, one]
    with pytest.raises(ValueError, match="no results"):
        vis.result_lists([])
    os.makedirs(tmp_path / "models_eval")
    assert vis.display_models_dir(str(tmp_path)) == str(tmp_path / "models_eval")
    os.makedirs(tmp_path / "models")
    assert vis.display_models_dir(str(tmp_path)) == str(tmp_path / "models")
    os.makedirs(tmp_path / "models_reconst")
    assert vis.display_models_dir(str(tmp_path)) == str(tmp_path / "models_reconst")
