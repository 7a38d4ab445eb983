"""Row f9 on the CPU: the detection selection against the reference's loaders (tests/golden/bop_run_selection.json,
oracle/make_golden_bop_run.py), the RLE readers against the numpy restatement of the toolkit's decoder
(oracle/bop_run_port.py), the dataset layout and image readers, and the checkpoint loader."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

from gigapose_b200 import bop_run
from gigapose_b200.bop_run import BopRunError
from oracle.bop_run_port import binary_mask_to_rle, rle_to_binary_mask, rle_to_string

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bop_run_selection.json")


def _cases():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", range(5))
def test_selection_equals_the_reference_loaders(case):
    c = _cases()[case]
    test_list, selected = bop_run.select_detections(c["detections"], c["dataset"], c["setting"], c["targets"])
    assert list(selected) == list(c["expect"])          # images, in the reference's order
    assert sorted(test_list) == sorted(selected)
    for key, exp in c["expect"].items():
        dets = selected[key]
        assert [d["det_idx"] for d in dets] == exp["det_idx"]
        assert [d["category_id"] for d in dets] == exp["label"]
        assert [d["score"] for d in dets] == exp["score"]
        xyxy = bop_run.xywh_to_xyxy([d["bbox"] for d in dets])
        assert xyxy.dtype == np.int64 and xyxy.tolist() == exp["xyxy"]
        assert [[t["obj_id"], t["inst_count"]] for t in test_list[key]] == exp["targets"]
        assert dets[0]["time"] == exp["time"]


def test_golden_covers_the_selection_cases():
    cases = _cases()
    assert {(c["dataset"], c["setting"]) for c in cases} >= {("lmo", "localization"), ("icbin", "localization"),
                                                             ("lmo", "detection")}
    loc = [c for c in cases if c["setting"] == "localization"]
    fallback = ties = over16 = over32 = fractional = False
    for c in loc:
        by = {}
        for d in c["detections"]:
            by.setdefault((d["scene_id"], d["image_id"], d["category_id"]), []).append(d)
            fractional |= any(v != int(v) for v in d["bbox"])
        for t in c["targets"]:
            got = by.get((t["scene_id"], t["im_id"], t["obj_id"]), [])
            fallback |= not got
            scores = [d["score"] for d in got]
            ties |= len(set(scores)) < len(scores)
            over16 |= len(got) > 16
            over32 |= len(got) > 32
    assert fallback and ties and over16 and over32 and fractional


def test_localization_refuses_a_target_image_without_detections():
    c = _cases()[0]
    targets = c["targets"] + [dict(scene_id=77, im_id=3, obj_id=1, inst_count=1)]
    with pytest.raises(BopRunError, match="000077_000003"):
        bop_run.select_detections(c["detections"], c["dataset"], "localization", targets)


def test_image_inputs_remap_lmo_and_concatenate_the_runs():
    dets = [dict(category_id=5, bbox=[1.5, 2.25, 10.0, 20.5], time=0.25,
                 segmentation=dict(size=[4, 3], counts=[2, 3, 7])),
            dict(category_id=12, bbox=[0, 0, 3, 4], time=0.5, segmentation=dict(size=[4, 3], counts=rle_to_string([0, 12])))]
    x = bop_run.image_inputs(dets, [dict(obj_id=5, inst_count=1), dict(obj_id=12, inst_count=1)], "lmo", (4, 3), "k")
    assert x["labels"].tolist() == [2, 8] and x["obj_id"] == [2, 8]
    assert x["boxes"].tolist() == [[1, 2, 11, 22], [0, 0, 3, 4]]
    assert x["counts"].tolist() == [2, 3, 7, 0, 12] and x["offsets"].tolist() == [0, 3, 5]
    assert x["detection_time"] == 0.25


# ---------------------------------------------------------------------------------------------------- RLE
def kernel_rule(counts, H, W):
    """The mask gp_crop_resize_pad_rle reads: pixel (row, col) is 1 when upper_bound(running sums, col * H + row) is
    odd and lies before the last run."""
    ends = np.cumsum(np.asarray(counts, np.int64))
    p = np.arange(H * W).reshape(W, H).T
    k = np.searchsorted(ends, p, side="right")
    return (k < len(ends)) & (k % 2 == 1)


def _edge_cases(H, W):
    n = H * W
    cases = [[n], [0, n], [], [0, 3, 2, n - 5], [H - 1, 2, H - 2, 5, n - 2 * H - 4],
             [3, n], [1, 2, n], [H + 3, 2 * H + 1, n], [0, 1, 1, 1, 1]]
    return [c for c in cases if min(c, default=0) >= 0]


@pytest.mark.parametrize("H,W", [(5, 7), (16, 9), (1, 30)])
def test_rle_decode_equals_the_port(H, W):
    rng = np.random.default_rng(H * 100 + W)
    masks = [rng.random((H, W)) < q for q in (0.0, 1.0, 0.1, 0.5, 0.9)]
    for m in masks:
        rle = binary_mask_to_rle(m)
        np.testing.assert_array_equal(rle_to_binary_mask(rle), m)
    cases = [binary_mask_to_rle(m)["counts"] for m in masks] + _edge_cases(H, W)
    for counts in cases:
        want = rle_to_binary_mask(dict(size=[H, W], counts=counts))
        np.testing.assert_array_equal(kernel_rule(counts, H, W), want, err_msg=str(counts))
        for form in (counts, rle_to_string(counts)):
            got = bop_run.rle_counts(dict(size=[H, W], counts=form), (H, W), "d")
            assert got.dtype == np.int32 and got.tolist() == list(counts)


def test_compressed_rle_round_trips_large_and_negative_differences():
    rng = np.random.default_rng(3)
    counts = rng.integers(0, 1 << 20, size=500).tolist() + [0, 5, 0, 1 << 30, 1]
    assert bop_run.rle_from_string(rle_to_string(counts)) == counts


def test_malformed_rle_is_refused_with_a_message():
    seg = lambda c, size=(4, 3): dict(size=list(size), counts=c)
    with pytest.raises(BopRunError, match="negative run length"):
        bop_run.rle_counts(seg([2, -1, 11]), (4, 3), "image 000001_000002, detection 3")
    with pytest.raises(BopRunError, match="differs from the image"):
        bop_run.rle_counts(seg([12], (3, 4)), (4, 3), "d")
    with pytest.raises(BopRunError, match="not a compressed RLE character"):
        bop_run.rle_counts(seg("0~"), (4, 3), "d")
    with pytest.raises(BopRunError, match="truncated"):
        bop_run.rle_counts(seg("0P"), (4, 3), "d")        # continuation bit set on the last byte


# ---------------------------------------------------------------------------------------------------- layout
def test_split_and_model_directories():
    assert bop_run.split_name("tless") == ("test_primesense", "models_cad")
    assert bop_run.split_name("hb") == ("test_primesense", "models")
    assert bop_run.split_name("lmo") == ("test", "models")
    assert bop_run.detection_year("hope") == ("24", "cnos-sam")
    assert bop_run.detection_year("icbin") == ("19", "cnos-fastsam")
    with pytest.raises(BopRunError):
        bop_run.detection_year("unknown")


def test_default_detection_file_lookup(tmp_path):
    d = tmp_path / "default_detections" / "core19_model_based_unseen" / "cnos-fastsam"
    d.mkdir(parents=True)
    (d / "cnos-fastsam_ycbv-test_b.json").write_text("[]")
    (d / "cnos-fastsam_ycbv-test_a.json").write_text("[]")
    (d / "cnos-fastsam_lmo-test_a.json").write_text("[]")
    assert bop_run.default_detections(str(tmp_path / "ycbv")).endswith("cnos-fastsam_ycbv-test_a.json")
    with pytest.raises(BopRunError, match="tudl"):
        bop_run.default_detections(str(tmp_path / "tudl"))


def test_image_resolution_and_decoding(tmp_path):
    from PIL import Image
    rng = np.random.default_rng(0)
    rgb = rng.integers(0, 256, (6, 5, 3), dtype=np.uint8)
    gray = rng.integers(0, 256, (6, 5), dtype=np.uint8)
    s = tmp_path / "test" / "000002"
    (s / "rgb").mkdir(parents=True)
    (s / "gray").mkdir()
    Image.fromarray(rgb).save(s / "rgb" / "000001.png")
    Image.fromarray(rgb).save(s / "rgb" / "000003.jpg")
    Image.fromarray(rgb).save(s / "rgb" / "000003.png")
    Image.fromarray(gray).save(s / "gray" / "000004.tif")
    Image.fromarray(rng.integers(0, 4000, (6, 5)).astype(np.uint16)).save(s / "gray" / "000005.tif")
    p = lambda im: bop_run.image_path(str(tmp_path), "test", 2, im)
    assert p(1).endswith("rgb/000001.png") and p(3).endswith("rgb/000003.jpg") and p(4).endswith("gray/000004.tif")
    np.testing.assert_array_equal(bop_run.read_image(p(1)), rgb)
    np.testing.assert_array_equal(bop_run.read_image(p(4)), np.stack([gray] * 3, -1))
    with pytest.raises(BopRunError, match="8-bit"):
        bop_run.read_image(p(5))
    with pytest.raises(BopRunError, match="000009"):
        p(9)


def test_cameras_without_ground_truth(tmp_path):
    from gigapose_b200.bop_eval import load_cameras
    d = tmp_path / "test" / "000001"
    d.mkdir(parents=True)
    (d / "scene_camera.json").write_text(json.dumps({"4": {"cam_K": list(range(1, 10)), "depth_scale": 0.1}}))
    cam = load_cameras(str(tmp_path), "test", 1)
    np.testing.assert_array_equal(cam["K"][4], np.arange(1, 10, dtype=np.float64).reshape(3, 3))
    assert cam["depth_scale"][4] == 0.1


# ---------------------------------------------------------------------------------------------------- checkpoint
def _lightning_file(path, state):
    """A checkpoint whose hyper-parameters pickle an instance of a class from a module that cannot be imported."""
    mod = types.ModuleType("hydra_only_config_module")

    class NodeConfig:
        def __init__(self):
            self.content = {"_target_": "src.models.gigaPose.GigaPose", "lr": 1e-4}

    NodeConfig.__module__ = mod.__name__
    NodeConfig.__qualname__ = "NodeConfig"
    mod.NodeConfig = NodeConfig
    sys.modules[mod.__name__] = mod
    try:
        torch.save({"epoch": 3, "state_dict": state, "hyper_parameters": {"cfg": NodeConfig()},
                    "pytorch-lightning_version": "1.8.1"}, path)
    finally:
        del sys.modules[mod.__name__]
    with pytest.raises(Exception):
        torch.load(path, weights_only=False)          # plain loading cannot find the class


def test_checkpoint_loader_reads_a_lightning_file_with_unimportable_hyper_parameters(tmp_path):
    torch.manual_seed(0)
    src = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    path = str(tmp_path / "model.ckpt")
    _lightning_file(path, src.state_dict())
    dst = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    bop_run.load_checkpoint(dst, path)
    for a, b in zip(src.state_dict().values(), dst.state_dict().values()):
        assert torch.equal(a, b)
    missing = {k: v for k, v in src.state_dict().items() if k != "1.bias"}
    _lightning_file(path, missing)
    with pytest.raises(BopRunError, match=r"missing keys \['1.bias'\]"):
        bop_run.load_checkpoint(dst, path)
    extra = dict(src.state_dict(), **{"2.weight": torch.zeros(1)})
    _lightning_file(path, extra)
    with pytest.raises(BopRunError, match=r"unexpected keys \['2.weight'\]"):
        bop_run.load_checkpoint(dst, path)


def test_checkpoint_without_state_dict_is_refused(tmp_path):
    path = str(tmp_path / "x.ckpt")
    torch.save({"weights": torch.zeros(2)}, path)
    with pytest.raises(BopRunError, match="no state_dict"):
        bop_run.load_state_dict(path)


def test_checkpoint_unpickler_does_not_resolve_other_callables(tmp_path):
    path = str(tmp_path / "evil.ckpt")

    class Call:
        def __reduce__(self):
            return (os.getcwd, ())

    torch.save({"state_dict": {}, "hyper_parameters": Call()}, path)
    ckpt = torch.load(path, map_location="cpu", pickle_module=bop_run._pickle, weights_only=False)
    assert isinstance(ckpt["hyper_parameters"], bop_run._Inert)


def test_rle_crop_refuses_bad_arguments_without_a_device():
    """gp_crop_resize_pad_rle checks its arguments on the host before touching the device: every pointer below is a
    null or host address that the device never sees."""
    import ctypes as C
    from gigapose_b200 import _lib, build
    build.build()
    lib = _lib.load()
    fake = C.c_void_p(16)                                  # never dereferenced: each call fails its checks first
    off = lambda *v: (C.c_int64 * len(v))(*v)

    def call(n=2, H=480, W=640, T=224, images=fake, offsets=off(0, 3, 5), out=fake):
        return lib.gp_crop_resize_pad_rle(n, H, W, T, images, fake, fake, fake, offsets, fake, out, fake, fake, None)

    for kw, msg in ((dict(n=-1), b"bad shape"), (dict(T=127), b"target_size"), (dict(T=4097), b"target_size"),
                    (dict(images=None), b"null"), (dict(offsets=None), b"null"), (dict(out=None), b"null"),
                    (dict(offsets=off(0, 3, 2)), b"offsets decrease at detection 1"),
                    (dict(offsets=off(-1, 3, 5)), b"negative")):
        assert call(**kw) == -1, kw
        assert msg in lib.gp_last_error(), (kw, lib.gp_last_error())
