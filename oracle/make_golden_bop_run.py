"""TEST INFRASTRUCTURE ONLY -- regenerates tests/golden/bop_run_selection.json by running the UNMODIFIED reference
detection loaders (`load_test_list_and_cnos_detections`, `generate_test_list`, the reference's
src/utils/inout.py:370-492; needs the reference checkout that `oracle.ref_import` finds) with the per-target caps of
`GigaPoseTestSet.load_detections` (dataloader/test.py:110-114), and the reference's own xywh -> xyxy box conversion (`BoundingBox`, src/utils/bbox.py, on the float32 tensor the collate
builds, scene_dataset.py:337), on seeded synthetic CNOS detection files and test-target lists.

Cases: targets whose object has no detection in the image (all of the image's detections, relabelled), tied scores,
more than 16 and more than 32 detections per object, an lmo and an icbin dataset, fractional boxes, both settings.

    python -m oracle.make_golden_bop_run
"""
from __future__ import annotations

import json
import os
import pathlib
import tempfile

import numpy as np
import torch

from . import ref_import

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "bop_run_selection.json")
LMO_IDS = [1, 5, 6, 8, 9, 10, 11, 12]


def make_case(dataset, seed):
    """-> (detections, targets): 4 images over 2 scenes; per image a few objects with 1 to 40 detections, scores on a
    coarse grid (ties), fractional xywh boxes; targets include objects with no detection in their image."""
    rng = np.random.default_rng(seed)
    objs = LMO_IDS if dataset == "lmo" else list(range(1, 9))
    images = [(1, 0), (1, 5), (3, 2), (3, 9)]
    dets, targets = [], []
    for i, (s, im) in enumerate(images):
        present = rng.choice(objs, size=3, replace=False).tolist()
        counts = [1, 17 if i % 2 == 0 else 5, 40 if i == 1 else int(rng.integers(2, 9))]
        for o, n in zip(present, counts):
            for _ in range(n):
                x, y = rng.uniform(-5, 600, 2)
                w, h = rng.uniform(0.5, 200, 2)
                dets.append(dict(scene_id=s, image_id=im, category_id=int(o), score=float(rng.integers(0, 8) / 8.0),
                                 bbox=[float(x), float(y), float(w), float(h)], time=float(0.1 + 0.01 * i),
                                 det_idx=len(dets)))
        absent = [o for o in objs if o not in present][:2]
        for o in present[1:] + absent:
            targets.append(dict(scene_id=s, im_id=im, obj_id=int(o), inst_count=int(rng.integers(1, 4))))
    perm = rng.permutation(len(dets))                     # file order is not grouped by image
    return [dets[k] for k in perm], targets


CASES = [("lmo", "localization", 5), ("icbin", "localization", 6), ("ycbv", "localization", 7), ("lmo", "detection", 8),
         ("icbin", "detection", 9)]


def main():
    io = ref_import.load_inout()
    io.inout.load_json = lambda path: json.load(open(path))
    with ref_import._ReferenceImports() as ctx:
        BoundingBox = ctx.import_reference("src.utils.bbox").BoundingBox
    out = []
    for dataset, setting, seed in CASES:
        dets, targets = make_case(dataset, seed)
        with tempfile.TemporaryDirectory() as root:
            d = os.path.join(root, "default_detections", "core19_model_based_unseen", "cnos-fastsam")
            os.makedirs(d)
            with open(os.path.join(d, f"cnos-fastsam_{dataset}-test_synthetic.json"), "w") as f:
                json.dump(dets, f)
            os.makedirs(os.path.join(root, dataset))
            with open(os.path.join(root, dataset, "test_targets_bop19.json"), "w") as f:
                json.dump(targets, f)
            cap = (32 if dataset == "icbin" else 16) if setting == "localization" else None
            test_list, selected = io.load_test_list_and_cnos_detections(pathlib.Path(root), dataset, setting,
                                                                        max_det_per_object_id=cap)
        expect = {}
        for key, im_dets in selected.items():
            boxes = BoundingBox(torch.stack([torch.tensor(np.array(d["bbox"])).float() for d in im_dets]), "xywh")
            expect[key] = dict(det_idx=[d["det_idx"] for d in im_dets], label=[d["category_id"] for d in im_dets],
                               score=[d["score"] for d in im_dets], xyxy=boxes.xyxy_box.tolist(),
                               time=im_dets[0]["time"],
                               targets=[[t["obj_id"], t["inst_count"]] for t in test_list[key]])
        assert sorted(test_list) == sorted(selected)
        out.append(dict(dataset=dataset, setting=setting, detections=dets, targets=targets, expect=expect))
        print(dataset, setting, len(dets), "detections ->", sum(len(v["det_idx"]) for v in expect.values()), "kept")
    with open(GOLDEN, "w") as f:
        json.dump(out, f)


if __name__ == "__main__":
    main()
