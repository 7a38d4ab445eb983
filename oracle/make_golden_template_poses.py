"""TEST INFRASTRUCTURE ONLY -- regenerates tests/golden/template_poses.npz from the reference's predefined template poses
(src/lib3d/predefined_poses/{obj,cam}_poses_level{0,1,2}.npy, written by its Blender script
src/lib3d/create_template_poses.py; needs the reference checkout that `oracle.ref_import` finds).  The arrays are
copied as they are, under the names obj_poses_level{L} and cam_poses_level{L}; tests/test_template_poses_cpu.py pins
`gigapose_b200.template_poses` to them.

    python -m oracle.make_golden_template_poses
"""
from __future__ import annotations

import os

import numpy as np

from . import ref_import

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "template_poses.npz")


def main():
    src = os.path.join(ref_import.REF_ROOT, "src", "lib3d", "predefined_poses")
    arrays = {f"{kind}_poses_level{level}": np.load(os.path.join(src, f"{kind}_poses_level{level}.npy"))
              for level in (0, 1, 2) for kind in ("obj", "cam")}
    np.savez_compressed(GOLDEN, **arrays)
    print(GOLDEN, {k: v.shape for k, v in arrays.items()})


if __name__ == "__main__":
    main()
