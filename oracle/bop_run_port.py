"""TEST INFRASTRUCTURE ONLY -- the COCO run-length encodings of CNOS masks in numpy, for the row f9 tests.

`rle_to_binary_mask` restates the BOP toolkit's `bop_toolkit_lib.pycoco_utils.rle_to_binary_mask`, which the reference's
test loader calls on every detection (dataloader/test.py:238): a flat boolean array of H * W zeros; run i + 1 of the
counts (i = 0 .. len - 2) covers [sum(counts[:i + 1]), sum(counts[:i + 2])) and is set to (i + 1) % 2, numpy slicing
cutting off whatever lies past H * W; the array is then reshaped to [H, W] in column-major ('F') order.  The toolkit is
neither vendored nor installed here, so this restatement is written from that description and is not pinned against
the toolkit itself.

The encoders are the inverse operations the tests use to build inputs: `binary_mask_to_rle` (the list form CNOS writes)
and `rle_to_string` (COCO's compressed string form, `rleToString` of the COCO mask API).
"""
from __future__ import annotations

import numpy as np


def rle_to_binary_mask(rle):
    """rle: dict(size [H, W], counts [int]) -> bool [H, W]."""
    binary_array = np.zeros(int(np.prod(rle["size"])), dtype=bool)
    counts = rle["counts"]
    start = 0
    for i in range(len(counts) - 1):
        start += counts[i]
        end = start + counts[i + 1]
        binary_array[start:end] = (i + 1) % 2
    return binary_array.reshape(*rle["size"], order="F")


def binary_mask_to_rle(mask):
    """bool / {0,1} [H, W] -> dict(size [H, W], counts [int]): column-major runs, the first counting zeros."""
    flat = np.asarray(mask, bool).reshape(-1, order="F")
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(bounds).tolist()
    if flat.size and flat[0]:
        counts = [0] + counts
    return {"size": list(np.asarray(mask).shape), "counts": [int(c) for c in counts]}


def rle_to_string(counts):
    """Run lengths -> COCO's compressed string: each count, minus the one two places before it from the fourth on, in
    little-endian groups of 5 bits with a continuation bit, offset by 48."""
    out = []
    for i, c in enumerate(counts):
        x = int(c) - (int(counts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            ch = x & 0x1F
            x >>= 5
            more = not ((ch & 0x10) == 0 and x == 0 or (ch & 0x10) != 0 and x == -1)
            if more:
                ch |= 0x20
            out.append(chr(ch + 48))
    return "".join(out)
