"""Query pre-processing on the GPU (row f3): `crop_resize_pad` is `CropResizePad.__call__` (reference
src/utils/crop.py:16-61) as one gather kernel, optionally fused with the dataloader's element-wise steps
(`process_real` dataloader/train.py:80-123: /255 and x mask; CLIP normalisation configs/data/transform.yaml:2-7).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def empty_crops(xyxy_boxes, height: int, width: int, target_size: int = 224) -> np.ndarray:
    """Indices of the boxes whose crop is empty once resized, on the host: the box's part inside the image (corner
    clamped to 0) has no rows or columns after `floor(size * scale)`, with the kernel's float32 scale
    `T * (1 / max(w, h))`.  The reference cannot crop such a box (`F.interpolate` refuses an empty output); the kernel
    writes zeros for it, so callers taking boxes from outside inputs refuse them with these indices."""
    b = np.asarray(xyxy_boxes, np.int64).reshape(-1, 4)
    x1, y1 = np.clip(b[:, 0], 0, width), np.clip(b[:, 1], 0, height)
    cw = np.maximum(np.minimum(b[:, 2], width) - x1, 0)
    ch = np.maximum(np.minimum(b[:, 3], height) - y1, 0)
    side = np.maximum(b[:, 2] - b[:, 0], b[:, 3] - b[:, 1])
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = (np.float32(1) / side.astype(np.float32)) * np.float32(target_size)     # __frcp_rn, __fmul_rn
        short = np.floor(np.minimum(ch, cw).astype(np.float64) * scale.astype(np.float64))
    return np.flatnonzero((side <= 0) | ~(short >= 1))


@torch.no_grad()
def crop_resize_pad(xyxy_boxes: torch.Tensor, images: torch.Tensor, target_size: int = 224,
                    image_index: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None, in_div: float = 1.0,
                    mean: Optional[Sequence[float]] = None, std: Optional[Sequence[float]] = None):
    """xyxy_boxes [n,4], images [n,C,H,W] (or [m,C,H,W] with image_index [n]) on a CUDA device ->
    dict(images [n,C,T,T], M [n,3,3][, mask [n,T,T]]).  mask [n,H,W] is multiplied in before the crop and returned
    cropped; in_div / mean / std apply `(x / in_div * mask - mean) / std` in the reference's operation order."""
    if not images.is_cuda:
        raise _lib.GigaPoseNativeError("crop_resize_pad runs on CUDA tensors only (no CPU fallback)")
    lib = _lib.load()
    dev = images.device
    images = images.to(torch.float32).contiguous()
    boxes = torch.as_tensor(xyxy_boxes, device=dev).long().contiguous()      # BoundingBox.convert_long (bbox.py:18-22)
    n = boxes.shape[0]
    _, C, H, W = images.shape
    idx = None
    if image_index is not None:
        idx = torch.as_tensor(image_index, device=dev).to(torch.int32).contiguous()
        assert idx.shape == (n,)
    else:
        assert images.shape[0] == n, "one image per box unless image_index is given"
    m = None
    if mask is not None:
        m = mask.to(device=dev, dtype=torch.float32).contiguous()
        assert m.shape == (n, H, W), tuple(m.shape)
    sub = torch.tensor(list(mean), dtype=torch.float32, device=dev) if mean is not None else None
    div = torch.tensor(list(std), dtype=torch.float32, device=dev) if std is not None else None
    assert sub is None or sub.numel() == C
    assert div is None or div.numel() == C
    T = int(target_size)
    out = torch.empty(n, C, T, T, device=dev)
    out_mask = torch.empty(n, T, T, device=dev) if m is not None else None
    M = torch.empty(n, 3, 3, device=dev)
    with torch.cuda.device(dev):
        check(lib.gp_crop_resize_pad(n, C, H, W, T, images.data_ptr(), ptr(idx), boxes.data_ptr(), ptr(m), float(in_div),
                                     ptr(sub), ptr(div), out.data_ptr(), ptr(out_mask), M.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream))
    res = {"M": M, "images": out}
    if out_mask is not None:
        res["mask"] = out_mask
    return res


@torch.no_grad()
def preprocess_queries(rgb_u8: torch.Tensor, masks: torch.Tensor, xyxy_boxes: torch.Tensor, batch_im_id: torch.Tensor,
                       target_size: int = 224):
    """Detections -> network inputs in one launch: rgb_u8 [m,3,H,W] (0..255), masks [n,H,W] {0,1}, boxes [n,4],
    batch_im_id [n] -> tar_img [n,3,T,T] (masked, CLIP-normalised), tar_mask [n,T,T], tar_M [n,3,3]."""
    r = crop_resize_pad(xyxy_boxes, rgb_u8.to(torch.float32), target_size, image_index=batch_im_id, mask=masks, in_div=255.0,
                        mean=CLIP_MEAN, std=CLIP_STD)
    return {"tar_img": r["images"], "tar_mask": r["mask"], "tar_M": r["M"]}


@torch.no_grad()
def crop_detections_rle(rgb_hwc: torch.Tensor, counts, offsets, xyxy_boxes, batch_im_id, target_size: int = 224):
    """`preprocess_queries` for masks given as COCO run-length encodings (row f9, gp_crop_resize_pad_rle): the dense
    masks are never built.  rgb_hwc u8 [m,H,W,3] on a CUDA device, counts i32 [sum of runs] (every detection's runs,
    concatenated; host or device), offsets [n+1] host ints (detection i owns counts[offsets[i]:offsets[i+1]]), boxes
    [n,4] xyxy, batch_im_id [n] -> tar_img [n,3,T,T], tar_mask [n,T,T], tar_M [n,3,3], bit for bit those of
    `preprocess_queries` on the decoded masks."""
    if not rgb_hwc.is_cuda:
        raise _lib.GigaPoseNativeError("crop_detections_rle runs on CUDA tensors only (no CPU fallback)")
    if rgb_hwc.dtype != torch.uint8 or rgb_hwc.dim() != 4 or rgb_hwc.shape[-1] != 3:
        raise ValueError(f"rgb_hwc must be uint8 [m,H,W,3], got {rgb_hwc.dtype} {tuple(rgb_hwc.shape)}")
    lib = _lib.load()
    dev = rgb_hwc.device
    images = rgb_hwc.contiguous()
    m, H, W, _ = images.shape
    boxes = torch.as_tensor(xyxy_boxes, device=dev).long().contiguous()
    n = boxes.shape[0]
    idx = torch.as_tensor(batch_im_id).to(torch.int64)
    if idx.shape != (n,) or (n and (int(idx.min()) < 0 or int(idx.max()) >= m)):
        raise ValueError(f"batch_im_id must be [{n}] indices into {m} images")
    idx = idx.to(device=dev, dtype=torch.int32, non_blocking=True)
    off = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
    if off.shape != (n + 1,):
        raise ValueError(f"offsets must have n + 1 = {n + 1} entries, got {off.shape[0]}")
    cnt = torch.as_tensor(counts, dtype=torch.int32).to(dev, non_blocking=True).contiguous()
    if cnt.numel() < off[-1]:
        raise ValueError(f"offsets end at {off[-1]} but counts holds {cnt.numel()} runs")
    ends = torch.empty(max(int(off[-1]), 1), dtype=torch.int64, device=dev)
    T = int(target_size)
    out = torch.empty(n, 3, T, T, device=dev)
    out_mask = torch.empty(n, T, T, device=dev)
    M = torch.empty(n, 3, 3, device=dev)
    with torch.cuda.device(dev):
        check(lib.gp_crop_resize_pad_rle(n, H, W, T, images.data_ptr(), idx.data_ptr(), boxes.data_ptr(), ptr(cnt),
                                         off.ctypes.data_as(C.POINTER(C.c_int64)), ends.data_ptr(), out.data_ptr(),
                                         out_mask.data_ptr(), M.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return {"tar_img": out, "tar_mask": out_mask, "tar_M": M}
