"""Executes the DINOv2 ViT-L/14 forward for `AENet` (row a1) on the native kernels of libgigapose_b200.so:
im2col -> wgmma GEMM (patch embedding) -> 24 x [LayerNorm -> wgmma QKV GEMM -> attention -> wgmma proj GEMM
(+LayerScale +residual) -> LayerNorm -> wgmma FC1 GEMM (+GELU) -> wgmma FC2 GEMM (+LayerScale +residual)].
All GEMM operands are bf16 hi/lo planes accumulated in fp32 (fp32-faithful); see csrc/vit_gemm.cu, csrc/vit_ops.cu.

The module passed in only supplies parameters (upstream DinoVisionTransformer attribute names); its own forward is
never called.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib
from ._lib import check

BACKEND = "native-wgmma"
TOK, DIM = 257, 1024


def _params_in_abi_order(m, device):
    """4 + 14*depth fp32 tensors in the order gp_vit_create documents."""
    f = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()
    ps = m.patch_size if isinstance(m.patch_size, int) else m.patch_size[0]
    assert ps == 14 and m.pos_embed.shape[-1] == DIM, "kernels are specialised for ViT-L/14"
    if hasattr(m, "interpolated_pos_embed"):
        pos = m.interpolated_pos_embed(16, 16)
    else:   # upstream hub module: same bicubic routine under a different name
        pos = m.interpolate_pos_encoding(torch.zeros(1, TOK, DIM, device=m.pos_embed.device), 224, 224)
    out = [f(m.patch_embed.proj.weight).reshape(DIM, -1), f(m.patch_embed.proj.bias), f(m.cls_token).reshape(DIM),
           f(pos).reshape(TOK, DIM)]
    for blk in m.blocks:
        assert blk.attn.num_heads == 16
        out += [f(blk.norm1.weight), f(blk.norm1.bias), f(blk.attn.qkv.weight), f(blk.attn.qkv.bias),
                f(blk.attn.proj.weight), f(blk.attn.proj.bias), f(blk.ls1.gamma), f(blk.norm2.weight), f(blk.norm2.bias),
                f(blk.mlp.fc1.weight), f(blk.mlp.fc1.bias), f(blk.mlp.fc2.weight), f(blk.mlp.fc2.bias), f(blk.ls2.gamma)]
    return out


def _version_key(m):
    """Staleness key over EVERY parameter (storage address + in-place version counter): the packed GEMM planes and the
    retained bias / norm pointers must be rebuilt when any tensor of the module is replaced (`.to()`, `load_state_dict`,
    `.half()`) or modified in place.  ~340 tensors for ViT-L: tens of microseconds per call."""
    return hash(tuple((p.data_ptr(), int(p._version)) for p in m.parameters()))


class NativeViT:
    def __init__(self, model, device, max_crops: int = 64, precision: str = "fp32_split"):
        self.lib = _lib.load()
        self.device = _lib.cuda_device(device, "the ViT kernels run")
        self.depth = len(model.blocks)
        self.max_crops = max_crops
        self.weights = _params_in_abi_order(model, self.device)          # kept alive: referenced in place
        wb, sb = C.c_size_t(), C.c_size_t()
        check(self.lib.gp_vit_query_sizes(self.depth, max_crops, C.byref(wb), C.byref(sb)))
        self._wmem, wview = _lib.aligned_buffer(wb.value, self.device)
        self._smem, sview = _lib.aligned_buffer(sb.value, self.device)
        arr = (C.c_void_p * len(self.weights))(*[w.data_ptr() for w in self.weights])
        h = C.c_void_p()
        prec = {"fp32_split": _lib.PRECISION_FP32_SPLIT, "bf16": _lib.PRECISION_BF16}[precision]
        check(self.lib.gp_vit_create(self.device.index, self.depth, max_crops, prec, arr, wview.data_ptr(), sview.data_ptr(),
                                     torch.cuda.current_stream(self.device).cuda_stream, C.byref(h)))
        self._h = h
        self.precision = precision

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                self.lib.gp_vit_destroy(h)
            except Exception:
                pass
            self._h = None

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        assert x.shape[1:] == (3, 224, 224), f"kernels are specialised for 224x224 crops, got {tuple(x.shape)}"
        x = x.to(self.device, dtype=torch.float32).contiguous()
        out = torch.empty(x.shape[0], TOK, DIM, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        for i in range(0, x.shape[0], self.max_crops):
            xi = x[i:i + self.max_crops]
            check(self.lib.gp_vit_forward(self._h, xi.shape[0], xi.data_ptr(), out[i:i + self.max_crops].data_ptr(), stream))
        return out


    def time_linears(self, b: int, iters: int = 5) -> float:
        """Average milliseconds of the 4 * depth linear layers of one forward over `b` crops (CUDA events, alone)."""
        ms = C.c_float()
        check(self.lib.gp_vit_time_linears(self._h, b, iters, C.byref(ms), torch.cuda.current_stream(self.device).cuda_stream))
        return ms.value


@torch.no_grad()
def vit_forward_features(model, x: torch.Tensor, precision: str = None) -> torch.Tensor:
    """x [b,3,224,224] -> x_prenorm [b,257,1024] (tokens after the last block, before the final norm)."""
    precision = precision or os.environ.get("GIGAPOSE_VIT_PRECISION", "fp32_split")
    key = (str(x.device), precision, _version_key(model))
    eng = getattr(model, "_gp_vit_engine", None)
    if eng is None or eng[0] != key:
        eng = (key, NativeViT(model, x.device, precision=precision))
        object.__setattr__(model, "_gp_vit_engine", eng)
    return eng[1].forward(x)
