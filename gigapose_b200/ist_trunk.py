"""Executes the IST trunk (`ResNet`, reference src/models/network/resnet.py:318-381, rows a6 / f1) on the native
kernels of libgigapose_b200.so: fused resize + stem im2col, then 21 implicit-GEMM convolutions on wgmma with
TMA-fetched filter taps (csrc/ist_trunk.cu, csrc/vit_gemm.cu).  BatchNorm is folded into the filters here (a
weight-only computation); activations stay NHWC bf16 hi/lo planes between layers (fp32-faithful 3-pass products).

The module passed in only supplies parameters (reference state-dict names); its own forward is never called.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib
from ._lib import check

BACKEND = "native-wgmma"
NUM_CONVS = 21
GEOMETRY = dict(input_size=256, initial_dim=128, block_dims=[128, 192, 256, 512], descriptor_size=256)


class ConvWeights(C.Structure):               # == gp_conv_weights_t
    _fields_ = [("weight", C.c_void_p), ("bias", C.c_void_p)]


def supports(resnet) -> bool:
    """The kernels are specialised for the shipped trunk (configs/model/ist_net/resnet.yaml)."""
    try:
        dims = [resnet.layer1[0].conv2.out_channels, resnet.layer2[0].conv2.out_channels,
                resnet.layer3[0].conv2.out_channels, resnet.layer4[0].conv2.out_channels]
        return (resnet.input_size == 256 and resnet.conv1.in_channels == 3 and resnet.conv1.out_channels == 128 and
                dims == GEOMETRY["block_dims"] and resnet.layer4_outconv.out_channels == 256)
    except AttributeError:
        return False


def _fold(conv, bn, device):
    """[cout, kh, kw, cin] filter with the inference-time BatchNorm scale folded in, and the folded bias."""
    w = conv.weight.detach().to(device=device, dtype=torch.float32)
    if bn is None:
        return w.permute(0, 2, 3, 1).contiguous(), None
    g = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).detach().to(device=device, dtype=torch.float32)
    b = (bn.bias.detach().to(device) - bn.running_mean.detach().to(device) * g).to(torch.float32).contiguous()
    return (w * g.view(-1, 1, 1, 1)).permute(0, 2, 3, 1).contiguous(), b


def folded_convs_in_abi_order(resnet, device):
    """The 21 (filter, bias) pairs in the execution order gp_ist_trunk_create documents."""
    out = [_fold(resnet.conv1, resnet.bn1, device)]
    for layer in (resnet.layer1, resnet.layer2, resnet.layer3, resnet.layer4):
        for blk in layer:
            out.append(_fold(blk.conv1, blk.bn1, device))
            if blk.downsample is not None:
                out.append(_fold(blk.downsample[0], blk.downsample[1], device))
            out.append(_fold(blk.conv2, blk.bn2, device))
    out.append(_fold(resnet.layer4_outconv, None, device))
    assert len(out) == NUM_CONVS
    return out


def _version_key(resnet):
    """Staleness key over every parameter and BatchNorm buffer (storage address + in-place version counter)."""
    return hash(tuple((t.data_ptr(), int(t._version)) for t in list(resnet.parameters()) + list(resnet.buffers())))


class NativeISTTrunk:
    def __init__(self, resnet, device, max_crops: int = 32, precision: str = "fp32_split"):
        self.lib = _lib.load()
        self.device = _lib.cuda_device(device, "the IST trunk kernels run")
        if not supports(resnet):
            raise _lib.GigaPoseNativeError("the IST trunk kernels are specialised for the shipped ResNet geometry")
        self.max_crops = max_crops
        with torch.no_grad():
            self.weights = folded_convs_in_abi_order(resnet, self.device)     # biases referenced in place: keep alive
        wb, sb = C.c_size_t(), C.c_size_t()
        check(self.lib.gp_ist_trunk_query_sizes(max_crops, C.byref(wb), C.byref(sb)))
        self._wmem, wview = _lib.aligned_buffer(wb.value, self.device)
        self._smem, sview = _lib.aligned_buffer(sb.value, self.device, zero=True)
        arr = (ConvWeights * NUM_CONVS)(*[ConvWeights(w.data_ptr(), _lib.ptr(b))
                                          for w, b in self.weights])
        h = C.c_void_p()
        prec = {"fp32_split": _lib.PRECISION_FP32_SPLIT, "bf16": _lib.PRECISION_BF16}[precision]
        check(self.lib.gp_ist_trunk_create(self.device.index, max_crops, prec, C.cast(arr, C.c_void_p), wview.data_ptr(),
                                           sview.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream, C.byref(h)))
        self._h = h
        self.precision = precision

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                self.lib.gp_ist_trunk_destroy(h)
            except Exception:
                pass
            self._h = None

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [n,3,224,224] -> [n,256,16,16] (a channels-last view of the patch-major buffer the kernels write)."""
        assert x.shape[1:] == (3, 224, 224), f"kernels are specialised for 224x224 crops, got {tuple(x.shape)}"
        x = x.to(self.device, dtype=torch.float32).contiguous()
        out = torch.empty(x.shape[0], 16, 16, 256, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        for i in range(0, x.shape[0], self.max_crops):
            xi = x[i:i + self.max_crops]
            check(self.lib.gp_ist_trunk_forward(self._h, xi.shape[0], xi.data_ptr(), out[i:i + self.max_crops].data_ptr(), stream))
        return out.permute(0, 3, 1, 2)

    @torch.no_grad()
    def activation_after(self, x: torch.Tensor, num_convs: int) -> torch.Tensor:
        """Test hook: NHWC output of the `num_convs`-th convolution (execution order) as fp32 [n,h,w,c]; num_convs = 0
        gives the stem's input, the resized crops with their zero border, as fp32 [n,262,264,4]."""
        shapes = []
        h = 128
        shapes.append((h, 128))
        for st, d in enumerate(GEOMETRY["block_dims"]):
            for blk in range(2):
                if blk == 0 and st > 0:
                    h //= 2
                    shapes += [(h, d), (h, d), (h, d)]
                else:
                    shapes += [(h, d), (h, d)]
        x = x.to(self.device, dtype=torch.float32).contiguous()
        assert x.shape[0] <= self.max_crops
        if num_convs == 0:
            shape = (262, 264, 4)
        else:
            hh, cc = shapes[num_convs - 1]
            shape = (hh, hh, cc)
        out = torch.empty(x.shape[0], *shape, device=self.device)
        check(self.lib.gp_debug_ist_trunk(self._h, x.shape[0], x.data_ptr(), num_convs, out.data_ptr(),
                                          torch.cuda.current_stream(self.device).cuda_stream))
        return out


@torch.no_grad()
def trunk_forward(resnet, x: torch.Tensor, precision: str = None) -> torch.Tensor:
    precision = precision or os.environ.get("GIGAPOSE_IST_PRECISION", "fp32_split")
    key = (str(x.device), precision, _version_key(resnet))
    eng = getattr(resnet, "_gp_trunk_engine", None)
    if eng is None or eng[0] != key:
        eng = (key, NativeISTTrunk(resnet, x.device, precision=precision))
        object.__setattr__(resnet, "_gp_trunk_engine", eng)
    return eng[1].forward(x)
