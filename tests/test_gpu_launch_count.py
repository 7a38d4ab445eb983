"""gp_launch_count() against the kernels the GPU actually ran.  bench.py reports the counter as `gpu_launches`; the
library counts a launch inside its one launcher (csrc/runtime.cu), so every entry-point family below must move the
counter by exactly the number of kernel records torch.profiler sees over the same region.  A second test runs the
same work on two devices of one process, which needs the dynamic shared memory opt-in on each device."""
import collections
import copy
import ctypes as C

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from gigapose_b200 import _lib, icp, synth
from gigapose_b200.engine import Engine
from gigapose_b200.ist_trunk import NativeISTTrunk
from gigapose_b200.preprocess import crop_resize_pad
from gigapose_b200.render import render_templates
from gigapose_b200.vit import DinoVisionTransformer
from gigapose_b200.vit_engine import NativeViT
from icp_scenes import DEV, K, T_ELL, ellipsoid, perturb, scene
from oracle import port

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _library_kernels(prof):
    """Names of the kernel records of a profile, without copies, memsets and torch's own kernels."""
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    return [n for n in names if not n.startswith(("Memcpy", "Memset")) and "at::" not in n]


def assert_counted(fn):
    """Runs fn() under the profiler; the library's launch count must move by the number of kernels the GPU ran."""
    lib = _lib.load()
    torch.cuda.synchronize(DEV)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        before = lib.gp_launch_count()
        result = fn()
        counted = lib.gp_launch_count() - before
        torch.cuda.synchronize(DEV)
    names = _library_kernels(prof)
    assert len(names) > 0, "the profiler recorded no kernels (no CUPTI?)"
    assert counted == len(names), (counted, collections.Counter(names))
    return result


def _engine_case():
    case = synth.make_feature_case(B=3, O=2, T=8, seed=5, device=DEV)
    return case, port.RegressorPort(seed=2).to(DEV)


@pytest.mark.parametrize("mlp_simt", ["1", "0"])
def test_engine_onboarding_and_retrieval(monkeypatch, mlp_simt):
    monkeypatch.setenv("GIGAPOSE_MLP_SIMT", mlp_simt)          # read by gp_create
    case, reg = _engine_case()
    ist = case.bank_ist.contiguous()
    ist_patch_major = ist.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)   # the channels-last view
    masks = case.bank_mask16.reshape(case.O, case.T, 16, 16)
    q_obj = case.q_label - 1

    def onboard():
        eng = Engine(case.O, case.T, case.B, device=DEV)
        eng.bank_write(0, 0, case.bank_feat[0], masks[0], ist_feat=ist[0])
        eng.bank_write(1, 0, case.bank_feat[1], masks[1], ist_feat=ist_patch_major[1])
        eng.set_poses(case.bank_K, case.bank_M, case.bank_poses)
        eng.set_ist_weights(reg)
        return eng

    eng = assert_counted(onboard)
    q_mask = case.q_mask16.reshape(-1, 16, 16)
    assert_counted(lambda: eng.retrieve(case.q_feat, q_mask, q_obj, case.q_ist, case.q_K, case.q_M))
    assert_counted(eng.debug_sim_tiles)
    assert_counted(lambda: eng.time_sim_kernel(iters=2))


def test_vit_create_forward_and_timing():
    vit = DinoVisionTransformer(depth=2).to(DEV)
    rgb, _ = synth.make_crops(2, seed=9, device=DEV)
    nv = assert_counted(lambda: NativeViT(vit, DEV, max_crops=2))
    assert_counted(lambda: nv.forward(rgb))
    assert_counted(lambda: nv.time_linears(2, iters=2))


def test_ist_trunk_create_forward_and_activation():
    from src.models.network.resnet import ResNet
    net = ResNet(dict(n_heads=0, input_dim=3, input_size=256, initial_dim=128, block_dims=[128, 192, 256, 512],
                      descriptor_size=256))
    net.load_state_dict(port.ISTBackbonePort().state_dict())
    net = net.to(DEV).eval()
    rgb, _ = synth.make_crops(2, seed=9, device=DEV)
    trunk = assert_counted(lambda: NativeISTTrunk(net, DEV, max_crops=2))
    assert_counted(lambda: trunk.forward(rgb))
    assert_counted(lambda: trunk.activation_after(rgb, 5))
    assert_counted(lambda: trunk.activation_after(rgb, 0))


def test_crop_render_and_icp():
    g = torch.Generator(device=DEV).manual_seed(1)
    images = torch.rand(2, 3, 120, 160, generator=g, device=DEV)
    boxes = torch.tensor([[10, 20, 90, 100], [0, 0, 160, 120]], device=DEV)
    assert_counted(lambda: crop_resize_pad(boxes, images, target_size=224))
    mesh = ellipsoid()
    poses = torch.as_tensor(np.stack([T_ELL, perturb(T_ELL, [0, 1, 0], 5, [3, 0, 0])])).to(DEV)
    assert_counted(lambda: render_templates(mesh, poses, K, size=(240, 320), device=DEV))
    depth, _ = scene(mesh, T_ELL)
    dm = icp.device_meshes([mesh], DEV)
    T0 = torch.as_tensor(perturb(T_ELL, [1, 0, 0], 3, [4, -2, 5]))[None].to(DEV)
    assert_counted(lambda: icp.refine_icp(dm, [0], T0, depth, torch.as_tensor(K), [0]))


def test_debug_hooks():
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(3)
    rand = lambda *s: torch.randn(*s, generator=g, device=DEV)
    planes = lambda *s: (rand(*s).to(torch.bfloat16), rand(*s).to(torch.bfloat16) * 2 ** -8)
    empty_planes = lambda *s: tuple(torch.empty(*s, dtype=torch.bfloat16, device=DEV) for _ in range(2))

    a, w, bias, out = planes(128, 64), planes(256, 64), rand(256), empty_planes(128, 256)
    d = _lib.GpDebugGemm(M=128, N=256, K=64, bn=256, passes=3, mode=_lib.GEMM_PLANES, a_hi=a[0].data_ptr(),
                         a_lo=a[1].data_ptr(), w_hi=w[0].data_ptr(), w_lo=w[1].data_ptr(), out_hi=out[0].data_ptr(),
                         out_lo=out[1].data_ptr(), bias=bias.data_ptr())
    assert_counted(lambda: _lib.check(lib.gp_debug_gemm(C.byref(d), _stream())))

    qkv, att = planes(3 * 16 * 257, 64), empty_planes(257, 1024)
    assert_counted(lambda: _lib.check(lib.gp_debug_attention(1, 1, 3, qkv[0].data_ptr(), qkv[1].data_ptr(),
                                                             att[0].data_ptr(), att[1].data_ptr(), _stream())))

    x, lw, lb, ln = rand(8, 1024), rand(1024), rand(1024), empty_planes(8, 1024)
    assert_counted(lambda: _lib.check(lib.gp_debug_layernorm(8, x.data_ptr(), lw.data_ptr(), lb.data_ptr(),
                                                             ln[0].data_ptr(), ln[1].data_ptr(), _stream())))

    bits = torch.randint(0, 1 << 30, (100,), generator=g, dtype=torch.int32, device=DEV)
    sel = torch.empty(2, dtype=torch.int32, device=DEV)
    assert_counted(lambda: _lib.check(lib.gp_debug_icp_select(bits.data_ptr(), 100, 10, sel.data_ptr(), _stream())))


def test_two_devices_compute_the_same_bits():
    """sim_topk and a 2-block ViT forward on cuda:0 and then on cuda:1, in one process: each device's kernels need
    their own dynamic shared memory opt-in, and the outputs must not depend on the device."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    case = synth.make_feature_case(B=3, O=2, T=8, seed=5)
    vit = DinoVisionTransformer(depth=2)
    rgb, _ = synth.make_crops(2, seed=9)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        with torch.cuda.device(dev):
            eng = Engine(case.O, case.T, case.B, device=dev)
            for o in range(case.O):
                eng.bank_write(o, 0, case.bank_feat[o], case.bank_mask16[o].reshape(-1, 16, 16))
            eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), (case.q_label - 1).to(dev))
            m = {k: v.cpu() for k, v in eng.sim_topk().items()}
            x = NativeViT(copy.deepcopy(vit).to(dev), dev, max_crops=2).forward(rgb.to(dev)).cpu()
            outs.append((m, x))
    (m0, x0), (m1, x1) = outs
    for k in m0:
        assert torch.equal(m0[k], m1[k]), k
    assert torch.equal(x0, x1)
