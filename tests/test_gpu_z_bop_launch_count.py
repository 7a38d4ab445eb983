"""gp_launch_count() against the kernels torch.profiler records around bop_eval.evaluate() (row f7), with the helper of
tests/test_gpu_launch_count.py restated.  This file sorts after that one on purpose: on an H100, a profiling session run
earlier in the same pytest process, or in a child process of it, made that file's later sessions record no kernels."""
import collections

import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from gigapose_b200 import _lib, bop_eval
from test_gpu_bop_eval import DEV, _tree

pytestmark = pytest.mark.gpu


def _library_kernels(prof):
    """Names of the kernel records of a profile, without copies, memsets and torch's own kernels."""
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    return [n for n in names if not n.startswith(("Memcpy", "Memset")) and "at::" not in n]


def test_launch_count_moves_by_the_kernels_evaluate_runs(tmp_path):
    results, _, _, _ = _tree(tmp_path)
    lib = _lib.load()
    torch.cuda.synchronize(DEV)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        before = lib.gp_launch_count()
        bop_eval.evaluate(results, str(tmp_path), device=DEV)
        counted = lib.gp_launch_count() - before
        torch.cuda.synchronize(DEV)
    names = _library_kernels(prof)
    assert len(names) > 0, "the profiler recorded no kernels (no CUPTI?)"
    assert counted == len(names), (counted, collections.Counter(names))
    kinds = collections.Counter(names)
    assert any("vsd_kernel" in k for k in kinds) and any("mssd_mspd_kernel" in k for k in kinds)
