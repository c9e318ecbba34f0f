"""CPU-side checks of the C-ABI boundary: the library builds for sm_90a, loads without a GPU, exports every
symbol include/vdk_b200.h declares, and its host-only entry points (plans, argument validation) behave."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from visiondk_b200 import _lib

ROOT = Path(__file__).resolve().parents[1]


def declared_symbols():
    text = (ROOT / "include" / "vdk_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vdk_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol(lib):
    names = declared_symbols()
    assert len(names) >= 10
    for name in names:
        assert hasattr(lib, name), f"{name} is declared in include/vdk_b200.h but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature in visiondk_b200/_lib.py"
    assert sorted(_lib.SIGNATURES) == names


def test_library_is_sm90a_only(lib):
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", str(_lib.lib_path())], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_version_and_error_string(lib):
    assert lib.vdk_version() >= 100
    assert isinstance(_lib.last_error(), str)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_compute_fails_loudly_without_gpu(lib):
    assert lib.vdk_device_check() == _lib.VDK_ERR_CUDA
    with pytest.raises(RuntimeError):
        _lib.require_device()
    from visiondk_b200.retrieval import FlatIPIndex
    with pytest.raises(RuntimeError):
        FlatIPIndex(64, "cpu")


def test_topk_plan_default(lib):
    plan = _lib.TopkPlan()
    assert lib.vdk_topk_plan_default(C.byref(plan), 10000, 1000000, 512, 100) == 0
    ends = list(plan.stage_end)[:plan.n_stages]
    assert ends == [4096, 32768, 262144, 1000000] and plan.cand_capacity == 16384 and plan.carry_capacity == 2048
    assert all(e % 256 == 0 for e in ends[:-1])
    assert lib.vdk_topk_workspace_bytes(C.byref(plan)) >= 10000 * (16384 + 2 * 2048) * 8
    assert lib.vdk_topk_plan_default(C.byref(plan), 5, 100, 64, 10) == 0
    assert plan.n_stages == 1 and plan.stage_end[0] == 100
    assert lib.vdk_topk_plan_default(C.byref(plan), 5, 100, 64, 1024) == 0
    assert plan.cand_capacity == 16384 and plan.carry_capacity == 4096
    assert lib.vdk_topk_plan_default(C.byref(plan), 5, 100, 100, 10) == _lib.VDK_ERR_INVALID
    assert "multiple of 64" in _lib.last_error()
    assert lib.vdk_topk_plan_default(C.byref(plan), 5, 100, 64, 0) == _lib.VDK_ERR_INVALID


def test_argument_validation_needs_no_gpu(lib):
    assert lib.vdk_gemm_tn(0, 0, 0, 8, 8, 8, 8, 8, 8, 0, 0, 0, 0, 0, 0, 0, 0) == _lib.VDK_ERR_INVALID
    assert lib.vdk_rows_prepare(0, 4, 64, 1, 0, 0, 0, 0, 0) == _lib.VDK_ERR_INVALID
    assert lib.vdk_topk_merge(0, 0, 2, 4, 4, 0, 0, 0) == _lib.VDK_ERR_INVALID


def test_ctypes_mirrors_have_the_c_struct_sizes():
    """The Python side mirrors the ABI structs by hand (ctypes.Structure): their sizes must equal the compiler's sizeof."""
    import ctypes as C
    from visiondk_b200 import _lib
    from visiondk_b200.backbone import ConvNeXtNetC, ConvNeXtTensorsC
    from visiondk_b200.vit import VitNetC, VitTensorsC
    lib = _lib.load()
    out = (C.c_size_t * 8)()
    n = lib.vdk_struct_sizes(out, 8)
    mirrors = [_lib.GemmDesc, _lib.TopkPlan, _lib.HeadDesc, ConvNeXtNetC, ConvNeXtTensorsC, VitNetC, VitTensorsC]
    assert n == len(mirrors)
    for i, m in enumerate(mirrors):
        assert C.sizeof(m) == out[i], (m.__name__, C.sizeof(m), out[i])
