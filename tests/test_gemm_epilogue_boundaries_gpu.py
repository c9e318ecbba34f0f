"""Boundaries of the GEMM's TMA epilogue that tests/test_gemm_gpu.py does not reach.

Each consumer warpgroup stores its own 64-row half of a 128-row tile through a ring of 64-row x 128-byte shared-memory
boxes, and TMA-loads the residual / saved pre-activation into that ring.  These cases put the boundaries of that scheme
on the fp64 references of test_gemm_gpu.py:
  * M % 128 <= 64: the second warpgroup's half of the last row tile lies entirely below M and skips its epilogue.  These
    cases check that the skip neither deadlocks the warpgroup's ring nor leaves rows of the first half unwritten; a stray
    store below M would be clipped by the output's tensor map, so they cannot see one (the NaN-guarded rows past M only
    show that nothing outside the map is written);
  * an fp32 residual wider than the ring (BN = 256: eight 32-column boxes, four ring slots), loaded box by box;
  * split-K slabs with split_stride > M * ldd and ldd > N, and atomic split-K (TMA reduce-add) with a ragged M.
"""
import ctypes as C

import pytest
import torch

from kernel_ref import check_within, split_k_bound
from test_gemm_gpu import E, check_epilogue, describe_tiles, operands, run, tile_n
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu


def epilogue_case(M, N, K, in_dtype, out_dtype, epilogue, seed, bias=True, aux=False, in_place=False, ldr_pad=0, ldd_pad=0, tb=0):
    a, b = operands(M, N, K, in_dtype, seed, 0.5, 0.25)
    odt = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}[out_dtype]
    bias_t = torch.randn(N, device="cuda") if bias else None
    gamma = beta = residual = None
    if epilogue == E.EPI_SCALE_RESIDUAL:
        gamma = torch.rand(N, device="cuda") * 2 - 0.5
        residual = torch.randn(M, N, device="cuda").to(odt)
    elif epilogue == E.EPI_LAYERNORM:
        gamma = torch.rand(N, device="cuda") + 0.5
        beta = torch.randn(N, device="cuda")
    elif epilogue == E.EPI_MUL_GELU_GRAD:
        residual = (3 * torch.randn(M, N, device="cuda")).to(odt)
    d, ax = run(a, b, odt, epilogue, bias=bias_t, gamma=gamma, beta=beta, residual=residual, ldr_pad=ldr_pad, ldd_pad=ldd_pad,
                aux=aux, tb=tb, in_place=in_place)
    check_epilogue(a, b, odt, epilogue, d, ax, bias=bias_t, gamma=gamma, beta=beta, residual=residual,
                   name=f"M{M} N{N} K{K} epi{epilogue}")


# M % 128 in {1, 40, 64}: the last row tile's second half is empty (40, 1) or the first half exactly full (64)
@pytest.mark.parametrize("tail", [1, 40, 64])
@pytest.mark.parametrize("case", [
    ("bf16", "bf16", E.EPI_GELU, 512, dict(aux=True)),
    ("bf16", "bf16", E.EPI_SCALE_RESIDUAL, 512, dict(in_place=True)),
    ("fp16", "fp16", E.EPI_MUL_GELU_GRAD, 200, dict(bias=False, ldr_pad=8)),
    ("bf16", "fp32", E.EPI_NONE, 520, dict(ldd_pad=4)),
    ("bf16", "bf16", E.EPI_LAYERNORM, 256, dict()),
], ids=["gelu_aux", "scale_res_inplace", "gelu_grad", "fp32_none", "layernorm"])
def test_gemm_half_tile_below_m(lib, tail, case):
    in_dtype, out_dtype, epilogue, N, opts = case
    M = 3 * 128 + tail
    assert M % 128 <= 64
    epilogue_case(M, N, 128, in_dtype, out_dtype, epilogue, seed=M + N, **opts)


@pytest.mark.parametrize("M", [1000, 4 * 132 * 128 // 2 + 17])
def test_gemm_fp32_residual_wider_than_ring(lib, M):
    """fp32 output and residual at BN = 256: each warpgroup's half tile spans eight 32-column boxes, four more than its
    ring holds, so boxes 4-7 load their residual after the stores of boxes 0-3 have read their slots."""
    N = 512
    assert tile_n(N, E.EPI_SCALE_RESIDUAL) == 256
    epilogue_case(M, N, 96, "bf16", "fp32", E.EPI_SCALE_RESIDUAL, seed=M, ldr_pad=12, ldd_pad=4)


def test_gemm_split_k_slabs_with_gaps(lib):
    """split_stride > M * ldd and ldd > N: each slab lands at its own offset; the gaps between slabs and the columns past N
    are never written."""
    torch.manual_seed(11)
    M, N, K, ldd = 300, 520, 4096, 536
    stride = M * ldd + 1000  # a multiple of 4 elements
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (0.05 * torch.randn(N, K, device="cuda")).to(torch.bfloat16)
    n_split = lib.vdk_gemm_effective_splits(K, 8)
    buf = torch.full((n_split * stride,), float("nan"), device="cuda")
    g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=buf.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=ldd,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0, beta=0,
                      residual=0, ldr=0, ln_eps=0.0, split_k=8, split_stride=stride, trans_a=0, trans_b=0)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    slabs = torch.stack([buf[s * stride: s * stride + M * ldd].view(M, ldd) for s in range(n_split)])
    assert torch.isfinite(slabs[:, :, :N]).all(), "a slab element inside [M, N] was not written"
    assert torch.isnan(slabs[:, :, N:]).all(), "a slab column past N was written"
    for s in range(n_split):
        assert torch.isnan(buf[s * stride + M * ldd: (s + 1) * stride]).all(), f"the gap after slab {s} was written"
    ref, bound = split_k_bound(a, w, n_split)
    check_within(slabs[:, :, :N].sum(0), ref, bound, "split-K slabs with gaps", describe_tiles(M, N, tile_n(N, E.EPI_NONE)))


def test_gemm_split_k_atomics_ragged_m(lib):
    """Atomic split-K (TMA reduce-add into a zeroed D) with M % 128 <= 64 and ldd > N: rows past M and columns past N
    stay untouched."""
    torch.manual_seed(12)
    M, N, K, ldd = 256 + 40, 512, 6144, 520
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (0.05 * torch.randn(N, K, device="cuda")).to(torch.bfloat16)
    d = torch.zeros(M + 1, ldd, device="cuda")
    d[:, N:] = float("nan")
    d[M:] = float("nan")
    g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=ldd,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0, beta=0,
                      residual=0, ldr=0, ln_eps=0.0, split_k=12, split_stride=0, trans_a=0, trans_b=0)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    assert torch.isnan(d[:, N:]).all() and torch.isnan(d[M:]).all(), "atomic split-K wrote outside [M, N]"
    ref, bound = split_k_bound(a, w, lib.vdk_gemm_effective_splits(K, 12))
    check_within(d[:M, :N], ref, bound, "split-K atomics, ragged M", describe_tiles(M, N, tile_n(N, E.EPI_NONE)))
