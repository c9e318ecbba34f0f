"""GPU parity of vdk_gemm_tn (wgmma/TMA GEMM) against a plain fp32 torch reference of the same op.

Inputs are drawn already rounded to the 16-bit input type, so the only differences are the fp32
accumulation order (tolerance 2e-3 relative to the row scale) and, for 16-bit outputs, one final rounding.
"""
import pytest
import torch

from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu

DT = {"bf16": (torch.bfloat16, _lib.DTYPE_BF16), "fp16": (torch.float16, _lib.DTYPE_FP16),
      "fp32": (torch.float32, _lib.DTYPE_FP32)}


def run_gemm(a, b, out_dtype, epilogue=_lib.EPI_NONE, bias=None, gamma=None, residual=None):
    lib = _lib.load()
    M, K = a.shape
    N = b.shape[0]
    d = torch.full((M, N), float("nan"), dtype=DT[out_dtype][0], device=a.device)
    in_code = _lib.DTYPE_BF16 if a.dtype == torch.bfloat16 else _lib.DTYPE_FP16
    rc = lib.vdk_gemm_tn(a.data_ptr(), b.data_ptr(), d.data_ptr(), M, N, K, a.stride(0), b.stride(0), d.stride(0),
                         in_code, DT[out_dtype][1], epilogue, _lib.ptr(bias), _lib.ptr(gamma), _lib.ptr(residual),
                         residual.stride(0) if residual is not None else 0, _lib.stream_ptr())
    _lib.check(rc, "vdk_gemm_tn")
    torch.cuda.synchronize()
    return d


def describe_mismatch(got, ref, tol):
    bad = (got.float() - ref).abs() > tol
    idx = bad.nonzero()
    rows = idx[:, 0]
    cols = idx[:, 1]
    return (f"{int(bad.sum())}/{bad.numel()} wrong; rows%8 hist {torch.bincount(rows % 8, minlength=8).tolist()} "
            f"cols%8 hist {torch.bincount(cols % 8, minlength=8).tolist()} "
            f"row tiles {torch.unique(rows // 128).tolist()[:8]} col tiles {torch.unique(cols // 128).tolist()[:8]} "
            f"first {idx[:4].tolist()} got {got[bad][:4].tolist()} ref {ref[bad][:4].tolist()} nan {int(torch.isnan(got.float()).sum())}")


@pytest.mark.parametrize("in_dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 256, 64), (128, 128, 256), (256, 512, 128),
                                   (1000, 384, 200), (300, 1000, 512), (4096, 512, 128), (77, 8, 8),
                                   (20000, 1024, 256)])
def test_gemm_plain_fp32_out(lib, in_dtype, M, N, K):
    torch.manual_seed(M * 7 + N * 3 + K)
    dt = DT[in_dtype][0]
    a = torch.randn(M, K, device="cuda").to(dt)
    b = torch.randn(N, K, device="cuda").to(dt)
    ref = a.float() @ b.float().t()
    got = run_gemm(a, b, "fp32")
    tol = 2e-3 * (K ** 0.5)
    assert torch.isfinite(got).all(), describe_mismatch(got, ref, tol)
    assert (got - ref).abs().max().item() <= tol, describe_mismatch(got, ref, tol)


def test_gemm_exact_small_integers(lib):
    # integer-valued operands: every product and partial sum is exact, so the result must be bit-exact
    torch.manual_seed(0)
    a = torch.randint(-4, 5, (256, 192), device="cuda").to(torch.bfloat16)
    b = torch.randint(-4, 5, (384, 192), device="cuda").to(torch.bfloat16)
    ref = a.float() @ b.float().t()
    got = run_gemm(a, b, "fp32")
    assert torch.equal(got, ref), describe_mismatch(got, ref, 0.0)


def test_gemm_strided_operands(lib):
    torch.manual_seed(1)
    abuf = torch.randn(500, 320, device="cuda").to(torch.bfloat16)
    bbuf = torch.randn(264, 448, device="cuda").to(torch.bfloat16)
    a, b = abuf[:, :256], bbuf[:, 64:320]  # pitches 320 / 448, 16-byte aligned starts
    ref = a.float() @ b.float().t()
    got = run_gemm(a, b, "fp32")
    assert (got - ref).abs().max().item() <= 2e-3 * 16, describe_mismatch(got, ref, 2e-3 * 16)


@pytest.mark.parametrize("out_dtype", ["bf16", "fp32"])
def test_gemm_bias_gelu(lib, out_dtype):
    torch.manual_seed(2)
    M, N, K = 1568, 512, 128
    a = (0.5 * torch.randn(M, K, device="cuda")).to(torch.bfloat16)
    b = (0.2 * torch.randn(N, K, device="cuda")).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    ref = torch.nn.functional.gelu(a.float() @ b.float().t() + bias)
    got = run_gemm(a, b, out_dtype, _lib.EPI_GELU, bias=bias).float()
    # the epilogue's GELU is a half-precision tanh form fitted to erf-GELU: |err| <= 1.2e-3 |x| (gemm.cu), |x| < ~6 here
    tol = 3e-2 if out_dtype == "bf16" else 8e-3
    assert (got - ref).abs().max().item() <= tol, describe_mismatch(got, ref, tol)


@pytest.mark.parametrize("out_dtype", ["bf16", "fp32"])
def test_gemm_layerscale_residual(lib, out_dtype):
    torch.manual_seed(3)
    M, N, K = 784, 256, 1024
    a = (0.3 * torch.randn(M, K, device="cuda")).to(torch.bfloat16)
    b = (0.1 * torch.randn(N, K, device="cuda")).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    gamma = torch.rand(N, device="cuda")
    res = torch.randn(M, N, device="cuda").to(DT[out_dtype][0])
    ref = res.float() + gamma * (a.float() @ b.float().t() + bias)
    got = run_gemm(a, b, out_dtype, _lib.EPI_SCALE_RESIDUAL, bias=bias, gamma=gamma, residual=res).float()
    tol = 4e-2 if out_dtype == "bf16" else 3e-3
    assert (got - ref).abs().max().item() <= tol, describe_mismatch(got, ref, tol)


def test_gemm_rejects_bad_arguments(lib):
    a = torch.zeros(8, 8, device="cuda", dtype=torch.bfloat16)
    d = torch.zeros(8, 8, device="cuda")
    rc = lib.vdk_gemm_tn(a.data_ptr(), a.data_ptr(), d.data_ptr(), 8, 7, 8, 8, 8, 8, 0, 2, 0, 0, 0, 0, 0, 0)
    assert rc == _lib.VDK_ERR_INVALID and "multiple of 8" in _lib.last_error()


@pytest.mark.parametrize("ta,tb", [(1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 192), (512, 2048, 50176 // 49), (1000, 384, 200), (2048, 512, 3000)])
def test_gemm_transposed_storage(lib, ta, tb, M, N, K):
    """MN-major operands (contraction index slow): the forms the backward GEMMs use (dgrad: trans_b, wgrad: both)."""
    import ctypes as C
    torch.manual_seed(M + N + K + ta * 2 + tb)
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    ref = a.float() @ b.float().t()
    a_st = a.t().contiguous() if ta else a          # [K, M] storage when transposed
    b_st = b.t().contiguous() if tb else b          # [K, N]
    d = torch.full((M, N), float("nan"), device="cuda")
    g = _lib.GemmDesc(A=a_st.data_ptr(), B=b_st.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=a_st.stride(0),
                      ldb=b_st.stride(0), ldd=N, in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE,
                      bias=0, gamma=0, beta=0, residual=0, ldr=0, ln_eps=0.0, split_k=1, trans_a=ta, trans_b=tb)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    tol = 2e-3 * K ** 0.5
    assert torch.isfinite(d).all(), describe_mismatch(d, ref, tol)
    assert (d - ref).abs().max().item() <= tol, describe_mismatch(d, ref, tol)


def test_gemm_wgrad_form_split_k(lib):
    """dW[N_out, K_in] = dY^T . X with the token index (M = 50k) as the contraction: both operands MN-major, split-K."""
    import ctypes as C
    torch.manual_seed(9)
    tokens, n_out, k_in = 50176, 512, 256
    dy = (0.1 * torch.randn(tokens, n_out, device="cuda")).to(torch.bfloat16)
    x = torch.randn(tokens, k_in, device="cuda").to(torch.bfloat16)
    ref = dy.float().t() @ x.float()
    d = torch.zeros(n_out, k_in, device="cuda")
    g = _lib.GemmDesc(A=dy.data_ptr(), B=x.data_ptr(), D=d.data_ptr(), M=n_out, N=k_in, K=tokens, lda=n_out, ldb=k_in,
                      ldd=k_in, in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0,
                      beta=0, residual=0, ldr=0, ln_eps=0.0, split_k=37, trans_a=1, trans_b=1)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    assert (d - ref).abs().max().item() <= 2e-3 * tokens ** 0.5 * 0.1 + 1e-2, describe_mismatch(d, ref, 0.05)


def test_gemm_split_k_slabs_are_deterministic(lib):
    """split_stride > 0: every split writes its own slab (no atomics); the slab sum is bitwise reproducible."""
    import ctypes as C
    torch.manual_seed(4)
    M, N, K = 200, 512, 12544
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (0.05 * torch.randn(N, K, device="cuda")).to(torch.bfloat16)
    n_split = lib.vdk_gemm_effective_splits(K, 40)
    outs = []
    for _ in range(2):
        d = torch.full((n_split, M, N), float("nan"), device="cuda")
        g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=N,
                          in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0, beta=0,
                          residual=0, ldr=0, ln_eps=0.0, split_k=40, split_stride=M * N, trans_a=0, trans_b=0)
        _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
        torch.cuda.synchronize()
        assert torch.isfinite(d).all()
        outs.append(d.sum(0))
    assert torch.equal(outs[0], outs[1])
    ref = a.float() @ w.float().t()
    assert (outs[0] - ref).abs().max().item() <= 2e-3 * K ** 0.5 * 0.05 + 1e-3
