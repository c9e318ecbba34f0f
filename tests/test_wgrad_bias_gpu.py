"""GPU checks of the weight-gradient GEMM's bias output: with `a_col_sums`, the split-K slab form with an MN-major A (A stored
[K, M], the output gradient of a Linear layer) also stores, per split, the column sums sum_k A[k, m] of its K range.

The sums are of the 16-bit values as stored, in fp32: a thread adds every other row of a 4-column piece in order (at most
kb_per_split * 32 terms), then the two partials of a piece meet in one more addition.  The recursive-summation bound over n terms
is gamma_n sum |a| with gamma_n = n u / (1 - n u), u = 2^-24.  Outputs sit in NaN-guarded buffers: rows past the effective
number of splits and a tail past the last one must stay NaN.  The dW slabs must not change by a bit when the sums are
requested, and two runs must give the same sums bit for bit.
"""
import ctypes as C

import pytest
import torch

from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 64  # floats of NaN past the column-sum rows


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_wgrad(lib, a, b, split_k, col_sums):
    """D slabs [splits][M][N] of A^T B (A stored [K, M], B stored [K, N]); col_sums: None or a NaN-filled fp32 buffer"""
    K, M = a.shape
    N = b.shape[1]
    n_split = lib.vdk_gemm_effective_splits(K, split_k)
    d = torch.full((n_split, M, N), float("nan"), device="cuda")
    g = _lib.GemmDesc(A=a.data_ptr(), B=b.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=M, ldb=N, ldd=N,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0, beta=0,
                      residual=0, ldr=0, ln_eps=0.0, split_k=split_k, split_stride=M * N, aux_out=0, trans_a=1, trans_b=1,
                      a_col_sums=col_sums.data_ptr() if col_sums is not None else 0)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    return d


def split_ranges(K, n_split):
    """the contraction rows [k0, k1) of each split (gemm.cu: 64-row K blocks, ceil-divided over the splits)"""
    kbt = -(-K // 64)
    per = -(-kbt // n_split)
    return [(s * per * 64, min((s + 1) * per * 64, K)) for s in range(n_split)], per


# (M, N, K, split_k): tile width BN = 128 for N = 128, 256 for N % 256 == 0; M % 128 != 0; K % 64 != 0 (the last split's range
# ends inside a stage); two splits, and the most splits (one 64-row K block each); more work items than three per SM
CASES = [
    pytest.param(128, 128, 4096, 2, False, id="BN128-2splits"),
    pytest.param(200, 128, 1000, 2, False, id="BN128-raggedM-raggedK-2splits"),
    pytest.param(200, 128, 1000, 1 << 20, False, id="BN128-raggedM-raggedK-maxsplits"),
    pytest.param(136, 512, 3137, 2, False, id="BN256-raggedM-raggedK-2splits"),
    pytest.param(264, 256, 3137, 1 << 20, False, id="BN256-raggedM-raggedK-maxsplits"),
    pytest.param(1032, 512, 12544, 40, True, id="BN256-many-work-items"),
]


@pytest.mark.parametrize("M,N,K,split_k,many", CASES)
def test_wgrad_col_sums(lib, M, N, K, split_k, many):
    torch.manual_seed(M + N + K)
    a = (0.1 * torch.randn(K, M, device="cuda")).to(torch.bfloat16)
    b = torch.randn(K, N, device="cuda").to(torch.bfloat16)
    n_split = lib.vdk_gemm_effective_splits(K, split_k)
    if many:  # work items: M tiles x N tiles (BN = 256) x splits
        items = (-(-M // 128)) * (-(-N // 256)) * n_split
        assert items > 3 * sm_count(), (items, sm_count())

    d_plain = run_wgrad(lib, a, b, split_k, None)
    sums = []
    for _ in range(2):
        cs = torch.full((n_split * M + GUARD,), float("nan"), device="cuda")
        d = run_wgrad(lib, a, b, split_k, cs)
        assert torch.isfinite(d).all()
        # the dW slabs are the same bits with and without the column sums
        assert torch.equal(d.view(torch.int32), d_plain.view(torch.int32)), "dW slabs changed when the column sums were requested"
        assert torch.isnan(cs[n_split * M:]).all(), "column sums written past the last split"
        sums.append(cs[:n_split * M].view(n_split, M))
    assert torch.equal(sums[0].view(torch.int32), sums[1].view(torch.int32)), "column sums differ between two runs"

    got = sums[0].double()
    assert torch.isfinite(got).all(), "a column sum was not written"
    ranges, per = split_ranges(K, n_split)
    assert len(ranges) == n_split and ranges[-1][1] == K
    a64 = a.double()
    n = per * 32 + 1  # longest chain of fp32 additions behind one sum
    gamma = n * U / (1 - n * U)
    for s, (k0, k1) in enumerate(ranges):
        ref = a64[k0:k1].sum(0)
        bound = gamma * a64[k0:k1].abs().sum(0)
        err = (got[s] - ref).abs()
        bad = (err > bound).nonzero().flatten()
        assert bad.numel() == 0, (f"split {s} rows [{k0}, {k1}): {bad.numel()} columns out of bound, first m = {bad[0].item()}: "
                                  f"got {got[s, bad[0]].item()}, ref {ref[bad[0]].item()}, bound {bound[bad[0]].item()}")
    # and the whole K range, as the training step's bias gradient reduces it
    total = got.sum(0)
    assert ((total - a64.sum(0)).abs() <= (gamma + n_split * U) * a64.abs().sum(0) + 1e-30).all()

