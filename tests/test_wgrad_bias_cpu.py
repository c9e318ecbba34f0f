"""Argument checks of vdk_gemm's `a_col_sums` output (the bias gradient of the weight-gradient form); no GPU needed: the
descriptor is rejected before any device work."""
import ctypes as C

from visiondk_b200 import _lib


def desc(trans_a, split_k, split_stride, col_sums):
    # placeholder 256-aligned addresses: validation reads no operand memory
    return _lib.GemmDesc(A=256, B=256, D=256, M=128, N=128, K=256, lda=128 if trans_a else 256, ldb=128, ldd=128,
                         in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, split_k=split_k,
                         split_stride=split_stride, trans_a=trans_a, trans_b=1, a_col_sums=col_sums)


def test_col_sums_need_the_mn_major_split_k_slab_form(lib):
    for ta, split, stride, cs in ((0, 2, 128 * 128, 512), (1, 1, 0, 512), (1, 2, 0, 512), (1, 2, 128 * 128, 516)):
        g = desc(ta, split, stride, cs)
        assert lib.vdk_gemm(C.byref(g), None) == _lib.VDK_ERR_INVALID, (ta, split, stride, cs)
        assert "a_col_sums" in _lib.last_error()
