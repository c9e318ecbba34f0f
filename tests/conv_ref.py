"""fp64 reference and elementwise error bound of the dense convolution (vdk_conv2d): y = epilogue(conv(x, w) + bias) on
NHWC bf16, w [Cout, k, k, Cin].  Test infrastructure shared by tests/test_conv_gpu.py."""
import torch
import torch.nn.functional as F

from kernel_ref import ulp


def conv_reference(x, w, stride, pad):
    """fp64 conv2d of the bf16 operands x [B, H, W, Cin], w [Cout, k, k, Cin] -> (out, sum of |terms|), both [B, Ho, Wo, Cout]."""
    xd, wd = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
    out = F.conv2d(xd, wd, stride=stride, padding=pad).permute(0, 2, 3, 1)
    mag = F.conv2d(xd.abs(), wd.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    return out, mag


def conv_bound(acc, mag, K, bias, residual, out_ref):
    """Elementwise bound of vdk_conv2d: the wgmma GEMM's fp32 accumulation (ceil(K/16) + 17) 2^-23 (|x| * |w|), one fp32
    rounding (2^-24 relative) per epilogue operation (+ bias, + residual), then one bf16 ulp of the output.  ReLU is exact
    and 1-Lipschitz."""
    e = (-(-K // 16) + 17) * 2.0 ** -23 * mag
    pre = acc.abs() + e
    if bias is not None:
        pre = pre + bias.double().abs()
        e = e + 2.0 ** -24 * pre
    if residual is not None:
        pre = pre + residual.double().abs()
        e = e + 2.0 ** -24 * pre
    return e + ulp(out_ref.abs() + e, torch.bfloat16)
