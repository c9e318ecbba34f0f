"""vdk_conv2d (implicit-GEMM convolution on the wgmma GEMM, csrc/gemm.cu) against an fp64 convolution of the same bf16
inputs, elementwise, within tests/conv_ref.conv_bound: 1x1 (plain GEMM) and k x k / stride-s (TMA im2col A tiles) shapes,
every ResNet-50 / Wide-ResNet stage shape, ragged maps, M tiles that cross image boundaries, zero padding under large inputs,
residuals in and out of place, NaN-guarded outputs, and batches that give every persistent CTA at least 3 tiles."""
import ctypes as C

import pytest
import torch

from conv_ref import conv_bound, conv_reference
from kernel_ref import Guarded, check_within
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu

RELU, RES_RELU, NONE = _lib.EPI_RELU, _lib.EPI_RESIDUAL_RELU, _lib.EPI_NONE


def run_conv(lib, x, w, bias, k, stride, pad, epi, residual=None, inplace=False, x_scale=None):
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    M = B * Ho * Wo
    y = Guarded(M, Cout, Cout, torch.bfloat16)
    res_ptr = 0
    if residual is not None:
        if inplace:
            y.fill_(residual.reshape(M, Cout))
            res_ptr = y.ptr()
        else:
            res_ptr = residual.data_ptr()
    d = _lib.ConvDesc(x=x.data_ptr(), w=w.data_ptr(), bias=_lib.ptr(bias), residual=res_ptr, y=y.ptr(), B=B, H=H, W=W, Cin=Cin,
                      Cout=Cout, kernel=k, stride=stride, pad=pad, epilogue=epi)
    _lib.check(lib.vdk_conv2d(C.byref(d), _lib.stream_ptr()), "vdk_conv2d")
    torch.cuda.synchronize()
    return y, (B, Ho, Wo, Cout)


def check_conv(lib, x, w, bias, k, stride, pad, epi, residual=None, inplace=False, name="conv"):
    y, shape = run_conv(lib, x, w, bias, k, stride, pad, epi, residual, inplace)
    acc, mag = conv_reference(x, w, stride, pad)
    ref = acc + (bias.double() if bias is not None else 0.0)
    if residual is not None:
        ref = ref + residual.double()
    if epi != NONE:
        ref = ref.clamp_min(0.0)
    bound = conv_bound(acc, mag, k * k * x.shape[3], bias, residual, ref)
    got = y.view.reshape(shape)
    B, Ho, Wo, _ = shape

    def describe(bad):
        pix = bad.reshape(-1, shape[3]).any(dim=1).nonzero().flatten()
        return f"output pixels {pix[:8].tolist()} (tile rows {sorted(set((pix // 128).tolist()))[:8]}; Ho*Wo = {Ho * Wo})"

    check_within(got, ref, bound, name, describe)
    assert y.guard_errors() == "", y.guard_errors()
    return got, ref


def make(B, H, W, Cin, Cout, k, seed, scale=1.0, positive=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g) * scale
    if positive:
        x = x.abs()
    w = torch.randn(Cout, k, k, Cin, device="cuda", generator=g) * (2.0 / (k * k * Cin)) ** 0.5
    bias = 0.1 * torch.randn(Cout, device="cuda", generator=g)
    return x.to(torch.bfloat16), w.to(torch.bfloat16), bias


CASES = [
    # B, H, W, Cin, Cout, k, stride, pad, epilogue
    (2, 14, 14, 64, 256, 1, 1, 0, RELU),
    (2, 15, 15, 256, 512, 1, 2, 0, NONE),
    (2, 14, 14, 128, 128, 3, 1, 1, RELU),
    (2, 9, 13, 64, 72, 3, 2, 1, RELU),      # ragged odd map at stride 2, Cout not a multiple of the N tile
    (3, 7, 5, 2048, 520, 1, 1, 0, RELU),    # Cin 2048, Cout 520 (two 256-wide tiles + a ragged one)
    (2, 10, 10, 1024, 264, 3, 2, 1, NONE),
    (2, 14, 14, 512, 1024, 2, 2, 0, NONE),  # the ResNet-D shortcut: AvgPool2d(2, 2) + 1x1 folded into a 2x2/s2 conv
    (1, 3, 3, 64, 64, 3, 1, 1, RELU),       # a map smaller than the filter window
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,pad,epi", CASES)
def test_conv_shapes(lib, B, H, W, Cin, Cout, k, stride, pad, epi):
    x, w, bias = make(B, H, W, Cin, Cout, k, seed=Cin + Cout + k)
    check_conv(lib, x, w, bias, k, stride, pad, epi, name=f"conv {B}x{H}x{W}x{Cin}->{Cout} k{k}s{stride}")


def resnet_stage_shapes(base_width, size=224):
    """Every distinct conv of a Bottleneck ResNet-50 at `size` (base_width 64) or its wide variant (128):
    (H, Cin, Cout, k, stride, pad, epilogue)."""
    shapes, inplanes, h = set(), 64, size // 4
    for i, planes in enumerate((64, 128, 256, 512)):
        stride, width, out = (1 if i == 0 else 2), planes * base_width // 64, planes * 4
        for j in range(2):  # the first block and a repeated block
            s = stride if j == 0 else 1
            shapes.add((h, inplanes, width, 1, 1, 0, RELU))
            shapes.add((h, width, width, 3, s, 1, RELU))
            shapes.add((h // s, width, out, 1, 1, 0, RES_RELU))
            if j == 0:
                shapes.add((h, inplanes, out, 1, s, 0, NONE))
                if s == 2:
                    shapes.add((h, inplanes, out, 2, 2, 0, NONE))
            h, inplanes = h // s, out
    return sorted(shapes)


@pytest.mark.parametrize("base_width", [64, 128])
def test_conv_resnet_stage_shapes(lib, base_width):
    for n, (h, cin, cout, k, s, p, epi) in enumerate(resnet_stage_shapes(base_width)):
        x, w, bias = make(2, h, h, cin, cout, k, seed=n)
        Ho = (h + 2 * p - k) // s + 1
        res = None
        if epi == RES_RELU:
            res = torch.randn(2, Ho, Ho, cout, device="cuda").to(torch.bfloat16)
        check_conv(lib, x, w, bias, k, s, p, epi, residual=res, name=f"wide{base_width} {h}x{h}x{cin}->{cout} k{k}s{s}")


@pytest.mark.parametrize("k,stride,pad", [(3, 1, 1), (3, 2, 1), (1, 2, 0), (1, 1, 0)])
def test_conv_tiles_cross_image_boundaries(lib, k, stride, pad):
    """81 output pixels per image (9x9 at stride 1): 128-row tiles straddle images.  The images differ by 10^4 in magnitude,
    so an input pixel gathered from the neighbouring image is far outside the bound."""
    x, w, bias = make(5, 9 * stride, 9 * stride, 128, 64, k, seed=7)
    mags = torch.tensor([1.0, 100.0, 0.01, 30.0, 0.3], device="cuda").view(5, 1, 1, 1)
    x = (x.float() * mags).to(torch.bfloat16)
    check_conv(lib, x, w, bias, k, stride, pad, NONE, name=f"cross-image k{k}s{stride}")


@pytest.mark.parametrize("stride", [1, 2])
def test_conv_zero_padding_under_large_inputs(lib, stride):
    """Large positive inputs and weights: a border tap that read anything but zero would move the output by ~100 x bound."""
    x, w, bias = make(2, 8, 8, 64, 128, 3, seed=11, scale=40.0, positive=True)
    w = w.float().abs().to(torch.bfloat16)
    check_conv(lib, x, w, bias, 3, stride, 1, NONE, name=f"padding s{stride}")


@pytest.mark.parametrize("inplace", [False, True])
def test_conv_residual_relu(lib, inplace):
    x, w, bias = make(3, 14, 14, 256, 512, 1, seed=5)
    res = torch.randn(3, 14, 14, 512, device="cuda").to(torch.bfloat16)
    check_conv(lib, x, w, bias, 1, 1, 0, RES_RELU, residual=res, inplace=inplace, name=f"residual inplace={inplace}")
    x, w, bias = make(2, 9, 9, 64, 256, 3, seed=6)
    res = torch.randn(2, 9, 9, 256, device="cuda").to(torch.bfloat16)
    check_conv(lib, x, w, bias, 3, 1, 1, RES_RELU, residual=res, inplace=inplace, name=f"3x3 residual inplace={inplace}")


@pytest.mark.parametrize("k,stride,pad,cout", [(3, 1, 1, 64), (3, 2, 1, 256), (1, 1, 0, 128)])
def test_conv_every_cta_runs_three_tiles(lib, k, stride, pad, cout):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bn = 256 if cout % 256 == 0 else 128
    n_tiles = -(-cout // bn)
    H = 14 * stride
    B = -(-3 * sms * 128 // (n_tiles * 14 * 14)) + 1  # M = B * 14 * 14 rows: >= 3 tiles for every CTA of the persistent grid
    x, w, bias = make(B, H, H, 64, cout, k, seed=B)
    got, _ = check_conv(lib, x, w, bias, k, stride, pad, RELU, name=f"persistent k{k}s{stride} B{B}")
    assert -(-got.shape[0] * 14 * 14 // 128) * n_tiles >= 3 * sms
