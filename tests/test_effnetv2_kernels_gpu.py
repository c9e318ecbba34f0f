"""The EfficientNetV2 building blocks against fp64 references of the same bf16 / fp32 inputs, elementwise within bounds
derived from their roundings:
  vdk_conv2d_ex     TF-"same" (0, 1) / (1, 1) / (0, 0) padding, Cin 24 / 32 / 48 / 80 / 96 and multiples of 64, the NONE /
                    SILU / SILU_RESIDUAL epilogues, ragged M tiles that cross images and ragged / wide N tiles
  vdk_dwconv3_silu  stride 1 and 2 on even and odd maps, C 32 .. 3840, batch 256 at 56^2 / 14^2 / 7^2; its SE mean, and
                    that mean bit-identical across launches
  vdk_effnet_se     the SiLU / sigmoid excitation and the gate applied in place, then the gated projection GEMM."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from conv_ref import conv_bound
from kernel_ref import Guarded, check_within, ulp
from visiondk_b200 import _lib
from visiondk_b200.efficientnet import ConvExDesc, pack_conv_ex

pytestmark = pytest.mark.gpu

NONE, SILU, SILU_RES = _lib.EPI_NONE, _lib.EPI_SILU, _lib.EPI_SILU_RESIDUAL


def same(size, k, s):
    total = max((math.ceil(size / s) - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def run_conv_ex(lib, x, w, bias, k, stride, pads, epi, residual=None):
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    (ht, hb), (wl, wr) = pads
    Ho, Wo = (H + ht + hb - k) // stride + 1, (W + wl + wr - k) // stride + 1
    wp = pack_conv_ex(w.permute(0, 3, 1, 2).float()).to(torch.bfloat16).contiguous()
    y = Guarded(B * Ho * Wo, Cout, Cout, torch.bfloat16)
    d = ConvExDesc(x=x.data_ptr(), w=wp.data_ptr(), bias=_lib.ptr(bias), residual=_lib.ptr(residual), y=y.ptr(), B=B, H=H, W=W,
                   Cin=Cin, Cout=Cout, kernel=k, stride=stride, pad_h_lo=ht, pad_h_hi=hb, pad_w_lo=wl, pad_w_hi=wr, epilogue=epi)
    _lib.check(lib.vdk_conv2d_ex(C.byref(d), _lib.stream_ptr()), "vdk_conv2d_ex")
    torch.cuda.synchronize()
    return y, (B, Ho, Wo, Cout)


CONV_CASES = [  # (B, H, W, Cin, Cout, k, stride, padding)
    (3, 9, 9, 24, 24, 3, 1, "same"),     # stage 0 of S / M: (1, 1), 243 rows: tiles cross images, ragged N
    (2, 16, 16, 32, 32, 3, 1, "same"),   # stage 0 of L
    (2, 16, 16, 32, 128, 3, 2, "same"),  # conv_exp s2 on an even map: (0, 1)
    (3, 10, 10, 48, 192, 3, 2, "same"),  # (0, 1), 75 rows
    (2, 8, 8, 80, 320, 3, 1, "same"),    # Cin 80: two K blocks per tap, the second mostly zero fill
    (2, 9, 9, 96, 384, 3, 2, "same"),    # odd map at stride 2: (1, 1)
    (2, 12, 12, 64, 256, 3, 2, "same"),  # Cin a multiple of 64, BN = 256
    (2, 7, 7, 128, 640, 3, 1, "same"),   # N > 512
    (3, 7, 7, 24, 40, 1, 1, "none"),     # 1x1: plain GEMM with K = 24 < 64, (0, 0)
    (2, 7, 7, 96, 1280, 1, 1, "none"),   # conv_head-like
    (2, 9, 9, 32, 64, 3, 1, "none"),     # 3x3 without padding (0, 0)
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("epi", [NONE, SILU, SILU_RES])
def test_conv2d_ex_matches_fp64(lib, case, epi):
    B, H, W, Cin, Cout, k, stride, padding = case
    pads = (same(H, k, stride), same(W, k, stride)) if padding == "same" else ((0, 0), (0, 0))
    g = torch.Generator(device="cuda").manual_seed(Cin * 131 + Cout + k + epi)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, device="cuda", generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16)
    bias = 0.1 * torch.randn(Cout, device="cuda", generator=g)
    (ht, hb), (wl, wr) = pads
    Ho, Wo = (H + ht + hb - k) // stride + 1, (W + wl + wr - k) // stride + 1
    residual = None
    if epi == SILU_RES:
        residual = torch.randn(B, Ho, Wo, Cout, device="cuda", generator=g).to(torch.bfloat16)
    y, shape = run_conv_ex(lib, x, w, bias, k, stride, pads, epi, residual)
    xd = F.pad(x.double().permute(0, 3, 1, 2), (wl, wr, ht, hb))
    wd = w.double().permute(0, 3, 1, 2)
    acc = F.conv2d(xd, wd, stride=stride).permute(0, 2, 3, 1)
    mag = F.conv2d(xd.abs(), wd.abs(), stride=stride).permute(0, 2, 3, 1)
    pre = acc + bias.double()
    ref = pre if epi == NONE else F.silu(pre)
    if residual is not None:
        ref = ref + residual.double()
    # conv_bound covers the accumulation, the bias and residual additions and the output rounding; SiLU is 1.1-Lipschitz
    # and its fast form adds 1e-6 relative
    bound = conv_bound(acc, mag, k * k * Cin, bias, residual, ref)
    if epi != NONE:
        bound = 1.1 * bound + 1e-6 * pre.abs() + 2.0 ** -24 * (ref.abs() + pre.abs())
    got = y.view.reshape(shape)
    check_within(got, ref, bound, f"conv_ex {case} epi {epi}", lambda bad: f"{int(bad.sum())} elements")
    assert y.guard_errors() == "", y.guard_errors()


def test_conv2d_ex_rejects_bad_arguments(lib):
    d = ConvExDesc(x=16, w=16, y=16, B=1, H=8, W=8, Cin=12, Cout=16, kernel=3, stride=1, pad_h_lo=1, pad_h_hi=1, pad_w_lo=1,
                   pad_w_hi=1, epilogue=SILU)
    assert lib.vdk_conv2d_ex(C.byref(d), 0) == _lib.VDK_ERR_INVALID and "multiple of 8" in _lib.last_error()
    d.Cin, d.pad_h_hi = 16, 3
    assert lib.vdk_conv2d_ex(C.byref(d), 0) == _lib.VDK_ERR_INVALID
    d.pad_h_hi, d.epilogue = 1, _lib.EPI_RELU
    assert lib.vdk_conv2d_ex(C.byref(d), 0) == _lib.VDK_ERR_INVALID


def dw_reference(x, w9, b, stride):
    """fp64: pre = depthwise conv (TF-same) + b, mag = the same over |x| |w|."""
    B, H, W, Cc = x.shape
    (ht, hb), (wl, wr) = same(H, 3, stride), same(W, 3, stride)
    xd = F.pad(x.double().permute(0, 3, 1, 2), (wl, wr, ht, hb))
    wd = w9.double().t().reshape(Cc, 1, 3, 3)
    pre = F.conv2d(xd, wd, stride=stride, groups=Cc).permute(0, 2, 3, 1) + b.double()
    mag = F.conv2d(xd.abs(), wd.abs(), stride=stride, groups=Cc).permute(0, 2, 3, 1) + b.double().abs()
    return pre, mag


def run_dw(lib, x, w9, b, stride):
    B, H, W, Cc = x.shape
    Ho, Wo = -(-H // stride), -(-W // stride)
    y = torch.empty(B, Ho, Wo, Cc, device="cuda", dtype=torch.bfloat16)
    mean = torch.empty(B, Cc, device="cuda")
    _lib.check(lib.vdk_dwconv3_silu(x.data_ptr(), B, H, W, Cc, stride, w9.data_ptr(), b.data_ptr(), y.data_ptr(), mean.data_ptr(),
                                    _lib.stream_ptr()), "vdk_dwconv3_silu")
    torch.cuda.synchronize()
    return y, mean


DW_CASES = [  # (B, H, W, C, stride)
    (2, 9, 9, 32, 1), (2, 9, 9, 64, 2), (2, 8, 8, 96, 2), (3, 14, 14, 384, 2), (2, 7, 7, 3840, 1), (2, 5, 11, 160, 2),
    (256, 56, 56, 64, 1), (256, 14, 14, 1152, 1), (256, 7, 7, 3840, 1), (256, 14, 14, 1344, 2),
]


@pytest.mark.parametrize("case", DW_CASES)
def test_dwconv3_silu_matches_fp64(lib, case):
    B, H, W, Cc, stride = case
    g = torch.Generator(device="cuda").manual_seed(B + H * 7 + Cc)
    x = torch.randn(B, H, W, Cc, device="cuda", generator=g).to(torch.bfloat16)
    w9 = torch.randn(9, Cc, device="cuda", generator=g) / 3.0
    b = 0.1 * torch.randn(Cc, device="cuda", generator=g)
    y, mean = run_dw(lib, x, w9, b, stride)
    pre, mag = dw_reference(x, w9, b, stride)
    ref = F.silu(pre)
    # fp32 FMAs over 10 terms: 10 * 2^-24 * mag; SiLU (1.1-Lipschitz) with __expf and one division: 4e-7 |pre| + 2^-23 |ref|;
    # then the bf16 rounding of the output
    e = 1.1 * 10 * 2.0 ** -24 * mag + 4e-7 * pre.abs() + 2.0 ** -23 * ref.abs()
    bound = e + ulp(ref.abs() + e, torch.bfloat16)
    check_within(y, ref, bound, f"dwconv3 {case}", lambda bad: f"{int(bad.sum())} elements")
    # the mean is an fp32 sum of the stored bf16 outputs in a fixed order: within HW 2^-24 of their fp64 sum
    HW = y.shape[1] * y.shape[2]
    yd = y.double().reshape(B, HW, Cc)
    mref = yd.mean(1)
    mbound = HW * 2.0 ** -24 * yd.abs().mean(1) + 2.0 ** -24 * mref.abs()
    assert bool(((mean.double() - mref).abs() <= mbound).all())
    y2, mean2 = run_dw(lib, x, w9, b, stride)
    assert torch.equal(mean, mean2) and torch.equal(y, y2)


@pytest.mark.parametrize("B,HW,Cc,rd", [(2, 49, 384, 24), (3, 196, 1152, 48), (256, 49, 3840, 160), (2, 1, 64, 16)])
def test_se_gate_and_gated_projection_match_fp64(lib, B, HW, Cc, rd):
    g = torch.Generator(device="cuda").manual_seed(B * HW + Cc)
    d = torch.randn(B, HW, Cc, device="cuda", generator=g).to(torch.bfloat16)
    mean = d.float().mean(1)
    w1 = torch.randn(rd, Cc, device="cuda", generator=g) / Cc ** 0.5
    b1 = 0.1 * torch.randn(rd, device="cuda", generator=g)
    w2 = torch.randn(Cc, rd, device="cuda", generator=g) / rd ** 0.5
    b2 = 0.1 * torch.randn(Cc, device="cuda", generator=g)
    gate = torch.empty(B, Cc, device="cuda")
    dg = d.clone()
    _lib.check(lib.vdk_effnet_se(dg.data_ptr(), mean.data_ptr(), B, HW, Cc, rd, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                 b2.data_ptr(), gate.data_ptr(), _lib.stream_ptr()), "vdk_effnet_se")
    torch.cuda.synchronize()
    h = mean.double() @ w1.double().t() + b1.double()
    s = F.silu(h)
    gref = torch.sigmoid(s @ w2.double().t() + b2.double())
    # fp32 dot products of C and rd terms (recursive summation: (n + 2) 2^-24 of the sum of |terms|), SiLU with expf and a
    # division (2^-21 relative, 1.1-Lipschitz), sigmoid (2^-21 absolute, 1/4-Lipschitz)
    hmag = mean.double().abs() @ w1.double().abs().t() + b1.double().abs()
    s_err = 1.1 * (Cc + 2) * 2.0 ** -24 * hmag + 2.0 ** -21 * s.abs()
    w2a = w2.double().abs().t()
    logit_err = (rd + 2) * 2.0 ** -24 * ((s.abs() + s_err) @ w2a + b2.double().abs()) + s_err @ w2a
    gbound = 0.25 * logit_err + 2.0 ** -21
    assert bool(((gate.double() - gref).abs() <= gbound).all()), float((gate.double() - gref).abs().max())
    ref = d.double() * gate.double()[:, None, :]
    check_within(dg, ref, ulp(ref.abs(), torch.bfloat16), "se gate apply", lambda bad: f"{int(bad.sum())} elements")
    # the projection reads the gated d: vdk_gemm with the residual epilogue at gamma = 1
    cout = 64
    wp = (torch.randn(cout, Cc, device="cuda", generator=g) / Cc ** 0.5).to(torch.bfloat16)
    bp = 0.1 * torch.randn(cout, device="cuda", generator=g)
    res = torch.randn(B * HW, cout, device="cuda", generator=g).to(torch.bfloat16)
    ones = torch.ones(cout, device="cuda")
    out = torch.empty(B * HW, cout, device="cuda", dtype=torch.bfloat16)
    _lib.check(lib.vdk_gemm_tn(dg.data_ptr(), wp.data_ptr(), out.data_ptr(), B * HW, cout, Cc, Cc, Cc, cout, _lib.DTYPE_BF16,
                               _lib.DTYPE_BF16, _lib.EPI_SCALE_RESIDUAL, bp.data_ptr(), ones.data_ptr(), res.data_ptr(), cout,
                               _lib.stream_ptr()), "vdk_gemm_tn")
    torch.cuda.synchronize()
    a = dg.double().reshape(B * HW, Cc)
    acc = a @ wp.double().t()
    pref = acc + bp.double() + res.double()
    mag = a.abs() @ wp.double().abs().t()
    e = (-(-Cc // 16) + 17) * 2.0 ** -23 * mag + 2.0 ** -23 * (pref.abs() + acc.abs() + 1)
    check_within(out, pref, e + ulp(pref.abs() + e, torch.bfloat16), "gated projection", lambda bad: f"{int(bad.sum())} elements")
