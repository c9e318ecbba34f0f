"""The MobileNetV3 building blocks against fp64 references of the same bf16 / fp32 inputs, elementwise within bounds derived
from their roundings:
  vdk_dwconv_mnv3  every distinct depthwise shape of the six models at 224^2 (C, H, kernel, stride, activation, padding
                   rule, SE mean or not) at batch 2, the same at batch 256 for the widest grids and the pixel-split maps,
                   and ragged shapes (odd maps, widths that leave a CTA's channel vectors partly idle); its SE mean, and
                   the mean and output bit-identical across launches
  vdk_conv2d_ex    the HARDSWISH epilogue on the 1x1 (stem rows, expansion, CN, conv_head) and k x k paths (the public
                   entry keeps refusing RELU; the forward's internal launcher takes it, covered by the minimal models)
  vdk_mnv3_se      the ReLU / hard-sigmoid excitation and the gate applied in place
  vdk_gemm         the projections, K = the depthwise width (not a multiple of 64), with and without the shortcut."""
import math

import pytest
import torch
import torch.nn.functional as F

from conv_ref import conv_bound
from kernel_ref import check_within, ulp
from test_effnetv2_kernels_gpu import run_conv_ex
from visiondk_b200 import _lib
from visiondk_b200.mobilenetv3 import ACTS, MOBILENETV3_ARCHS, decode_blocks

pytestmark = pytest.mark.gpu

RELU, HSWISH = ACTS["relu"], ACTS["hard_swish"]
SAME, SYM = 0, 1


def pads(size, k, s, rule):
    if rule == SYM:
        return k // 2, k // 2
    total = max((math.ceil(size / s) - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def act_ref(v, act):
    return F.hardswish(v) if act == HSWISH else F.relu(v)


def model_dw_cases(size=224):
    """(C, H, kernel, stride, act, pad rule, with SE mean) of every depthwise conv of the six models."""
    cases = set()
    for spec in MOBILENETV3_ARCHS.values():
        H = size // 2
        for stage in decode_blocks(spec["arch"], spec["act"]):
            for kind, cin, cout, k, stride, mid, act, se_rd in stage:
                if kind != "cn":
                    cases.add((mid, H, k, stride, ACTS[act], 0 if spec["tf"] else 1, se_rd > 0))
                H = -(-H // stride)
    return sorted(cases)


def run_dw(lib, x, w, b, k, stride, rule, act, with_mean):
    B, H, W, Cc = x.shape
    (ht, hb), (wl, wr) = pads(H, k, stride, rule), pads(W, k, stride, rule)
    Ho, Wo = (H + ht + hb - k) // stride + 1, (W + wl + wr - k) // stride + 1
    y = torch.empty(B, Ho, Wo, Cc, device="cuda", dtype=torch.bfloat16)
    mean = torch.empty(B, Cc, device="cuda") if with_mean else None
    _lib.check(lib.vdk_dwconv_mnv3(x.data_ptr(), B, H, W, Cc, k, stride, rule, act, w.data_ptr(), b.data_ptr(), y.data_ptr(),
                                   _lib.ptr(mean), _lib.stream_ptr()), "vdk_dwconv_mnv3")
    torch.cuda.synchronize()
    return y, mean


def check_dw(lib, B, H, W, Cc, k, stride, act, rule, with_mean, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cc, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(k * k, Cc, device="cuda", generator=g) / k
    b = 0.1 * torch.randn(Cc, device="cuda", generator=g)
    y, mean = run_dw(lib, x, w, b, k, stride, rule, act, with_mean)
    (ht, hb), (wl, wr) = pads(H, k, stride, rule), pads(W, k, stride, rule)
    xd = F.pad(x.double().permute(0, 3, 1, 2), (wl, wr, ht, hb))
    wd = w.double().t().reshape(Cc, 1, k, k)
    pre = (F.conv2d(xd, wd, stride=stride, groups=Cc) + b.double().view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    mag = (F.conv2d(xd.abs(), wd.abs(), stride=stride, groups=Cc) + b.double().abs().view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    ref = act_ref(pre, act)
    # fp32 FMAs over k^2 + 1 terms: (k^2 + 1) 2^-24 mag, through an activation at most 1.5-Lipschitz (hard-swish); hard-swish's
    # own three roundings and its 1/6 constant: 2^-21 |ref|; then the bf16 rounding of the output
    e = 1.5 * (k * k + 1) * 2.0 ** -24 * mag + 2.0 ** -21 * ref.abs()
    check_within(y, ref, e + ulp(ref.abs() + e, torch.bfloat16), f"dwconv {(B, H, W, Cc, k, stride, act, rule)}",
                 lambda bad: f"{int(bad.sum())} elements")
    if with_mean:
        # the mean is an fp32 sum of the stored bf16 outputs in a fixed order: within HW 2^-24 of their fp64 sum
        HW = y.shape[1] * y.shape[2]
        yd = y.double().reshape(B, HW, Cc)
        mref = yd.mean(1)
        mbound = HW * 2.0 ** -24 * yd.abs().mean(1) + 2.0 ** -24 * mref.abs()
        assert bool(((mean.double() - mref).abs() <= mbound).all())
    y2, mean2 = run_dw(lib, x, w, b, k, stride, rule, act, with_mean)
    assert torch.equal(y, y2) and (mean is None or torch.equal(mean, mean2))


@pytest.mark.parametrize("case", model_dw_cases(), ids=str)
def test_dwconv_model_shapes_match_fp64(lib, case):
    Cc, H, k, stride, act, rule, se = case
    check_dw(lib, 2, H, H, Cc, k, stride, act, rule, se, seed=Cc * 7 + H + k)


@pytest.mark.parametrize("case", [
    (256, 112, 112, 16, 3, 1, RELU, SAME, False),   # large DS block: 2 channel vectors per image, split over the map
    (256, 112, 112, 16, 3, 2, RELU, SYM, True),     # small DS block with its SE mean: one CTA per image
    (256, 56, 56, 72, 5, 2, RELU, SAME, True),
    (256, 14, 14, 672, 5, 2, HSWISH, SAME, True),
    (256, 7, 7, 960, 5, 1, HSWISH, SYM, True),
    (256, 14, 14, 200, 3, 1, HSWISH, SAME, False),
], ids=str)
def test_dwconv_batch_256_matches_fp64(lib, case):
    B, H, W, Cc, k, stride, act, rule, se = case
    check_dw(lib, B, H, W, Cc, k, stride, act, rule, se, seed=B + Cc)


@pytest.mark.parametrize("case", [
    (3, 9, 9, 8, 3, 2, HSWISH, SAME, True),       # one channel vector, odd map: TF pads (1, 1)
    (2, 11, 7, 264, 3, 1, RELU, SYM, True),       # 33 vectors: two CTAs of 17 + 16
    (2, 13, 10, 40, 5, 2, HSWISH, SAME, True),    # odd / even axes at 5x5/s2: (2, 2) and (1, 2)
    (2, 5, 5, 4096, 5, 1, RELU, SAME, True),      # the widest width
    (1, 3, 3, 24, 5, 1, HSWISH, SYM, False),      # map smaller than the kernel's reach
    (4, 64, 64, 8, 5, 1, RELU, SAME, False),      # pixel-split with a ragged last range
], ids=str)
def test_dwconv_ragged_shapes_match_fp64(lib, case):
    B, H, W, Cc, k, stride, act, rule, se = case
    check_dw(lib, B, H, W, Cc, k, stride, act, rule, se, seed=H * W + Cc)


CONV_CASES = [  # (B, H, W, Cin, Cout, k, stride)
    (3, 16, 16, 64, 16, 1, 1),     # the stem's patch rows -> 16 channels
    (2, 14, 14, 80, 200, 1, 1),    # expansion, ragged M tile across images, ragged N
    (2, 7, 7, 160, 960, 1, 1),     # CN 1x1
    (2, 7, 7, 576, 1024, 1, 1),    # conv_head (small), with its bias
    (2, 9, 9, 24, 72, 3, 2),       # a padded k x k shape on the im2col path
]


@pytest.mark.parametrize("case", CONV_CASES, ids=str)
@pytest.mark.parametrize("epi", [_lib.EPI_HARDSWISH])
def test_conv2d_ex_hardswish_matches_fp64(lib, case, epi):
    B, H, W, Cin, Cout, k, stride = case
    pd = (pads(H, k, stride, SAME), pads(W, k, stride, SAME)) if k > 1 else ((0, 0), (0, 0))
    g = torch.Generator(device="cuda").manual_seed(Cin * 131 + Cout + epi)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, device="cuda", generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16)
    bias = 0.5 * torch.randn(Cout, device="cuda", generator=g)
    y, shape = run_conv_ex(lib, x, w, bias, k, stride, pd, epi)
    (ht, hb), (wl, wr) = pd
    xd = F.pad(x.double().permute(0, 3, 1, 2), (wl, wr, ht, hb))
    wd = w.double().permute(0, 3, 1, 2)
    acc = F.conv2d(xd, wd, stride=stride).permute(0, 2, 3, 1)
    mag = F.conv2d(xd.abs(), wd.abs(), stride=stride).permute(0, 2, 3, 1)
    pre = acc + bias.double()
    ref = act_ref(pre, ACTS["hard_swish"] if epi == _lib.EPI_HARDSWISH else ACTS["relu"])
    # conv_bound covers the accumulation, the bias addition and the output rounding; hard-swish is 1.5-Lipschitz and its
    # fp32 evaluation adds 2^-21 relative
    bound = 1.5 * conv_bound(acc, mag, k * k * Cin, bias, None, ref) + 2.0 ** -21 * ref.abs()
    check_within(y.view.reshape(shape), ref, bound, f"conv_ex {case} epi {epi}", lambda bad: f"{int(bad.sum())} elements")
    assert y.guard_errors() == "", y.guard_errors()


@pytest.mark.parametrize("B,HW,Cc,rd", [(2, 3136, 16, 8), (3, 784, 72, 24), (256, 49, 960, 240), (2, 196, 576, 144)])
def test_hard_sigmoid_se_matches_fp64(lib, B, HW, Cc, rd):
    g = torch.Generator(device="cuda").manual_seed(B * HW + Cc)
    d = torch.randn(B, HW, Cc, device="cuda", generator=g).to(torch.bfloat16)
    mean = torch.randn(B, Cc, device="cuda", generator=g)  # any mean: the excitation does not recompute it
    w1 = torch.randn(rd, Cc, device="cuda", generator=g) / Cc ** 0.5
    b1 = 0.1 * torch.randn(rd, device="cuda", generator=g)
    w2 = 8 * torch.randn(Cc, rd, device="cuda", generator=g) / rd ** 0.5  # logits spread over both clamps of the gate
    b2 = 0.1 * torch.randn(Cc, device="cuda", generator=g)
    gate = torch.empty(B, Cc, device="cuda")
    dg = d.clone()
    _lib.check(lib.vdk_mnv3_se(dg.data_ptr(), mean.data_ptr(), B, HW, Cc, rd, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                               b2.data_ptr(), gate.data_ptr(), _lib.stream_ptr()), "vdk_mnv3_se")
    torch.cuda.synchronize()
    h = F.relu(mean.double() @ w1.double().t() + b1.double())
    logit = h @ w2.double().t() + b2.double()
    gref = F.hardsigmoid(logit)
    assert 0 < float((gref == 0).double().mean()) + float((gref == 1).double().mean()) < 1
    # fp32 dot products of C and rd terms ((n + 2) 2^-24 of the sum of |terms|), ReLU exact, hard sigmoid 1/6-Lipschitz with
    # the + 3 and the division rounded (2^-23 relative)
    hmag = mean.double().abs() @ w1.double().abs().t() + b1.double().abs()
    h_err = (Cc + 2) * 2.0 ** -24 * hmag
    w2a = w2.double().abs().t()
    logit_err = (rd + 2) * 2.0 ** -24 * ((h + h_err) @ w2a + b2.double().abs()) + h_err @ w2a
    gbound = logit_err / 6 + 2.0 ** -23 * (gref.abs() + (logit.abs() + 3) / 6)
    assert bool(((gate.double() - gref).abs() <= gbound).all()), float((gate.double() - gref).abs().max())
    ref = d.double() * gate.double()[:, None, :]
    check_within(dg, ref, ulp(ref.abs(), torch.bfloat16), "se gate apply", lambda bad: f"{int(bad.sum())} elements")


@pytest.mark.parametrize("K", [16, 72, 88, 120, 184, 200, 240, 576])
@pytest.mark.parametrize("shortcut", [False, True])
def test_projection_with_k_not_a_multiple_of_64(lib, K, shortcut):
    M, N = 3 * 49 + 5, 40 if K != 16 else 16
    g = torch.Generator(device="cuda").manual_seed(K + shortcut)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    wp = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bp = 0.1 * torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16) if shortcut else None
    ones = torch.ones(N, device="cuda")
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    epi = _lib.EPI_SCALE_RESIDUAL if shortcut else _lib.EPI_NONE
    _lib.check(lib.vdk_gemm_tn(a.data_ptr(), wp.data_ptr(), out.data_ptr(), M, N, K, K, K, N, _lib.DTYPE_BF16, _lib.DTYPE_BF16, epi,
                               bp.data_ptr(), ones.data_ptr() if shortcut else 0, _lib.ptr(res), N, _lib.stream_ptr()), "vdk_gemm_tn")
    torch.cuda.synchronize()
    acc = a.double() @ wp.double().t()
    pref = acc + bp.double() + (res.double() if shortcut else 0)
    mag = a.double().abs() @ wp.double().abs().t()
    e = (-(-K // 16) + 17) * 2.0 ** -23 * mag + 2.0 ** -23 * (pref.abs() + acc.abs() + 1)
    check_within(out, pref, e + ulp(pref.abs() + e, torch.bfloat16), f"projection K={K}", lambda bad: f"{int(bad.sum())} elements")
