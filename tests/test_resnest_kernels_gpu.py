"""The new kernels of the ResNeSt forward against fp64 references of the same inputs:
- vdk_conv2d_grouped_ex (kConvGroupedEx mode of the wgmma GEMM) elementwise within tests/conv_ref.conv_bound at the executed
  K = 9 * cpb * 64: conv_reference of the dense weight that is zero outside each output channel's group is exactly the
  grouped conv.  Every split-conv shape of the five ResNeSts at 224, ragged maps with M tiles crossing images, NaN-guarded
  outputs, batches giving every persistent CTA at least 3 tiles, and the groups = 1 form (Cin 80 / 96 / 160) with an in-place
  residual;
- the split-attention gate (vdk_split_attn_gate: radix mean, excitation with radix softmax / sigmoid, combine with and
  without the fused stride-2 average pool) within bounds derived from its fp32 and bf16 roundings;
- avd_first's average pool (vdk_avgpool3s2) within one fp32 sum and one bf16 rounding."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from conv_ref import conv_bound, conv_reference
from kernel_ref import Guarded, check_within, ulp
from visiondk_b200 import _lib
from visiondk_b200.resnest import RESNEST_ARCHS, attn_width, group_width, pack_split, split_conv_blocks

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def dense_grouped(w, groups):
    """[Cout, cgi, k, k] grouped weight -> the dense [Cout, k, k, Cin] weight, zero outside each output channel's group."""
    cout, cgi, k = w.shape[0], w.shape[1], w.shape[2]
    cgo = cout // groups
    dense = w.new_zeros(cout, k, k, cgi * groups)
    for g in range(groups):
        dense[g * cgo:(g + 1) * cgo, :, :, g * cgi:(g + 1) * cgi] = w[g * cgo:(g + 1) * cgo].permute(0, 2, 3, 1)
    return dense


def run_conv(lib, x, w, bias, groups, k, epi, residual=None, y=None):
    B, H, W, cin = x.shape
    cout = w.shape[0]
    M = B * H * W  # stride 1, "same" padding
    y = y if y is not None else Guarded(M, cout, cout, torch.bfloat16)
    d = _lib.ConvDesc(x=x.data_ptr(), w=w.data_ptr(), bias=bias.data_ptr(), residual=0 if residual is None else residual, y=y.ptr(),
                      B=B, H=H, W=W, Cin=cin, Cout=cout, kernel=k, stride=1, pad=k // 2, epilogue=epi)
    _lib.check(lib.vdk_conv2d_grouped_ex(C.byref(d), groups, _lib.stream_ptr()), "vdk_conv2d_grouped_ex")
    torch.cuda.synchronize()
    return y


def check_split(lib, B, H, W, cin, cout, groups, seed, mags=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, cin, device="cuda", generator=g)
    if mags is not None:
        x = x * torch.tensor(mags, device="cuda").view(B, 1, 1, 1)
    x = x.to(torch.bfloat16)
    cgi = cin // groups
    w = (torch.randn(cout, cgi, 3, 3, device="cuda", generator=g) * (2.0 / (9 * cgi)) ** 0.5).to(torch.bfloat16)
    bias = 0.1 * torch.randn(cout, device="cuda", generator=g)
    packed = pack_split(w.float(), groups).to(torch.bfloat16).contiguous()  # exact: bf16 values and zeros
    y = run_conv(lib, x, packed, bias, groups, 3, _lib.EPI_RELU)
    acc, mag = conv_reference(x, dense_grouped(w, groups), 1, 1)
    ref = (acc + bias.double()).clamp_min(0.0)
    bound = conv_bound(acc, mag, 9 * split_conv_blocks(cin, cout, groups) * 64, bias, None, ref)
    got = y.view.reshape(B, H, W, cout)

    def describe(bad):
        pix = bad.reshape(-1, cout).any(dim=1).nonzero().flatten()
        ch = bad.reshape(-1, cout).any(dim=0).nonzero().flatten()
        return f"output pixels {pix[:8].tolist()} (tile rows {sorted(set((pix // 128).tolist()))[:8]}), channels {ch[:8].tolist()}"

    check_within(got, ref, bound, f"split conv {B}x{H}x{W} {cin}->{cout} g{groups}", describe)
    assert y.guard_errors() == "", y.guard_errors()
    return got


def split_conv_shapes(size=224):
    """(H, Cin, Cout, groups) of every distinct split conv of the five ResNeSts at `size`."""
    out = set()
    for a in RESNEST_ARCHS.values():
        h = size // 4
        for s in range(4):
            gw = group_width(64 << s, a["base_width"], a["cardinality"])
            ho = h if s == 0 else h // 2
            for hh in {ho if a["avd_first"] else h, ho}:
                out.add((hh, gw, gw * a["radix"], a["cardinality"] * a["radix"]))
            h = ho
    return sorted(out)


@pytest.mark.parametrize("H,cin,cout,groups", split_conv_shapes())
def test_split_conv_every_resnest_shape(lib, H, cin, cout, groups):
    check_split(lib, 2, H, H, cin, cout, groups, seed=H + cin + groups)


def test_split_conv_ragged_tiles_cross_images(lib):
    """81 output pixels per image: 128-row tiles straddle images whose magnitudes differ by 10^4; a non-square map."""
    check_split(lib, 5, 9, 9, 80, 320, 8, seed=7, mags=[1.0, 100.0, 0.01, 30.0, 0.3])
    check_split(lib, 3, 7, 11, 96, 96, 4, seed=8)
    check_split(lib, 3, 5, 13, 24, 40, 8, seed=9)  # cgi = 3, cgo = 5: groups straddle every tile boundary


def test_split_conv_every_cta_runs_three_tiles(lib):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_tiles = 640 // 128
    B = -(-3 * sms * 128 // (n_tiles * 14 * 14)) + 1
    got = check_split(lib, B, 14, 14, 160, 640, 8, seed=B)
    assert -(-got.shape[0] * 14 * 14 // 128) * n_tiles >= 3 * sms


@pytest.mark.parametrize("cin,cout", [(80, 320), (96, 384), (160, 640)])
def test_groups_one_conv3_with_in_place_residual(lib, cin, cout):
    g = torch.Generator(device="cuda").manual_seed(cin)
    B, H = 3, 14
    x = torch.randn(B, H, H, cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(cout, cin, device="cuda", generator=g) * cin ** -0.5).to(torch.bfloat16)
    bias = 0.1 * torch.randn(cout, device="cuda", generator=g)
    res = torch.randn(B * H * H, cout, device="cuda", generator=g).to(torch.bfloat16)
    y = Guarded(B * H * H, cout, cout, torch.bfloat16).fill_(res)
    run_conv(lib, x, w, bias, 1, 1, _lib.EPI_RESIDUAL_RELU, residual=y.ptr(), y=y)
    acc, mag = conv_reference(x, w.view(cout, 1, 1, cin), 1, 0)
    ref = (acc + bias.double() + res.double().view(B, H, H, cout)).clamp_min(0.0)
    bound = conv_bound(acc, mag, cin, bias, res.view(B, H, H, cout), ref)
    check_within(y.view.reshape(B, H, H, cout), ref, bound, f"conv3 {cin}->{cout} in place", lambda bad: "")
    assert y.guard_errors() == "", y.guard_errors()


# ---- split-attention gate ----

def gate_weights(C_, R, card, A, g):
    Cg, Ag = C_ // card, A // card
    w1 = torch.randn(A, Cg, device="cuda", generator=g) * Cg ** -0.5
    b1 = 0.1 * torch.randn(A, device="cuda", generator=g)
    w2 = torch.randn(R * C_, Ag, device="cuda", generator=g) * Ag ** -0.5
    b2 = 0.1 * torch.randn(R * C_, device="cuda", generator=g)
    return w1, b1, w2, b2


def block_diag(w, card):
    """grouped 1x1 weight [out, in / card] -> dense [out, in], zero outside the groups."""
    o, i = w.shape
    d = w.new_zeros(o, i * card)
    for g in range(card):
        d[g * (o // card):(g + 1) * (o // card), g * i:(g + 1) * i] = w[g * (o // card):(g + 1) * (o // card)]
    return d


@pytest.mark.parametrize("B,H,C_,R,card,pool", [(3, 56, 64, 2, 1, 1), (11, 7, 512, 2, 1, 0), (4, 28, 96, 1, 4, 0),
                                                (9, 7, 768, 1, 4, 1), (2, 56, 80, 4, 2, 0), (17, 14, 320, 4, 2, 1),
                                                (5, 7, 640, 4, 2, 0), (2, 9, 80, 4, 2, 1)])
def test_split_attn_gate_against_fp64(lib, B, H, C_, R, card, pool):
    A = attn_width(C_, R)
    g = torch.Generator(device="cuda").manual_seed(B * H + C_)
    u = torch.relu(torch.randn(B, H, H, R * C_, device="cuda", generator=g) + 0.5).to(torch.bfloat16)  # post-ReLU maps
    w1, b1, w2, b2 = gate_weights(C_, R, card, A, g)
    gap = torch.empty(B, C_, device="cuda")
    attn = torch.empty(B, R * C_, device="cuda")
    Ho = (H - 1) // 2 + 1 if pool else H
    v = Guarded(B * Ho * Ho, C_, C_, torch.bfloat16)
    _lib.check(lib.vdk_split_attn_gate(u.data_ptr(), B, H, H, C_, R, card, A, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                       b2.data_ptr(), gap.data_ptr(), attn.data_ptr(), pool, v.ptr(), _lib.stream_ptr()),
               "vdk_split_attn_gate")
    torch.cuda.synchronize()
    name = f"B{B} {H}x{H} C{C_} R{R} card{card} pool{pool}"
    ud = u.double().view(B, H * H, R, C_)
    # gap: per lane ceil(HW / 32) * R sequential fp32 adds, a 5-level tree, one division
    g_ref = ud.sum(dim=2).mean(dim=1)
    g_bound = (math.ceil(H * H / 32) * R + 6) * U * ud.abs().sum(dim=2).mean(dim=1) + 1e-300
    check_within(gap, g_ref, g_bound, f"gap {name}", lambda bad: "")
    # attention from the kernel's gap: fc1 (ceil(Cg / 32) FMAs per lane + 5 shuffle adds + bias), fc2 (Ag FMAs + bias), then
    # softmax over the radix (sum_s |d a_r / d z_s| <= 1/2; expf, the sum and the division <= 8 u relative) or sigmoid
    W1, W2 = block_diag(w1.double(), card), block_diag(w2.double(), card)
    gd = gap.double()
    hid = (gd @ W1.T + b1.double()).clamp_min(0.0)
    e_h = (math.ceil(C_ // card / 32) + 7) * U * (gd.abs() @ W1.abs().T + b1.double().abs())
    z = hid @ W2.T + b2.double()
    e_z = (A // card + 2) * U * ((hid.abs() + e_h) @ W2.abs().T + b2.double().abs()) + e_h @ W2.abs().T
    Cg = C_ // card
    # fc2 row g R Cg + r Cg + i holds attention entry r C + g Cg + i
    perm = torch.tensor([(c // Cg) * R * Cg + r * Cg + c % Cg for r in range(R) for c in range(C_)], device="cuda")
    z, e_z = z[:, perm].view(B, R, C_), e_z[:, perm].view(B, R, C_)
    if R == 1:
        a_ref = torch.sigmoid(z)
        a_bound = 0.25 * e_z + 4 * U * a_ref
    else:
        a_ref = torch.softmax(z, dim=1)
        a_bound = 0.5 * e_z.max(dim=1, keepdim=True).values + 8 * U * a_ref
    check_within(attn.view(B, R, C_), a_ref, a_bound, f"attn {name}", lambda bad: "")
    # combine from the kernel's attention: the r = 0 product and R - 1 FMAs per tap; pooled: up to 9 tap sums, / 9
    ad = attn.double().view(B, 1, R, C_)
    comb = (ad * ud).sum(dim=2).view(B, H, H, C_)
    mag = (ad * ud).abs().sum(dim=2).view(B, H, H, C_)
    if pool:
        avg = lambda t: F.avg_pool2d(t.permute(0, 3, 1, 2), 3, 2, 1, count_include_pad=True).permute(0, 2, 3, 1)
        v_ref, e = avg(comb), (R + 10) * U * avg(mag)
    else:
        v_ref, e = comb, R * U * mag
    check_within(v.view.reshape(B, Ho, Ho, C_), v_ref, e + ulp(v_ref.abs() + e, torch.bfloat16), f"combine {name}", lambda bad: "")
    assert v.guard_errors() == "", v.guard_errors()


@pytest.mark.parametrize("B,H,W,C_", [(4, 56, 56, 80), (3, 28, 28, 320), (2, 7, 7, 640), (3, 9, 12, 96)])
def test_avgpool3s2_against_fp64(lib, B, H, W, C_):
    x = torch.randn(B, H, W, C_, device="cuda", generator=torch.Generator(device="cuda").manual_seed(H * C_)).to(torch.bfloat16)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = Guarded(B * Ho * Wo, C_, C_, torch.bfloat16)
    _lib.check(lib.vdk_avgpool3s2(x.data_ptr(), B, H, W, C_, y.ptr(), _lib.stream_ptr()), "vdk_avgpool3s2")
    torch.cuda.synchronize()
    avg = lambda t: F.avg_pool2d(t.permute(0, 3, 1, 2), 3, 2, 1, count_include_pad=True).permute(0, 2, 3, 1)
    ref = avg(x.double())
    e = 10 * U * avg(x.double().abs())
    check_within(y.view.reshape(B, Ho, Wo, C_), ref, e + ulp(ref.abs() + e, torch.bfloat16), f"avgpool {B}x{H}x{W}x{C_}",
                 lambda bad: "")
    assert y.guard_errors() == "", y.guard_errors()
