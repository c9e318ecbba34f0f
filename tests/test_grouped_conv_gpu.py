"""The new kernels of the ResNeXt / legacy SENet forward against fp64 references of the same inputs:
- vdk_conv2d_grouped (kConvGrouped mode of the wgmma GEMM) elementwise within tests/conv_ref.conv_bound at the executed
  K = k*k*128: conv_reference of the block-diagonal dense weight is exactly the grouped conv.  Channels per group 4 .. 64
  at stride 1 and 2, every ResNeXt / SE-ResNeXt stage shape, ragged maps with M tiles crossing images, NaN-guarded
  outputs, and batches giving every persistent CTA at least 3 tiles;
- the SE gate (vdk_se_gate: spatial mean, excitation, scale + residual + ReLU) within bounds derived from its fp32 and
  bf16 roundings, with means near zero and large offsets;
- the ceil-mode stem pool (vdk_stem_maxpool) bit-exact against F.max_pool2d(..., ceil_mode=True)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from conv_ref import conv_bound, conv_reference
from kernel_ref import Guarded, check_within, ulp
from resnext_senet_ref import block_diagonal
from visiondk_b200 import _lib
from visiondk_b200.resnet import STEM_POOL_CEIL, STEM_POOL_PAD1, pack_grouped

pytestmark = pytest.mark.gpu


def make(B, H, W, Cch, cg, seed, mags=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cch, device="cuda", generator=g)
    if mags is not None:
        x = x * torch.tensor(mags, device="cuda").view(B, 1, 1, 1)
    w = torch.randn(Cch, cg, 3, 3, device="cuda", generator=g) * (2.0 / (9 * cg)) ** 0.5
    bias = 0.1 * torch.randn(Cch, device="cuda", generator=g)
    return x.to(torch.bfloat16), w.to(torch.bfloat16), bias


def check_grouped(lib, x, w, bias, stride, name):
    B, H, W, Cch = x.shape
    cg = w.shape[1]
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    M = B * Ho * Wo
    packed = pack_grouped(w.float()).to(torch.bfloat16).contiguous()  # exact: a permutation of bf16 values and zeros
    y = Guarded(M, Cch, Cch, torch.bfloat16)
    d = _lib.ConvDesc(x=x.data_ptr(), w=packed.data_ptr(), bias=bias.data_ptr(), residual=0, y=y.ptr(), B=B, H=H, W=W, Cin=Cch,
                      Cout=Cch, kernel=3, stride=stride, pad=1, epilogue=_lib.EPI_RELU)
    _lib.check(lib.vdk_conv2d_grouped(C.byref(d), Cch // cg, _lib.stream_ptr()), "vdk_conv2d_grouped")
    torch.cuda.synchronize()
    acc, mag = conv_reference(x, block_diagonal(w), stride, 1)
    ref = (acc + bias.double()).clamp_min(0.0)
    bound = conv_bound(acc, mag, 9 * 128, bias, None, ref)
    got = y.view.reshape(B, Ho, Wo, Cch)

    def describe(bad):
        pix = bad.reshape(-1, Cch).any(dim=1).nonzero().flatten()
        ch = bad.reshape(-1, Cch).any(dim=0).nonzero().flatten()
        return f"output pixels {pix[:8].tolist()} (tile rows {sorted(set((pix // 128).tolist()))[:8]}), channels {ch[:8].tolist()}"

    check_within(got, ref, bound, name, describe)
    assert y.guard_errors() == "", y.guard_errors()
    return got


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("cg", [4, 8, 16, 32, 64])
def test_grouped_conv_channels_per_group(lib, cg, stride):
    x, w, bias = make(2, 14, 14, 256, cg, seed=cg + stride)
    check_grouped(lib, x, w, bias, stride, f"grouped cg{cg} s{stride}")


def resnext_stage_shapes(width0, groups, size=224):
    """(H_in, width, stride) of every distinct grouped 3x3 conv of a ResNeXt / SE-ResNeXt with stage-0 width `width0`."""
    out, h = [], size // 4
    for i in range(4):
        width = width0 << i
        s = 1 if i == 0 else 2
        out.append((h, width, s))
        h //= s
        if s == 2:
            out.append((h, width, 1))
    return [(hh, wd, s, wd // groups) for hh, wd, s in out]


@pytest.mark.parametrize("arch,width0,groups", [("resnext50_32x4d / seresnext", 128, 32), ("resnext101_32x8d", 256, 32),
                                                ("resnext101_64x4d", 256, 64)])
def test_grouped_conv_every_stage_shape(lib, arch, width0, groups):
    for n, (h, width, s, cg) in enumerate(resnext_stage_shapes(width0, groups)):
        x, w, bias = make(2, h, h, width, cg, seed=n)
        check_grouped(lib, x, w, bias, s, f"{arch} {h}x{h}x{width} s{s} cg{cg}")


@pytest.mark.parametrize("stride", [1, 2])
def test_grouped_conv_ragged_tiles_cross_images(lib, stride):
    """81 output pixels per image: 128-row tiles straddle images whose magnitudes differ by 10^4."""
    x, w, bias = make(5, 9 * stride, 9 * stride, 384, 16, seed=7, mags=[1.0, 100.0, 0.01, 30.0, 0.3])
    check_grouped(lib, x, w, bias, stride, f"cross-image s{stride}")
    x, w, bias = make(3, 7, 11, 128, 8, seed=8)  # ragged, non-square map
    check_grouped(lib, x, w, bias, stride, f"ragged 7x11 s{stride}")


@pytest.mark.parametrize("stride", [1, 2])
def test_grouped_conv_every_cta_runs_three_tiles(lib, stride):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cch = 256
    B = -(-3 * sms * 128 // (2 * 14 * 14)) + 1
    x, w, bias = make(B, 14 * stride, 14 * stride, cch, 8, seed=B)
    got = check_grouped(lib, x, w, bias, stride, f"persistent s{stride} B{B}")
    assert -(-got.shape[0] * 14 * 14 // 128) * (cch // 128) >= 3 * sms


# ---- SE gate ----

def run_se(lib, y, w1, b1, w2, b2, res):
    B, HW, Cch = y.shape
    rd = w1.shape[0]
    mean = torch.empty(B, Cch, device="cuda")
    gate = torch.empty(B, Cch, device="cuda")
    out = res.clone()
    _lib.check(lib.vdk_se_gate(y.data_ptr(), B, HW, Cch, rd, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                               mean.data_ptr(), gate.data_ptr(), out.data_ptr(), _lib.stream_ptr()), "vdk_se_gate")
    torch.cuda.synchronize()
    return mean, gate, out


@pytest.mark.parametrize("B,HW,Cch,offset", [(3, 3136, 256, 0.0), (2, 784, 512, 50.0), (4, 49, 2048, 0.0), (2, 196, 1024, -200.0),
                                             (5, 5, 64, 3.0)])
def test_se_gate_against_fp64(lib, B, HW, Cch, offset):
    u = 2.0 ** -24
    g = torch.Generator(device="cuda").manual_seed(HW + Cch)
    rd = max(Cch // 16, 1)
    # per-channel offsets: with offset 0 the means sit near zero, with a large offset they carry a big common part
    y = (torch.randn(B, HW, Cch, device="cuda", generator=g) + offset * torch.rand(1, 1, Cch, device="cuda", generator=g))
    y = y.to(torch.bfloat16)
    w1 = torch.randn(rd, Cch, device="cuda", generator=g) * Cch ** -0.5
    b1 = 0.1 * torch.randn(rd, device="cuda", generator=g)
    w2 = torch.randn(Cch, rd, device="cuda", generator=g) * rd ** -0.5
    b2 = 0.1 * torch.randn(Cch, device="cuda", generator=g)
    res = torch.randn(B, HW, Cch, device="cuda", generator=g).to(torch.bfloat16)
    mean, gate, out = run_se(lib, y, w1, b1, w2, b2, res)
    yd = y.double()
    # mean: per lane ceil(HW / 32) sequential fp32 adds, a 5-level tree, one division
    m_ref = yd.mean(dim=1)
    m_bound = (math.ceil(HW / 32) + 5 + 1) * u * yd.abs().mean(dim=1) + 1e-300
    check_within(mean, m_ref, m_bound, f"se mean {B}x{HW}x{Cch} off {offset}", lambda bad: "")
    # excitation from the kernel's own fp32 mean: fc1 (ceil(C / 32) sequential FMAs per lane + 5 shuffle adds + bias),
    # fc2 (rd sequential FMAs + bias), sigmoid (slope <= 1/4; expf, 1 + e and the division: <= 4 u relative)
    md = mean.double()
    w1d, b1d, w2d, b2d = w1.double(), b1.double(), w2.double(), b2.double()
    pre1 = md @ w1d.T + b1d
    hid = pre1.clamp_min(0.0)
    e_h = (math.ceil(Cch / 32) + 7) * u * (md.abs() @ w1d.abs().T + b1d.abs())
    pre2 = hid @ w2d.T + b2d
    e_z = (rd + 2) * u * ((hid.abs() + e_h) @ w2d.abs().T + b2d.abs()) + e_h @ w2d.abs().T
    s_ref = torch.sigmoid(pre2)
    check_within(gate, s_ref, 0.25 * e_z + 4 * u * s_ref, f"se gate {B}x{HW}x{Cch}", lambda bad: "")
    # out = ReLU(y * gate + res) from the kernel's gate: one fp32 FMA rounding, then the bf16 store
    pre = yd * gate.double()[:, None, :] + res.double()
    o_ref = pre.clamp_min(0.0)
    e = u * pre.abs()
    check_within(out, o_ref, e + ulp(o_ref + e, torch.bfloat16), f"se out {B}x{HW}x{Cch}", lambda bad: "")


# ---- stem pool ----

@pytest.mark.parametrize("H,W", [(112, 112), (32, 32), (144, 144), (9, 12), (7, 7)])
@pytest.mark.parametrize("mode", [STEM_POOL_CEIL, STEM_POOL_PAD1])
def test_stem_pool_bit_exact(lib, H, W, mode):
    x = torch.randn(3, H, W, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(H * W)).to(torch.bfloat16)
    ref = (F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 0, ceil_mode=True) if mode == STEM_POOL_CEIL
           else F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1)).permute(0, 2, 3, 1).to(torch.bfloat16)
    Ho, Wo = ref.shape[1], ref.shape[2]
    y = Guarded(3 * Ho * Wo, 64, 64, torch.bfloat16)
    _lib.check(lib.vdk_stem_maxpool(x.data_ptr(), 3, H, W, 64, mode, y.ptr(), _lib.stream_ptr()), "vdk_stem_maxpool")
    torch.cuda.synchronize()
    assert torch.equal(y.view.reshape(3, Ho, Wo, 64), ref)
    assert y.guard_errors() == "", y.guard_errors()
