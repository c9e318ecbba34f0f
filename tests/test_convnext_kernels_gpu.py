"""Elementwise parity of the ConvNeXt training kernels that are not GEMMs (csrc/train_ops.cu, csrc/convnext.cu) against
fp64 references of the same bf16 / fp32 inputs, with bounds derived from each kernel's roundings (the derivations are the
docstrings in kernel_ref.py).  Cases are sized from the device's SM count so that the loops the batch-128 training step
depends on run: depthwise weight-gradient CTAs with several images (ragged last group, the 16-image cap), LayerNorm
backward warps with at least three grid-stride trips, and channel counts that are not multiples of 64."""
import pytest
import torch

from kernel_ref import (Guarded, batchnorm_bwd_bound, batchnorm_bwd_reference, batchnorm_fwd_bound, batchnorm_fwd_reference,
                        bf16_store_bound, check_within, describe_dw_tiles, describe_pixels, describe_wgrad,
                        dwconv7_bwd_data_bound, dwconv7_ln_bound, dwconv7_ln_reference, dwconv7_reference, dwconv_launch,
                        layernorm_bwd_bound, layernorm_bwd_dgamma, layernorm_bwd_reference, ln_bwd_launch, wgrad_bound,
                        wgrad_launch, wgrad_reference)
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu
STATS = {}


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bf16_randn(*shape, scale=1.0, gen=None):
    return (torch.randn(*shape, device="cuda", generator=gen) * scale).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------------------------
# depthwise weight gradient: dw49[tap, c] += sum g x, dbias[c] += sum g

# (B, H, W, C, regime): T = 14 / 7 / runtime, ipc >= 2 with a ragged last group, the 16-image cap, ragged 64-channel chunks
WGRAD_CASES = [
    (128, 56, 56, 128, "T14 ipc>=2 ragged"),     # ConvNeXt-B stage 0 at the bench's batch
    (128, 7, 7, 1024, "T7 ipc>=2 ragged"),       # ConvNeXt-B stage 3
    (200, 28, 28, 80, "T14 ipc>=2 ragged, masked chunk"),
    (64, 10, 12, 96, "runtime T, masked chunk"),
    (8456, 14, 14, 40, "ipc 16, masked chunk"),
    (32, 56, 56, 40, "atto stage 0"),
    (16, 56, 56, 48, "femto stage 0"),
    (6, 5, 5, 136, "runtime T below 7"),
]


@pytest.mark.parametrize("B,H,W,C,regime", WGRAD_CASES, ids=[c[4].replace(" ", "_") for c in WGRAD_CASES])
def test_dwconv7_wgrad_elementwise(lib, B, H, W, C, regime):
    sm = sm_count()
    L = wgrad_launch(B, H, W, C, sm)
    if "ipc 16" in regime:
        assert L["ipc"] == 16 and B % 16 != 0, L
    elif "ipc>=2" in regime:
        assert L["ipc"] >= 2 and B % L["ipc"] != 0, L
    if "T14" in regime:
        assert L["T"] == 14
    if "T7" in regime:
        assert L["T"] == 7
    if "runtime" in regime:
        assert L["T"] not in (7, 14)
    if "masked" in regime:
        assert C % 64 != 0
    gen = torch.Generator(device="cuda").manual_seed(B * 7 + C)
    x = bf16_randn(B, H, W, C, gen=gen)
    g = bf16_randn(B, H, W, C, gen=gen)
    dw = Guarded(49, C, C, torch.float32, extra_rows=1, tail=64)
    db = Guarded(1, C, C, torch.float32, extra_rows=1, tail=64)
    dw_init = torch.randn(49, C, device="cuda", generator=gen)
    db_init = torch.randn(1, C, device="cuda", generator=gen)
    dw.fill_(dw_init)
    db.fill_(db_init)
    _lib.check(lib.vdk_dwconv7_wgrad(x.data_ptr(), g.data_ptr(), B, H, W, C, dw.ptr(), db.ptr(), _lib.stream_ptr()), "wgrad")
    torch.cuda.synchronize()
    ref, mag, bref, bmag = wgrad_reference(x, g)
    check_within(dw.view, dw_init.double() + ref, wgrad_bound(mag, dw_init, L), f"wgrad dw {regime}",
                 lambda bad: describe_wgrad(bad, L), STATS)
    check_within(db.view, db_init.double() + bref[None], wgrad_bound(bmag[None], db_init, L), f"wgrad dbias {regime}",
                 lambda bad: describe_wgrad(bad, L), STATS)
    assert not dw.guard_errors(), "dw49: " + dw.guard_errors()
    assert not db.guard_errors(), "dbias: " + db.guard_errors()


# ------------------------------------------------------------------------------------------------------------------------------
# depthwise forward (mode 0: LayerNorm_C(conv + bias), rstd_out) and backward-data (mode 1: bf16(sum_49 w x + addend))

def run_dwconv_case(lib, B, H, W, C, mode, edge="", pipe=True, stats=STATS):
    """Runs vdk_dwconv7 on seeded inputs into NaN-guarded outputs and checks every element against the fp64 reference.
    Persistent-kernel cases must give every group at least 3 tiles.  Edges (mode 0): "zero-var" (image 0 all zero and
    one bias for every channel: those pixels have zero variance and must give exactly bf16(beta)), "chunk-means" (the
    bias of 128-channel chunk k is 1e3 k: Chan's combination of chunk means 1e3 apart), "offset" (bias + 1e3)."""
    L = dwconv_launch(B, H, W, C, torch.cuda.get_device_properties(0).multi_processor_count, pipe)
    if L["kind"] == "pipe":
        assert L["min_tiles_per_group"] >= 3, L
    gen = torch.Generator(device="cuda").manual_seed(C * 11 + H * 3 + B + mode)
    x = bf16_randn(B, H, W, C, gen=gen)
    w49 = 0.2 * torch.randn(49, C, device="cuda", generator=gen)
    out = Guarded(B * H * W, C, C, torch.bfloat16, extra_rows=0, tail=4096)
    tag = f"dwconv7 mode {mode} {L['kind']} chunk={L['chunk']}x{L['nchunks']} TH={L['TH']} {edge}".rstrip()
    if mode == 1:
        add = bf16_randn(B, H, W, C, gen=gen)
        _lib.check(lib.vdk_dwconv7(1, x.data_ptr(), B, H, W, C, w49.data_ptr(), 0, 0, 0, 0.0, out.ptr(), 0, add.data_ptr(),
                                   _lib.stream_ptr()), tag)
        torch.cuda.synchronize()
        ref, mag = dwconv7_reference(x, w49)
        ref += add.double()
        check_within(out.view.view(B, H, W, C), ref, dwconv7_bwd_data_bound(ref, mag, add), tag,
                     lambda bad: describe_dw_tiles(bad, L), stats)
        assert not out.guard_errors(), out.guard_errors()
        return L
    bias = 0.3 * torch.randn(C, device="cuda", generator=gen)
    gamma = 1 + 0.3 * torch.randn(C, device="cuda", generator=gen)
    beta = 0.2 * torch.randn(C, device="cuda", generator=gen)
    if edge == "zero-var":
        x[0] = 0
        bias.fill_(0.75)  # every partial sum exact: the computed mean is 0.75 up to one rounding of 1 / nchunks or 1 / C
        beta = (torch.sign(beta) * (0.25 + beta.abs())).to(torch.bfloat16).float()  # half a bf16 ulp >> that error
    elif edge == "chunk-means":
        bias += 1e3 * (torch.arange(C, device="cuda") // 128).float()
    elif edge == "offset":
        bias += 1e3
    eps = 1e-6
    rstd = Guarded(1, B * H * W, B * H * W, torch.float32, extra_rows=0, tail=256)
    _lib.check(lib.vdk_dwconv7(0, x.data_ptr(), B, H, W, C, w49.data_ptr(), bias.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                               eps, out.ptr(), rstd.ptr(), 0, _lib.stream_ptr()), tag)
    torch.cuda.synchronize()
    ref = dwconv7_ln_reference(x, w49, bias, gamma, beta, eps)
    yb, rb = dwconv7_ln_bound(ref, gamma, beta, eps, L["chunk"])
    got = out.view.view(B, H, W, C)
    check_within(got, ref["y"], yb, tag + " y", lambda bad: describe_dw_tiles(bad, L), stats)
    check_within(rstd.view.view(B, H, W), ref["rstd"], rb, tag + " rstd_out",
                 lambda bad: describe_dw_tiles(bad[..., None], L), stats)
    if edge == "zero-var":
        assert torch.equal(got[0], beta.to(torch.bfloat16).expand(H, W, C)), "zero-variance pixels must give exactly beta"
    assert not out.guard_errors(), "y: " + out.guard_errors()
    assert not rstd.guard_errors(), "rstd_out: " + rstd.guard_errors()
    return L


# (B, H, W, C, edge): every CHUNK x TH instantiation of the persistent kernel, one chunk (no cluster) and clustered
# (2-12 chunks; 12 is a non-portable cluster), batches sized so that every group runs >= 3 tiles; the four ConvNeXt-B 224
# stage shapes at the bench's batch 128; ragged H and W; the LayerNorm edges; the all-channel fallback at T = 7, 4, 2
DW_FWD_CASES = [
    (50, 28, 28, 64, ""), (800, 7, 7, 64, ""), (200, 14, 14, 96, ""), (800, 7, 7, 96, ""), (800, 7, 7, 128, ""),
    (128, 56, 56, 128, ""), (128, 28, 28, 256, ""), (128, 14, 14, 512, ""), (128, 7, 7, 1024, ""),
    (100, 14, 14, 192, ""), (132, 7, 7, 576, ""), (32, 13, 19, 320, ""), (156, 7, 7, 320, ""),
    (66, 7, 7, 1536, ""), (17, 14, 14, 1536, ""),
    (66, 7, 7, 1536, "zero-var"), (50, 14, 14, 512, "chunk-means"), (100, 14, 14, 256, "offset"),
    (16, 56, 56, 40, ""), (8, 14, 14, 680, ""), (4, 7, 7, 1576, ""), (16, 14, 14, 680, "zero-var"),
]


@pytest.mark.parametrize("B,H,W,C,edge", DW_FWD_CASES, ids=[f"{c[3]}x{c[1]}x{c[2]}b{c[0]}{'-' + c[4] if c[4] else ''}"
                                                          for c in DW_FWD_CASES])
def test_dwconv7_ln_forward_elementwise(lib, B, H, W, C, edge):
    run_dwconv_case(lib, B, H, W, C, 0, edge)


# the same kernels in mode 1 (no cluster: grid = slots / nchunks groups, each running >= 3 tiles)
DW_BWD_CASES = [
    (128, 56, 56, 128), (128, 28, 28, 256), (128, 14, 14, 512), (128, 7, 7, 1024), (64, 28, 28, 192), (132, 7, 7, 768),
    (96, 13, 19, 320), (66, 7, 7, 1536), (50, 28, 28, 64), (800, 7, 7, 96), (16, 56, 56, 40), (8, 14, 14, 680), (4, 7, 7, 1576),
]


@pytest.mark.parametrize("B,H,W,C", DW_BWD_CASES, ids=[f"{c[3]}x{c[1]}x{c[2]}b{c[0]}" for c in DW_BWD_CASES])
def test_dwconv7_bwd_data_elementwise(lib, B, H, W, C):
    run_dwconv_case(lib, B, H, W, C, 1)


# the round-1 chunk kernel (one tile per CTA; the dispatcher's fallback when the persistent grid does not fit) at its
# three chunk widths, clustered up to the non-portable 12, in both modes.  VDK_DWCONV_PIPE is read once per process.
CHUNK_KERNEL_CASES = [(8, 14, 14, 320, 0), (8, 14, 14, 192, 0), (8, 7, 7, 1536, 0), (4, 28, 28, 128, 0), (6, 13, 19, 512, 0),
                      (8, 14, 14, 320, 1), (8, 14, 14, 192, 1), (8, 7, 7, 1536, 1)]


def run_chunk_kernel_cases():
    from visiondk_b200 import build
    build.build()
    lib = _lib.load()
    stats = {}
    for B, H, W, C, mode in CHUNK_KERNEL_CASES:
        assert run_dwconv_case(lib, B, H, W, C, mode, pipe=False, stats=stats)["kind"] == "chunk"


def test_dwconv7_chunk_kernel_elementwise_in_subprocess():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, VDK_DWCONV_PIPE="0")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_convnext_kernels_gpu as t; t.run_chunk_kernel_cases()"
            % (root, os.path.join(root, "tests")))
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------------------------------------
# LayerNorm backward

# every ConvNeXt width (atto ... large) and ViT's 384 / 768 / 1024: every (LPP, IT, U) instantiation, masked lanes
LN_WIDTHS = [40, 48, 64, 80, 96, 128, 160, 192, 256, 320, 384, 512, 640, 768, 1024, 1536]


def ln_case(C, patch, sm):
    """An NHWC shape (14 x 14 images) on which every warp of the launch makes at least 3 grid-stride trips."""
    H = W = 14
    B = 1
    while ln_bwd_launch(B * H * W, C, sm)["min_trips"] < 3:
        B *= 2
    return B, H, W


@pytest.mark.parametrize("patch", [1, 2])
@pytest.mark.parametrize("C", LN_WIDTHS)
def test_layernorm_bwd_elementwise(lib, C, patch):
    """dx, dgamma += and dbeta += of vdk_layernorm_bwd against fp64, with |beta / gamma| up to 30 on one channel in eight
    (the saved-bf16 amplification of layernorm_bwd_bound), a gamma = 0 channel whose beta bf16 cannot represent, the
    addend, and nonzero initial dgamma / dbeta."""
    sm = sm_count()
    B, H, W = ln_case(C, patch, sm)
    P = B * H * W
    L = ln_bwd_launch(P, C, sm)
    assert L["min_trips"] >= 3, L
    gen = torch.Generator(device="cuda").manual_seed(C * 3 + patch)
    x = torch.randn(P, C, device="cuda", dtype=torch.float64, generator=gen) * 2 + 0.3
    mean = x.mean(-1, keepdim=True)
    rstd64 = ((x - mean).pow(2).mean(-1) + 1e-6).rsqrt()
    xhat = (x - mean) * rstd64[:, None]
    sign = torch.where(torch.rand(C, device="cuda", generator=gen) < 0.5, -1.0, 1.0)
    gamma = (sign * (0.2 + 1.3 * torch.rand(C, device="cuda", generator=gen))).float()
    beta = 0.2 * torch.randn(C, device="cuda", generator=gen)
    far = torch.arange(C, device="cuda") % 8 == 3
    beta[far] = (gamma[far] * 30 * (2 * torch.rand(int(far.sum()), device="cuda", generator=gen) - 1)).float()
    gamma[5] = 0.0
    beta[5] = 0.1  # not a bf16 value: y = bf16(0.1) on every pixel of channel 5
    y = (gamma.double() * xhat + beta.double()).to(torch.float32).to(torch.bfloat16)
    rstd = rstd64.float()
    dy = bf16_randn(P, C, gen=gen)
    add = bf16_randn(P, C, gen=gen)
    if patch == 2:
        def to_patch(t):
            return t.view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * C).contiguous()
        dy_k, y_k = to_patch(dy), to_patch(y)
    else:
        dy_k, y_k = dy, y
    dg_init = torch.randn(C, device="cuda", generator=gen)
    db_init = torch.randn(C, device="cuda", generator=gen)
    dx = Guarded(P, C, C, torch.bfloat16, extra_rows=0, tail=4096)
    dg = Guarded(1, C, C, torch.float32, extra_rows=0, tail=64).fill_(dg_init[None])
    db = Guarded(1, C, C, torch.float32, extra_rows=0, tail=64).fill_(db_init[None])
    _lib.check(lib.vdk_layernorm_bwd(dy_k.data_ptr(), y_k.data_ptr(), rstd.data_ptr(), B, H, W, C, gamma.data_ptr(),
                                     beta.data_ptr(), patch, dx.ptr(), add.data_ptr(), dg.ptr(), db.ptr(), _lib.stream_ptr()),
               "ln_bwd")
    torch.cuda.synchronize()
    dx_ref, _, db_ref, m1, m2 = layernorm_bwd_reference(xhat, rstd64, gamma, dy, add, patch)
    e32, _, db_b = layernorm_bwd_bound(xhat, rstd64, gamma, beta, y, dy, add, m1, m2, L, dg_init, db_init)
    tag = f"ln_bwd C={C} LPP={L['lpp']} IT={L['it']} U={L['u']} patch={patch}"
    check_within(dx.view, dx_ref, bf16_store_bound(dx_ref, e32), tag + " dx",
                 lambda bad: describe_pixels(bad.any(-1), P, L), STATS)
    keep = gamma != 0
    dg_ref, dg_b = layernorm_bwd_dgamma(y, beta, gamma, dy, L, dg_init)  # against the xhat the saved y holds
    check_within(dg.view[0][keep], dg_ref[keep], dg_b[keep], tag + " dgamma",
                 lambda bad: f"channels {keep.nonzero().flatten()[bad.nonzero().flatten()][:8].tolist()}", STATS)
    # gamma = 0: y holds no trace of xhat, so that channel's dgamma receives nothing and keeps its initial value
    assert float(dg.view[0][5]) == float(dg_init[5])
    check_within(db.view[0], db_init.double() + db_ref, db_b, tag + " dbeta",
                 lambda bad: f"channels {bad.nonzero().flatten()[:8].tolist()}", STATS)
    for name, buf in (("dx", dx), ("dgamma", dg), ("dbeta", db)):
        assert not buf.guard_errors(), f"{name}: " + buf.guard_errors()


# ------------------------------------------------------------------------------------------------------------------------------
# BatchNorm with batch statistics: forward (+ running statistics) and backward (dweight / dbias +=)

# (R, C, dtype, mean): the 8-channel vector kernel (bf16, C % 8 == 0) at the neck's BN2d of ConvNeXt-B at batch 128
# (R = 49 x 128, C = 1024) and at R = 2, the generic bf16 kernel (C = 100), the fp32 kernel; means near 0 and at 100
BN_CASES = [(49 * 128, 1024, torch.bfloat16, 0.4), (2, 1024, torch.bfloat16, 0.4), (49 * 128, 1024, torch.bfloat16, 100.0),
            (300, 100, torch.bfloat16, 0.4), (6272, 100, torch.bfloat16, 100.0), (2, 100, torch.bfloat16, 0.4),
            (300, 200, torch.float32, 0.4), (6272, 1024, torch.float32, 100.0), (2, 64, torch.float32, 0.4)]


@pytest.mark.parametrize("R,C,dt,mean", BN_CASES, ids=[f"R{c[0]}-C{c[1]}-{str(c[2])[6:]}-mean{c[3]:g}" for c in BN_CASES])
def test_batchnorm_train_elementwise(lib, R, C, dt, mean):
    gen = torch.Generator(device="cuda").manual_seed(R + C)
    x = (torch.randn(R, C, device="cuda", generator=gen) * 1.5 + mean).to(dt)
    w = 0.5 + torch.rand(C, device="cuda", generator=gen)
    b = 0.2 * torch.randn(C, device="cuda", generator=gen)
    rm0 = torch.randn(C, device="cuda", generator=gen)
    rv0 = 1 + torch.rand(C, device="cuda", generator=gen)
    rm, rv = rm0.clone(), rv0.clone()
    y = Guarded(R, C, C, dt, extra_rows=0, tail=256)
    smean, srstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    is_bf16 = int(dt == torch.bfloat16)
    tag = f"batchnorm R={R} C={C} {'bf16' if is_bf16 else 'fp32'} mean={mean:g}"
    _lib.check(lib.vdk_batchnorm_train_fwd(x.data_ptr(), R, C, is_bf16, w.data_ptr(), b.data_ptr(), 1e-5, 0.1, y.ptr(),
                                           smean.data_ptr(), srstd.data_ptr(), rm.data_ptr(), rv.data_ptr(), _lib.stream_ptr()), tag)
    torch.cuda.synchronize()
    ref = batchnorm_fwd_reference(x, w, b, 1e-5, 0.1, rm0, rv0)
    yb, rb, mub, rmb, rvb = batchnorm_fwd_bound(ref, w, b, 1e-5, 0.1, rm0, rv0, dt)
    rows = lambda bad: f"rows {bad.any(-1).nonzero().flatten()[:6].tolist()}, channels {bad.any(0).nonzero().flatten()[:6].tolist()}"
    chans = lambda bad: f"channels {bad.nonzero().flatten()[:8].tolist()} (8-channel blocks or 32-channel blocks)"
    check_within(y.view, ref["y"], yb, tag + " y", rows, STATS)
    check_within(srstd, ref["rstd"], rb, tag + " rstd", chans, STATS)
    check_within(smean, ref["mu"], mub, tag + " mean", chans, STATS)
    check_within(rm, ref["rm"], rmb, tag + " running_mean", chans, STATS)
    check_within(rv, ref["rv"], rvb, tag + " running_var", chans, STATS)
    assert not y.guard_errors(), y.guard_errors()
    dy = (torch.randn(R, C, device="cuda", generator=gen)).to(dt)
    dw0, db0 = torch.randn(C, device="cuda", generator=gen), torch.randn(C, device="cuda", generator=gen)
    dw, db = dw0.clone(), db0.clone()
    dx = Guarded(R, C, C, dt, extra_rows=0, tail=256)
    _lib.check(lib.vdk_batchnorm_train_bwd(dy.data_ptr(), x.data_ptr(), R, C, is_bf16, w.data_ptr(), smean.data_ptr(),
                                           srstd.data_ptr(), dx.ptr(), dw.data_ptr(), db.data_ptr(), _lib.stream_ptr()), tag)
    torch.cuda.synchronize()
    bref = batchnorm_bwd_reference(x, dy, w, smean, srstd)
    dxb, dwb, dbb = batchnorm_bwd_bound(bref, w, srstd, dw0, db0, dt)
    check_within(dx.view, bref["dx"], dxb, tag + " dx", rows, STATS)
    check_within(dw, dw0.double() + bref["dw"], dwb, tag + " dweight", chans, STATS)
    check_within(db, db0.double() + bref["db"], dbb, tag + " dbias", chans, STATS)
    assert not dx.guard_errors(), dx.guard_errors()
