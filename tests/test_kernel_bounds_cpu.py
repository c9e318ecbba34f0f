"""CPU self-tests of the ConvNeXt kernel bounds in kernel_ref.py: an fp32 emulation of each kernel's arithmetic, in the
kernel's order, must stay inside its bound, and a plausible defect (a missing image of a group, a tap one pixel off, a
dropped addend, another pixel's statistics) must fall outside it."""
import math

import torch

from kernel_ref import (bf16_store_bound, dwconv7_bwd_data_bound, dwconv7_reference, layernorm_bwd_bound,
                        layernorm_bwd_reference, wgrad_bound, wgrad_reference)


def within(got, ref, bound):
    return bool(((got.double() - ref).abs() <= bound).all())


def bf16(t):
    return t.to(torch.bfloat16)


def emulate_wgrad(x, g, init, T, ipc, skip_image=None):
    """dwconv7_wgrad_kernel in fp32: per image group, each (strip half, filter row) thread chains its images, tile rows
    and strip pixels; the halves are added; each group's partial is added to the output.  One tile covers the image."""
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.float(), (0, 0, 3, 3, 3, 3))
    gf = g.float()
    nh = -(-T // 7)
    out = init.clone().float()
    for b0 in range(0, B, ipc):
        halves = [torch.zeros(49, C) for _ in range(nh)]
        for b in range(b0, min(B, b0 + ipc)):
            if b == skip_image:
                continue
            for py in range(H):
                for px in range(W):
                    win = xp[b, py:py + 7, px:px + 7, :].reshape(49, C)
                    halves[px // 7] = halves[px // 7] + gf[b, py, px] * win  # exact bf16 products, one rounding each
        s = torch.zeros(49, C)
        for h in halves:
            s = s + h
        out = out + s
    return out


def test_wgrad_bound_holds_for_kernel_order_and_catches_a_missing_image():
    torch.manual_seed(0)
    B, H, W, C, ipc = 5, 9, 9, 16, 2
    x, g = bf16(torch.randn(B, H, W, C)), bf16(torch.randn(B, H, W, C))
    init = torch.randn(49, C)
    launch = dict(T=9, nh=2, ipc=ipc, groups=3, tiles=1)
    ref, mag, _, _ = wgrad_reference(x, g)
    bound = wgrad_bound(mag, init, launch)
    assert within(emulate_wgrad(x, g, init, 9, ipc), init.double() + ref, bound)
    assert not within(emulate_wgrad(x, g, init, 9, ipc, skip_image=4), init.double() + ref, bound)


def emulate_dwconv_mode1(x, w49, add, shift=0):
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.float(), (0, 0, 3, 3 + abs(shift), 3, 3))
    acc = torch.zeros(B, H, W, C)
    for t in range(49):
        dy, dx = divmod(t, 7)
        if t == 48:
            dx += shift
        acc = acc + w49[t] * xp[:, dy:dy + H, dx:dx + W, :]
    return bf16(acc + add.float())


def test_dwconv_bwd_data_bound_holds_and_catches_a_shifted_tap():
    torch.manual_seed(1)
    x, add = bf16(torch.randn(2, 9, 11, 24)), bf16(torch.randn(2, 9, 11, 24))
    w49 = 0.2 * torch.randn(49, 24)
    ref, mag = dwconv7_reference(x, w49)
    ref += add.double()
    bound = dwconv7_bwd_data_bound(ref, mag, add)
    assert within(emulate_dwconv_mode1(x, w49, add), ref, bound)
    assert not within(emulate_dwconv_mode1(x, w49, add, shift=1), ref, bound)
    assert not within(emulate_dwconv_mode1(x, w49, torch.zeros_like(add)), ref, bound)


def emulate_ln_bwd_dx(dy, y, rstd, gamma, beta, add, lpp, it):
    """ln_bwd_kernel's dx in fp32: lane `sub` of a pixel's LPP lanes sums channels (sub + i LPP) 8 + j in (i, j) order,
    the lanes meet in an xor butterfly, then o = rs (g - m1 - h m2) + addend."""
    P, C = dy.shape
    w = gamma.clone()
    iw = torch.where(w == 0, torch.zeros_like(w), 1.0 / w)
    dyf, yf = dy.float(), y.float()
    h = (yf - beta) * iw
    g = dyf * w
    s1 = torch.zeros(P, lpp)
    s2 = torch.zeros(P, lpp)
    for sub in range(lpp):
        for i in range(it):
            for j in range(8):
                c = (sub + i * lpp) * 8 + j
                if c < C:
                    s1[:, sub] = s1[:, sub] + g[:, c]
                    s2[:, sub] = s2[:, sub] + g[:, c] * h[:, c]
    lanes = torch.arange(lpp)
    off = lpp // 2
    while off > 0:
        s1 = s1 + s1[:, lanes ^ off]
        s2 = s2 + s2[:, lanes ^ off]
        off //= 2
    inv_c = torch.tensor(1.0 / C, dtype=torch.float32)
    m1, m2 = s1[:, :1] * inv_c, s2[:, :1] * inv_c
    o = rstd[:, None] * (g - m1 - h * m2)
    return bf16(o + add.float())


def ln_inputs(P, C, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(P, C, dtype=torch.float64, generator=gen) * 2 + 0.3
    mean = x.mean(-1, keepdim=True)
    rstd64 = ((x - mean).pow(2).mean(-1) + 1e-6).rsqrt()
    xhat = (x - mean) * rstd64[:, None]
    gamma = (0.2 + 1.3 * torch.rand(C, generator=gen)).float()
    beta = 0.2 * torch.randn(C, generator=gen)
    far = torch.arange(C) % 8 == 3
    beta[far] = gamma[far] * 30
    gamma[5], beta[5] = 0.0, 0.1
    y = bf16((gamma.double() * xhat + beta.double()).float())
    return xhat, rstd64, gamma, beta, y, bf16(torch.randn(P, C, generator=gen)), bf16(torch.randn(P, C, generator=gen))


def test_ln_bwd_bound_holds_and_needs_the_saved_output_term():
    P, C, lpp, it = 64, 80, 16, 1
    xhat, rstd64, gamma, beta, y, dy, add = ln_inputs(P, C, 2)
    launch = dict(lpp=lpp, it=it, u=4, blocks=1, max_trips=1)
    ref, _, _, m1, m2 = layernorm_bwd_reference(xhat, rstd64, gamma, dy, add, 1)
    zeros = torch.zeros(C)
    e32, _, _ = layernorm_bwd_bound(xhat, rstd64, gamma, beta, y, dy, add, m1, m2, launch, zeros, zeros)
    bound = bf16_store_bound(ref, e32)
    got = emulate_ln_bwd_dx(dy, y, rstd64.float(), gamma, beta, add, lpp, it)
    assert within(got, ref, bound)
    # defects: another pixel's rstd, a dropped addend
    assert not within(emulate_ln_bwd_dx(dy, y, rstd64.float().roll(1), gamma, beta, add, lpp, it), ref, bound)
    assert not within(emulate_ln_bwd_dx(dy, y, rstd64.float(), gamma, beta, torch.zeros_like(add), lpp, it), ref, bound)
    # the ulp(y) / |gamma| term is what covers the |beta / gamma| = 30 channels: a bound that assumes an exact xhat fails
    exact_y = bf16_store_bound(ref, layernorm_bwd_bound(xhat, rstd64, gamma, beta, (gamma.double() * xhat + beta.double()),
                                                        dy, add, m1, m2, launch, zeros, zeros)[0])
    assert not within(got, ref, exact_y)
    assert math.isfinite(float(bound.max()))


def test_wgrad_dbias_bound_catches_a_missing_image():
    torch.manual_seed(3)
    B, H, W, C, ipc = 5, 9, 9, 16, 2
    x, g = bf16(torch.randn(B, H, W, C)), bf16(torch.randn(B, H, W, C))
    init = torch.randn(1, C)
    launch = dict(T=9, nh=2, ipc=ipc, groups=3, tiles=1)
    _, _, bref, bmag = wgrad_reference(x, g)
    bound = wgrad_bound(bmag[None], init, launch)

    def emulate(skip=None):
        out = init.clone()
        for b0 in range(0, B, ipc):
            s = torch.zeros(1, C)
            for b in range(b0, min(B, b0 + ipc)):
                if b != skip:
                    for row in g[b].float().reshape(-1, C):
                        s = s + row
            out = out + s
        return out
    assert within(emulate(), init.double() + bref[None], bound)
    assert not within(emulate(skip=3), init.double() + bref[None], bound)


def emulate_dwconv_ln(x, w49, bias, gamma, beta, eps, chunk, stats_shift=0):
    """Mode 0 in fp32: z = bias + 49 FMAs; per-chunk two-pass (mean, M2), Chan's combination; y = (z - m) rstd g + b.
    stats_shift rolls the statistics by that many pixels (another tile's statistics)."""
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.float(), (0, 0, 3, 3, 3, 3))
    z = bias.float().expand(B, H, W, C).clone()
    for t in range(49):
        dy, dx = divmod(t, 7)
        z = z + w49[t] * xp[:, dy:dy + H, dx:dx + W, :]
    zk = z.unflatten(-1, (C // chunk, chunk))
    mk = zk.sum(-1) * torch.tensor(1.0 / chunk, dtype=torch.float32)
    m2k = (zk - mk[..., None]).pow(2).sum(-1)
    m = mk.sum(-1) * torch.tensor(1.0 / (C // chunk), dtype=torch.float32)
    q = (chunk * (mk - m[..., None]).pow(2) + m2k).sum(-1)
    r = torch.rsqrt(q * torch.tensor(1.0 / C, dtype=torch.float32) + eps)
    if stats_shift:
        m, r = m.roll(stats_shift, 2), r.roll(stats_shift, 2)
    return bf16((z - m[..., None]) * r[..., None] * gamma + beta), r


def test_dwconv_ln_bound_holds_with_chunk_means_far_apart_and_catches_wrong_statistics():
    from kernel_ref import dwconv7_ln_bound, dwconv7_ln_reference
    torch.manual_seed(4)
    B, H, W, C, chunk = 2, 7, 9, 64, 16
    x = bf16(torch.randn(B, H, W, C))
    w49 = 0.2 * torch.randn(49, C)
    gamma, beta = 1 + 0.3 * torch.randn(C), 0.2 * torch.randn(C)
    for bias in (0.3 * torch.randn(C), 1e3 * (torch.arange(C) // chunk).float(), 1e3 + 0.3 * torch.randn(C)):
        ref = dwconv7_ln_reference(x, w49, bias, gamma, beta, 1e-6)
        yb, rb = dwconv7_ln_bound(ref, gamma, beta, 1e-6, chunk)
        got, r = emulate_dwconv_ln(x, w49, bias, gamma, beta, 1e-6, chunk)
        assert within(got, ref["y"], yb) and within(r, ref["rstd"], rb)
        bad, _ = emulate_dwconv_ln(x, w49, bias, gamma, beta, 1e-6, chunk, stats_shift=1)
        assert not within(bad, ref["y"], yb)
    bias = 0.3 * torch.randn(C)
    ref = dwconv7_ln_reference(x, w49, bias, gamma, beta, 1e-6)
    yb, _ = dwconv7_ln_bound(ref, gamma, beta, 1e-6, chunk)
    assert not within(emulate_dwconv_ln(x, w49.roll(1, 0), bias, gamma, beta, 1e-6, chunk)[0], ref["y"], yb)


def test_batchnorm_bounds_hold_with_a_far_mean_and_catch_a_missing_row():
    from kernel_ref import batchnorm_bwd_bound, batchnorm_bwd_reference, batchnorm_fwd_bound, batchnorm_fwd_reference
    torch.manual_seed(5)
    R, C = 40, 16
    for mean in (0.4, 100.0):
        x = bf16(torch.randn(R, C) * 1.5 + mean)
        w, b = 0.5 + torch.rand(C), 0.2 * torch.randn(C)
        rm, rv = torch.randn(C), 1 + torch.rand(C)
        ref = batchnorm_fwd_reference(x, w, b, 1e-5, 0.1, rm, rv)
        yb, rb, mub, rmb, rvb = batchnorm_fwd_bound(ref, w, b, 1e-5, 0.1, rm, rv, torch.bfloat16)
        xf = x.float()
        mu = xf.sum(0) * torch.tensor(1.0 / R, dtype=torch.float32)   # the vector kernel's order
        q = (xf - mu).pow(2).sum(0)
        r = torch.rsqrt(q * torch.tensor(1.0 / R, dtype=torch.float32) + 1e-5)
        sc = r * w
        y = bf16(xf * sc + (b - mu * sc))
        assert within(y, ref["y"], yb) and within(r, ref["rstd"], rb) and within(mu, ref["mu"], mub)
        assert within(0.9 * rm + 0.1 * mu, ref["rm"], rmb) and within(0.9 * rv + 0.1 * q / (R - 1), ref["rv"], rvb)
        mu_short = xf[:-1].sum(0) / (R - 1)   # a dropped row
        assert not within(mu_short, ref["mu"], mub)
        dy = bf16(torch.randn(R, C))
        dw0, db0 = torch.randn(C), torch.randn(C)
        bref = batchnorm_bwd_reference(x, dy, w, mu, r)
        dxb, dwb, dbb = batchnorm_bwd_bound(bref, w, r, dw0, db0, torch.bfloat16)
        g = dy.float()
        xh = (xf - mu) * r
        s1, s2 = g.sum(0), (g * xh).sum(0)
        dx = bf16(w * r * (g - s1 / R - xh * (s2 / R)))
        assert within(dx, bref["dx"], dxb) and within(dw0 + s2, dw0.double() + bref["dw"], dwb)
        assert within(db0 + s1, db0.double() + bref["db"], dbb)
        assert not within(db0 + g[1:].sum(0), db0.double() + bref["db"], dbb)
        assert not within(dw0 + (g * xh)[1:].sum(0), dw0.double() + bref["dw"], dwb)


def test_ln_bwd_dgamma_bound_catches_a_dropped_trip():
    from kernel_ref import layernorm_bwd_dgamma
    P, C = 12, 80
    xhat, rstd64, gamma, beta, y, dy, add = ln_inputs(P, C, 6)
    launch = dict(lpp=32, it=3, u=1, blocks=1, max_trips=6)   # 2 warps of one pixel per trip, 6 trips each
    init = torch.randn(C)
    ref, bound = layernorm_bwd_dgamma(y, beta, gamma, dy, launch, init)
    keep = gamma != 0
    iw = torch.where(gamma == 0, torch.zeros_like(gamma), 1.0 / gamma)
    h = (y.float() - beta) * iw

    def emulate(drop=None):
        out = init.clone()
        for w in range(2):
            acc = torch.zeros(C)
            for p in range(w, P, 2):
                if p != drop:
                    acc = acc + dy[p].float() * h[p]
            out = out + acc
        return out
    assert within(emulate()[keep], ref[keep], bound[keep])
    assert not within(emulate(drop=7)[keep], ref[keep], bound[keep])
