"""CPU checks of the optimizer references in tests/optim_ref.py: the exact fmaf emulation against rational arithmetic, the exact
sum of squares against math.fsum, the fp64 semantic reference against torch.optim.SGD + clip_grad_norm_ + ModelEMA on fp64
parameters, and the skip-on-non-finite rule against torch's own GradScaler."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from optim_ref import (F32, ema_decay, exact_sumsq, fmaf, fmaf_exact, kernel_step, reference_step, round_fraction_to_f32,
                       step_bounds, sumsq_depth)


def _bits(x):
    return np.asarray(x, F32).view(np.uint32)


def test_round_fraction_to_f32_matches_numpy_on_doubles():
    rng = np.random.default_rng(0)
    xs = np.concatenate([rng.standard_normal(2000) * 10.0 ** rng.integers(-45, 39, 2000), [1e-46, -3e-45, 3.5e38, -1e39]])
    got = np.array([round_fraction_to_f32(Fraction(float(x))) for x in xs], F32)
    with np.errstate(over="ignore"):
        want = xs.astype(F32)   # one rounding of an fp64 value: correct, no double rounding involved
    assert np.array_equal(_bits(got), _bits(want))


def test_fmaf_emulation_equals_rational_fma_on_random_triples():
    rng = np.random.default_rng(1)
    n = 6000
    scale = lambda lo, hi: 2.0 ** rng.integers(lo, hi, n)
    a = (rng.standard_normal(n) * scale(-30, 30)).astype(F32)
    b = (rng.standard_normal(n) * scale(-30, 30)).astype(F32)
    c = (rng.standard_normal(n) * scale(-60, 60)).astype(F32)
    c[:500] = -(a[:500].astype(np.float64) * b[:500]).astype(F32)          # heavy cancellation
    a[500:700] = (rng.standard_normal(200) * 2.0 ** -75).astype(F32)       # products in the fp32 subnormal range
    c[500:700] = (rng.standard_normal(200) * 2.0 ** -140).astype(F32)
    got = fmaf(a, b, c)
    want = np.array([fmaf_exact(x, y, z) for x, y, z in zip(a, b, c)], F32)
    assert np.array_equal(_bits(got), _bits(want))


def test_fmaf_emulation_is_right_on_midpoints_where_double_rounding_is_wrong():
    """c + a*b with a*b = +-2^-24 * (1 + k u)(1 - k u) * ulp-scale: the fp64 sum lands exactly on an fp32 midpoint while the exact
    value lies k^2 * 2^-47 ulps to one side of it (below fp64's resolution for k < 128).  Rounding fp64 then fp32 goes to the
    even neighbour, which is the wrong one whenever c's last mantissa bit is odd; fmaf must not."""
    rng = np.random.default_rng(2)
    n = 3000
    u = 2.0 ** -23
    c = (1 + rng.integers(0, 2 ** 23, n) * u) * 2.0 ** rng.integers(-20, 20, n)
    c = c.astype(F32)
    half_ulp = np.ldexp(1.0, np.frexp(c.astype(np.float64))[1] - 25)        # half an fp32 ulp of c
    k = rng.integers(1, 128, n)
    sign = rng.choice([-1.0, 1.0], n)
    a = (sign * half_ulp * (1 + k * u)).astype(F32)
    b = (1 - k * u).astype(F32)
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
    got = fmaf(a, b, c)
    want = np.array([fmaf_exact(x, y, z) for x, y, z in zip(a, b, c)], F32)
    assert np.array_equal(_bits(got), _bits(want))
    wrong = int((_bits(naive) != _bits(want)).sum())
    assert wrong > n // 4, f"only {wrong} crafted cases defeat double rounding"


def test_exact_sumsq_matches_fsum_and_fractions():
    rng = np.random.default_rng(3)
    for g in (rng.standard_normal(10001).astype(F32),
              (rng.standard_normal(3000) * 10.0 ** rng.uniform(-30, 30, 3000)).astype(F32),
              np.array([1e-45, 3e-42, -2e-39, 3.4e38], F32), np.zeros(7, F32), np.zeros(0, F32)):
        s = exact_sumsq(g)
        assert s == sum((Fraction(float(v)) ** 2 for v in g), Fraction(0))
        assert float(s) == math.fsum(float(v) * float(v) for v in g)


def test_sumsq_depth_counts_the_kernel_chain():
    assert sumsq_depth(3) == 1 + 8 + 1 + 8 + 1
    assert sumsq_depth(4 * 256 * 1184) == 4 + 1 + 8 + 5 + 8 + 1
    assert sumsq_depth(4 * 256 * 1184 + 4) == 8 + 1 + 8 + 5 + 8 + 1


# ---- fp64 reference against torch ---------------------------------------------------------------------------------------
class _EMA:
    """models/ema.py ModelEMA.update restated on a parameter list."""

    def __init__(self, params):
        self.v = [p.detach().clone() for p in params]
        self.updates = 0

    def update(self, params):
        self.updates += 1
        d, omd = ema_decay(self.updates)
        for v, p in zip(self.v, params):
            v.mul_(d).add_(omd * p.detach())


CASES = {  # name: (max_norm, momentum schedule, weight decay)
    "clip_active": (0.5, [0.9] * 5, 5e-4),
    "clip_inactive": (1e6, [0.9] * 5, 5e-4),
    "momentum_0": (0.5, [0.0] * 5, 5e-4),
    "weight_decay_0": (0.5, [0.8] * 5, 0.0),
    "momentum_switch": (0.5, [0.8, 0.8, 0.9, 0.9, 0.9], 5e-4),
    "momentum_from_0": (0.5, [0.0, 0.0, 0.9, 0.9, 0.0, 0.9], 5e-4),
}


@pytest.mark.parametrize("case", list(CASES))
def test_fp64_reference_equals_torch_sgd_clip_and_ema(case):
    max_norm, moms, wd = CASES[case]
    gen = torch.Generator().manual_seed(4)
    shapes = [(7, 5), (5,), (13,)]
    params = [torch.nn.Parameter(torch.randn(s, generator=gen, dtype=torch.float64)) for s in shapes]
    lrs = [0.05, 0.5, 0.5]
    opt = torch.optim.SGD([{"params": params[:1], "lr": lrs[0]}, {"params": params[1:], "lr": lrs[1]}], lr=lrs[0],
                          momentum=moms[0], weight_decay=wd)
    ema = _EMA(params)
    ours = [p.detach().numpy().ravel().copy() for p in params]
    mom = [np.zeros_like(x) for x in ours]
    ev = [x.copy() for x in ours]
    has_buf = [False] * 3
    for t, m in enumerate(moms):
        for pg in opt.param_groups:
            pg["momentum"] = m
        grads = [torch.randn(s, generator=gen, dtype=torch.float64) * (t + 1) for s in shapes]
        for p, g in zip(params, grads):
            p.grad = g.clone()
        torch.nn.utils.clip_grad_norm_(params, max_norm)
        opt.step()
        ema.update(params)
        d, omd = ema_decay(ema.updates)
        S = sum(float((g.double() ** 2).sum()) for g in grads)
        assert (max_norm / (math.sqrt(S) + 1e-6) < 1) == (case != "clip_inactive")
        for i in range(3):
            ours[i], mom[i], ev[i], has_buf[i], applied = reference_step(
                ours[i], grads[i].numpy().ravel(), mom[i], ev[i], S, max_norm, lrs[i], m, wd, has_buf[i], d, omd)
            assert applied
            np.testing.assert_allclose(ours[i], params[i].detach().numpy().ravel(), rtol=1e-13, atol=1e-15)
            np.testing.assert_allclose(ev[i], ema.v[i].numpy().ravel(), rtol=1e-13, atol=1e-15)
            st = opt.state.get(params[i], {})
            assert has_buf[i] == ("momentum_buffer" in st)
            if has_buf[i]:
                np.testing.assert_allclose(mom[i], st["momentum_buffer"].numpy().ravel(), rtol=1e-13, atol=1e-15)


# ---- the skip rule, from torch's GradScaler ------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("when", ["first", "later"])
def test_gradscaler_skips_sgd_on_nonfinite_gradient_and_reference_agrees(bad, when):
    """GradScaler("cpu") on an fp32 model: with one non-finite gradient after unscale_, scaler.step does not call
    optimizer.step (parameters unchanged, no momentum buffer created or advanced); zero_grad and the EMA still run.  The fp64
    reference's skip reproduces the same trajectory, including the first applied step cloning its update into the buffer."""
    torch.manual_seed(5)
    model = torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.Linear(4, 3))
    params = list(model.parameters())
    opt = torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=5e-4)
    scaler = torch.amp.GradScaler("cpu", init_scale=2.0 ** 10, growth_interval=1000)
    ema = _EMA(params)
    bad_step = 0 if when == "first" else 2
    ref_p = [p.detach().double().numpy().ravel().copy() for p in params]
    ref_m = [np.zeros_like(x) for x in ref_p]
    ref_e = [x.copy() for x in ref_p]
    has_buf = False
    for t in range(4):
        x, y = torch.randn(8, 6), torch.randint(0, 3, (8,))
        loss = torch.nn.functional.cross_entropy(model(x), y)
        scaler.scale(loss).backward()
        if t == bad_step:
            params[1].grad[2] = bad
        before = [p.detach().clone() for p in params]
        buf_before = [opt.state.get(p, {}).get("momentum_buffer") for p in params]
        buf_before = [None if b is None else b.clone() for b in buf_before]
        scaler.unscale_(opt)
        grads = [p.grad.detach().double().numpy().ravel().copy() for p in params]
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=False)
        ema.update(params)
        d, omd = ema_decay(ema.updates)
        with np.errstate(over="ignore", invalid="ignore"):
            S = float(sum((g * g).sum() for g in grads))
        applied_all = []
        for i in range(len(params)):
            ref_p[i], ref_m[i], ref_e[i], hb, applied = reference_step(
                ref_p[i], grads[i], ref_m[i], ref_e[i], S, 10.0, 0.1, 0.9, 5e-4, has_buf, d, omd)
            applied_all.append(applied)
        has_buf = hb
        if t == bad_step:
            assert not any(applied_all)
            for p, b in zip(params, before):
                assert torch.equal(p.detach(), b), "GradScaler applied a step with a non-finite gradient"
            for p, b in zip(params, buf_before):
                st = opt.state.get(p, {})
                if b is None:
                    assert "momentum_buffer" not in st, "a skipped first step created the momentum buffer"
                else:
                    assert torch.equal(st["momentum_buffer"], b), "a skipped step advanced the momentum buffer"
        else:
            assert all(applied_all)
        assert all(bool((p.grad == 0).all()) for p in params)
        for i, p in enumerate(params):
            np.testing.assert_allclose(ref_p[i], p.detach().double().numpy().ravel(), rtol=2e-6, atol=1e-7)
            np.testing.assert_allclose(ref_e[i], ema.v[i].double().numpy().ravel(), rtol=2e-6, atol=1e-7)
            if "momentum_buffer" in opt.state.get(p, {}):
                np.testing.assert_allclose(ref_m[i], opt.state[p]["momentum_buffer"].double().numpy().ravel(), rtol=2e-6,
                                           atol=1e-7)
    assert has_buf


# ---- the restatement against the reference, within the bound ------------------------------------------------------------
@pytest.mark.parametrize("sumsq_scale", [1e-4, 1.0, 1e4])
@pytest.mark.parametrize("momentum,has_buf", [(0.9, True), (0.9, False), (0.0, False)])
def test_kernel_restatement_lies_within_the_bound_of_the_reference(sumsq_scale, momentum, has_buf):
    """The bound is a bound on the kernel's fp32 sequence: kernel_step, the bit-exact restatement, must satisfy it."""
    rng = np.random.default_rng(6)
    n = 20000
    p = rng.standard_normal(n).astype(F32)
    g = (rng.standard_normal(n) * math.sqrt(sumsq_scale / n) * 40).astype(F32)
    mom = (rng.standard_normal(n) * 0.1).astype(F32)
    ema = rng.standard_normal(n).astype(F32)
    S = float(exact_sumsq(g))
    lr, wd = F32(0.1), F32(5e-4)
    for updates in (1, 2000, 10 ** 6):
        d, omd = ema_decay(updates)
        d32, omd32 = float(F32(d)), float(F32(omd))
        kp, _, km, ke = kernel_step(p, g, mom, ema, S, 10.0, lr, momentum, wd, not has_buf, d32, omd32, 1)
        rp, rm, re, _, _ = reference_step(p, g, mom, ema, S, 10.0, float(lr), float(F32(momentum)), float(wd), has_buf,
                                          d32, omd32)
        e_p, e_m, e_e = step_bounds(p, g, mom, ema, S, 10.0, float(lr), float(F32(momentum)), float(wd), has_buf, d32,
                                    omd32, sumsq_depth(n))
        assert (np.abs(kp - rp) <= e_p).all()
        assert (np.abs(ke - re) <= e_e).all()
        if momentum != 0:
            assert (np.abs(km - rm) <= e_m).all()
        else:
            assert np.array_equal(km, mom)
