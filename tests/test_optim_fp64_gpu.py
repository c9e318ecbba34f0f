"""The fused clip + SGD + EMA step (csrc/optim.cu) against tests/optim_ref.py: each kernel called directly through the C ABI
(bit for bit against the numpy restatement of its fp32 sequence, and within the derived bound of the fp64 reference), then
FusedSGDClipEMA as the face trainer drives it (full-size groups, resume, no host sync, pack invalidation, non-finite gradients).
The bounds and the restatement are derived in tests/optim_ref.py's docstring."""
import copy
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from optim_ref import (F32, U64, GuardedVec, ema_bound, ema_decay, exact_sumsq, kernel_coef, kernel_ema, kernel_step,
                       reference_step, step_bounds, sumsq_depth)
from visiondk_b200 import _lib
from visiondk_b200.optim import FusedSGDClipEMA
from visiondk_b200.train import cosine_with_warm_lr

pytestmark = pytest.mark.gpu
RED_EDGE = 4 * 256 * 1184        # n at which vdk_grad_sumsq's partial count reaches kRedBlocksMax
STEP_EDGE = 132 * 16 * 256       # n at which the step's grid reaches its cap and the grid-stride loop starts a second lap


def _bits(x):
    return np.asarray(x, F32).view(np.uint32)


def _assert_bits(got, want, what):
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert bad.size == 0, (f"{what}: {bad.size} elements differ from the restatement, first at {bad[:5].tolist()}: "
                           f"got {np.asarray(got)[bad[:3]]}, want {np.asarray(want)[bad[:3]]}")


def _within(got, ref, bound, what):
    err = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    bad = ~(err <= np.asarray(bound))
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the bound, first at {np.flatnonzero(bad)[:5].tolist()}"


@pytest.fixture(scope="module")
def ws(lib):
    return torch.empty(lib.vdk_grad_sumsq_workspace_bytes(), dtype=torch.uint8, device="cuda")


def _sumsq(lib, gv, ws, acc=None, accumulate=0):
    acc = torch.zeros((), dtype=torch.float64, device="cuda") if acc is None else acc
    _lib.check(lib.vdk_grad_sumsq(gv.ptr(), gv.n, acc.data_ptr(), accumulate, ws.data_ptr(), ws.numel(), _lib.stream_ptr()),
               "vdk_grad_sumsq")
    torch.cuda.synchronize()
    return acc


def _check_sumsq(lib, g, ws):
    gv = GuardedVec(torch.from_numpy(g))
    got = float(_sumsq(lib, gv, ws).item())
    exact = exact_sumsq(g)
    assert abs(Fraction(got) - exact) <= Fraction(sumsq_depth(g.size) * U64) * exact, (g.size, got, float(exact))
    assert not gv.guard_errors()
    return got


# ---- vdk_grad_sumsq -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", list(range(10)) + [1023, 1024, 1025] + [RED_EDGE + k for k in range(-5, 6)] + [3_000_001])
def test_grad_sumsq_is_the_exact_sum_within_its_depth(lib, ws, n):
    g = np.random.default_rng(n).standard_normal(n).astype(F32)
    got = _check_sumsq(lib, g, ws)
    if n == 0:
        assert got == 0.0


@pytest.mark.parametrize("kind", ["zeros", "subnormals", "near_flt_max", "wide_mixture"])
@pytest.mark.parametrize("n", [7, 100_003])
def test_grad_sumsq_contents(lib, ws, kind, n):
    rng = np.random.default_rng(11)
    if kind == "zeros":
        g = np.zeros(n, F32)
    elif kind == "subnormals":
        g = (rng.standard_normal(n) * 2.0 ** -135).astype(F32)
        assert (np.abs(g) < np.finfo(F32).tiny).all() and (g != 0).any()
    elif kind == "near_flt_max":
        g = rng.standard_normal(n).astype(F32)
        g[n // 2] = np.finfo(F32).max * F32(0.99)
    else:
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(F32)
    got = _check_sumsq(lib, g, ws)
    if kind == "zeros":
        assert got == 0.0


@pytest.mark.slow
def test_grad_sumsq_convnext_b_sized_group(lib, ws):
    n = 88_000_003
    g = (np.random.default_rng(12).standard_normal(n, dtype=np.float32) * F32(1e-3))
    _check_sumsq(lib, g, ws)


def test_grad_sumsq_accumulates_overwrites_and_repeats_bitwise(lib, ws):
    g1 = np.random.default_rng(13).standard_normal(50_001).astype(F32)
    g2 = np.random.default_rng(14).standard_normal(3_001).astype(F32)
    v1, v2 = GuardedVec(torch.from_numpy(g1)), GuardedVec(torch.from_numpy(g2))
    acc = torch.full((), float("nan"), dtype=torch.float64, device="cuda")
    _sumsq(lib, v1, ws, acc, accumulate=0)          # overwrites the NaN
    first = float(acc.item())
    _sumsq(lib, v2, ws, acc, accumulate=1)
    both = exact_sumsq(g1) + exact_sumsq(g2)
    depth = max(sumsq_depth(g1.size), sumsq_depth(g2.size)) + 1
    assert abs(Fraction(float(acc.item())) - both) <= Fraction(depth * U64) * both
    repeats = {float(_sumsq(lib, v1, ws).item()) for _ in range(3)}
    assert repeats == {first}


def test_grad_sumsq_rejects_misaligned_pointer_and_short_workspace(lib, ws):
    g = torch.zeros(64, device="cuda")
    acc = torch.zeros((), dtype=torch.float64, device="cuda")
    s = _lib.stream_ptr()
    assert lib.vdk_grad_sumsq(g.data_ptr() + 4, 60, acc.data_ptr(), 0, ws.data_ptr(), ws.numel(), s) != _lib.VDK_OK
    assert "aligned" in _lib.last_error()
    assert lib.vdk_grad_sumsq(g.data_ptr(), 64, acc.data_ptr(), 0, ws.data_ptr(), ws.numel() - 8, s) != _lib.VDK_OK
    assert "workspace" in _lib.last_error()


# ---- vdk_sgd_clip_ema_step ----------------------------------------------------------------------------------------------
def _run_step(lib, p, g, mom, ema, sumsq, max_norm=10.0, lr=0.1, momentum=0.9, wd=5e-4, first_step=0, updates=5,
              zero_grad=1):
    """One kernel call on NaN-guarded copies of (p, g, mom, ema); checks the result bit for bit against kernel_step and every
    guard element, returns (p, g, mom, ema) from the device."""
    d, omd = ema_decay(updates)
    bufs = [GuardedVec(torch.from_numpy(np.ascontiguousarray(x))) if x is not None else None for x in (p, g, mom, ema)]
    S = torch.tensor(sumsq, dtype=torch.float64, device="cuda")
    _lib.check(lib.vdk_sgd_clip_ema_step(bufs[0].ptr(), bufs[1].ptr(), bufs[2].ptr(), bufs[3].ptr() if ema is not None else 0,
                                         p.size, S.data_ptr(), max_norm, lr, momentum, wd, first_step, d, omd, zero_grad,
                                         _lib.stream_ptr()), "vdk_sgd_clip_ema_step")
    torch.cuda.synchronize()
    out = [b.host() if b is not None else None for b in bufs]
    for name, b in zip(("p", "g", "mom", "ema"), bufs):
        assert b is None or not b.guard_errors(), f"{name}: {b.guard_errors()}"
    want = kernel_step(p, g, mom, ema, sumsq, max_norm, lr, momentum, wd, first_step, d, omd, zero_grad)
    for name, got, w in zip(("p", "g", "mom", "ema"), out, want):
        if w is not None:
            _assert_bits(got, w, name)
    return out


def _state(n, seed, gscale=1.0):
    rng = np.random.default_rng(seed)
    p = rng.standard_normal(n).astype(F32)
    g = (rng.standard_normal(n) * gscale).astype(F32)
    mom = (rng.standard_normal(n) * 0.1).astype(F32)
    ema = (p + rng.standard_normal(n).astype(F32) * F32(0.01)).astype(F32)
    return p, g, mom, ema


def _check_bound(p, g, mom, ema, out, S, max_norm=10.0, lr=0.1, momentum=0.9, wd=5e-4, has_buf=True, updates=5):
    d, omd = ema_decay(updates)
    hp = (float(F32(max_norm)), float(F32(lr)), float(F32(momentum)), float(F32(wd)), has_buf, float(F32(d)), float(F32(omd)))
    rp, rm, re, _, _ = reference_step(p, g, mom, ema, S, *hp)
    e_p, e_m, e_e = step_bounds(p, g, mom, ema, S, *hp, sumsq_depth(g.size))
    _within(out[0], rp, e_p, "p")
    if momentum != 0:
        _within(out[2], rm, e_m, "momentum")
    if ema is not None:
        _within(out[3], re, e_e, "ema")


def _threshold_norms(max_norm=10.0):
    """The largest fp32 norm whose coef is exactly 1, and the next one up (clipping just active)."""
    t = F32(max_norm)
    while kernel_coef(float(t) ** 2, max_norm) < 1:
        t = np.nextafter(t, F32(0))
    return t, np.nextafter(t, F32(np.inf))


@pytest.mark.parametrize("clip", ["inactive", "active", "at_threshold", "just_above_threshold"])
@pytest.mark.parametrize("n", [1, 255, 256, 257, STEP_EDGE - 1, STEP_EDGE, STEP_EDGE + 1])
def test_step_clip_bitwise_and_within_bound(lib, clip, n):
    p, g, mom, ema = _state(n, n)
    S = float(exact_sumsq(g))
    if clip == "inactive":
        max_norm = 2 * math.sqrt(S) + 1
    elif clip == "active":
        max_norm = 0.25 * math.sqrt(S) + 1e-3
    else:
        max_norm = 10.0
        at, above = _threshold_norms(max_norm)
        t = at if clip == "at_threshold" else above
        S = float(t) ** 2                    # exact: t has 24 significant bits
        assert (kernel_coef(S, max_norm) == 1) == (clip == "at_threshold")
    out = _run_step(lib, p, g, mom, ema, S, max_norm=max_norm)
    assert (out[1] == 0).all()
    _check_bound(p, g, mom, ema, out, S, max_norm=max_norm)


def test_step_momentum_zero_never_reads_or_writes_the_buffer(lib):
    p, g, _, ema = _state(4099, 21)
    mom = np.full(p.size, np.nan, F32)
    S = float(exact_sumsq(g))
    out = _run_step(lib, p, g, mom, ema, S, momentum=0.0)
    assert np.isfinite(out[0]).all()
    _assert_bits(out[2], mom, "momentum buffer at momentum 0")
    _check_bound(p, g, mom, ema, out, S, momentum=0.0, has_buf=False)


def test_step_first_step_clones_the_update_into_a_poisoned_buffer(lib):
    p, g, _, ema = _state(4099, 22)
    mom = np.full(p.size, np.nan, F32)
    S = float(exact_sumsq(g))
    out = _run_step(lib, p, g, mom, ema, S, first_step=1, max_norm=1.0)
    assert np.isfinite(out[2]).all()
    _check_bound(p, g, np.zeros_like(mom), ema, out, S, max_norm=1.0, has_buf=False)


def test_step_zero_buffer_equals_first_step_up_to_the_sign_of_zero(lib):
    """What the optimizer relies on: from a zero buffer, momentum * 0 + d is d (first_step's clone) except that -0 becomes +0."""
    p, g, _, ema = _state(4099, 23)
    g[:8] = -0.0
    zero = np.zeros_like(p)
    S = float(exact_sumsq(g))
    a = _run_step(lib, p, g, zero, ema, S, first_step=0, wd=0.0)
    b = _run_step(lib, p, g, zero, ema, S, first_step=1, wd=0.0)
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[0], b[0])
    assert _bits(b[2][:8]).tolist() == [0x80000000] * 8 and _bits(a[2][:8]).tolist() == [0] * 8


def test_step_weight_decay_zero_and_lr_zero(lib):
    p, g, mom, ema = _state(2053, 24)
    S = float(exact_sumsq(g))
    out = _run_step(lib, p, g, mom, ema, S, wd=0.0)
    _check_bound(p, g, mom, ema, out, S, wd=0.0)
    out = _run_step(lib, p, g, mom, ema, S, lr=0.0)
    _assert_bits(out[0], p, "p at lr 0")


def test_step_without_ema_and_without_zero_grad(lib):
    p, g, mom, _ = _state(2053, 25)
    S = float(exact_sumsq(g))
    out = _run_step(lib, p, g, mom, None, S, zero_grad=0)
    _assert_bits(out[1], g, "g with zero_grad = 0")
    _check_bound(p, g, mom, None, out, S)


@pytest.mark.parametrize("updates", [1, 2000, 10 ** 6])
def test_step_ema_along_the_decay_ramp(lib, updates):
    p, g, mom, ema = _state(70_001, 26)
    S = float(exact_sumsq(g))
    out = _run_step(lib, p, g, mom, ema, S, updates=updates)
    _check_bound(p, g, mom, ema, out, S, updates=updates)


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_step_with_nonfinite_sumsq_keeps_p_and_momentum(lib, bad):
    p, g, mom, ema = _state(STEP_EDGE + 1, 27)
    g[5] = bad
    out = _run_step(lib, p, g, mom, ema, bad)
    _assert_bits(out[0], p, "p after a skipped step")
    _assert_bits(out[2], mom, "momentum after a skipped step")
    assert (out[1] == 0).all()
    d, omd = ema_decay(5)
    _within(out[3], np.asarray(ema, np.float64) * float(F32(d)) + float(F32(omd)) * np.asarray(p, np.float64),
            ema_bound(ema, p, float(F32(d)), float(F32(omd))), "ema after a skipped step")


# ---- vdk_ema_update -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("updates", [1, 10 ** 6])
@pytest.mark.parametrize("n", [1, 512, STEP_EDGE + 1])
def test_ema_update_bitwise_on_batchnorm_like_buffers(lib, updates, n):
    rng = np.random.default_rng(n + updates)
    ema = rng.gamma(2.0, 0.5, n).astype(F32)                       # running_var-like: positive, spread over decades
    src = (ema * rng.uniform(0.5, 2.0, n) + rng.uniform(0, 1e-5, n)).astype(F32)
    ema[: min(n, 3)] = [1e-5, 1.0, 3e4][: min(n, 3)]
    d, omd = ema_decay(updates)
    e, s = GuardedVec(torch.from_numpy(ema)), GuardedVec(torch.from_numpy(src))
    _lib.check(lib.vdk_ema_update(e.ptr(), s.ptr(), n, d, omd, _lib.stream_ptr()), "vdk_ema_update")
    torch.cuda.synchronize()
    assert not e.guard_errors() and not s.guard_errors()
    _assert_bits(e.host(), kernel_ema(ema, src, d, omd), "ema buffer")
    _within(e.host(), np.asarray(ema, np.float64) * float(F32(d)) + float(F32(omd)) * np.asarray(src, np.float64),
            ema_bound(ema, src, float(F32(d)), float(F32(omd))), "ema buffer")


# ---- FusedSGDClipEMA as the face trainer drives it ----------------------------------------------------------------------
class _Net(torch.nn.Module):
    """A small model with two parameter groups (backbone, head) and BatchNorm buffers."""

    def __init__(self):
        super().__init__()
        self.body = torch.nn.Sequential(torch.nn.Linear(37, 64), torch.nn.BatchNorm1d(64), torch.nn.Linear(64, 16))
        self.head = torch.nn.Linear(16, 11, bias=False)


def _small(seed=0, groups=2, momentum=0.9, max_norm=10.0, lr=0.05):
    torch.manual_seed(seed)
    model = _Net().cuda()
    with torch.no_grad():
        model.body[1].running_mean.uniform_(-1, 1)
        model.body[1].running_var.uniform_(0.5, 2)
    ema = copy.deepcopy(model).eval()
    for q in ema.parameters():
        q.requires_grad_(False)
    if groups == 2:
        pg = [{"params": list(model.body.parameters()), "lr": lr}, {"params": list(model.head.parameters()), "lr": lr * 10}]
    else:
        pg = [{"params": list(model.parameters()), "lr": lr}]
    opt = FusedSGDClipEMA(pg, lr=lr, momentum=momentum, weight_decay=5e-4, max_norm=max_norm, model=model, ema_model=ema)
    return model, ema, opt


def _grads(opt, seed, scale=1.0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for g in opt.groups:
        g.g.copy_(torch.randn(g.n, device="cuda", generator=gen) * scale)


def _snapshot(opt):
    return {"p": [g.p.clone() for g in opt.groups], "mom": [g.mom.clone() for g in opt.groups],
            "ema": [g.ema.clone() for g in opt.groups], "bufs": [e.clone() for e, _ in opt._buffers]}


def _equal_bits(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def _convnext_b_face_model():
    from visiondk_b200.train import FaceTrainingModel, layer_wise_groups
    cfg = {"backbone": {"timm-convnext_base": {"pretrained": False, "image_size": 224, "feat_dim": 512}},
           "head": {"arcface": {"feat_dim": 512, "num_class": 1000, "margin_arc": 0.35, "margin_am": 0.0, "scale": 32}}}
    torch.manual_seed(0)
    model = FaceTrainingModel(cfg).cuda()
    return model, layer_wise_groups(model, True, 0.01)


@pytest.mark.slow
def test_full_size_groups_step_within_bound_and_follow_torch(lib):
    """The bench's ConvNeXt-B parameter set (backbone at lr, the 512 x 1000 ArcFace head at 10 lr), twenty steps of synthetic
    gradients under cosine_with_warm_lr with the momentum switch at the end of warm-up, some steps clipped.  Every step is
    checked from the device's own state before it against the fp64 reference (one-step bound), and the whole trajectory
    against torch.optim.SGD + clip_grad_norm_ + ModelEMA in fp32."""
    model, groups = _convnext_b_face_model()
    ema = copy.deepcopy(model).eval()
    for q in ema.parameters():
        q.requires_grad_(False)
    twin = copy.deepcopy(model)
    lr0, warm, total, steps = 0.01, 4, 20, 20
    base = [g["lr"] for g in groups]
    opt = FusedSGDClipEMA(groups, lr=lr0, momentum=0.8, weight_decay=5e-4, max_norm=10.0, model=model, ema_model=ema)
    assert opt._buffers and sum(g.n for g in opt.groups) > 80_000_000 and opt.groups[1].n == 512 * 1000
    tparams = [list(twin.trainingwrapper["backbone"].parameters()), list(twin.trainingwrapper["head"].parameters())]
    tgroups = [{"params": ps, "lr": b} for ps, b in zip(tparams, base)]
    topt = torch.optim.SGD(tgroups, lr=lr0, momentum=0.8, weight_decay=5e-4)
    t_all = tparams[0] + tparams[1]
    t_ema = [q.detach().clone() for q in t_all]
    t_bufs = [b.detach().clone() for b in twin.buffers() if b.dtype.is_floating_point]
    clipped = []
    for t in range(steps):
        mom = 0.8 if t < warm else 0.937
        for pg, tpg, b in zip(opt.param_groups, topt.param_groups, base):
            pg["lr"] = tpg["lr"] = cosine_with_warm_lr(t, b, lr0, warm, total, None)
            pg["momentum"] = tpg["momentum"] = mom
        scale = 3e-4 if t % 3 else 3e-3                         # every third step's norm is far above max_norm
        _grads(opt, 100 + t, scale)
        for tq, g in zip(t_all, [q.grad for q in list(model.trainingwrapper["backbone"].parameters()) +
                                  list(model.trainingwrapper["head"].parameters())]):
            tq.grad = g.clone()
        before = _snapshot(opt)
        gs = [g.g.clone() for g in opt.groups]
        opt.step()
        S = sum(float((x.double() ** 2).sum()) for x in gs)
        clipped.append(10.0 / (math.sqrt(S) + 1e-6) < 1)
        d, omd = ema_decay(opt.updates)
        d32, omd32 = float(F32(d)), float(F32(omd))
        depth = sumsq_depth(max(g.n for g in opt.groups)) + len(opt.groups)
        for i, g in enumerate(opt.groups):
            hp = (10.0, float(F32(opt.param_groups[i]["lr"])), float(F32(mom)), float(F32(5e-4)), t > 0, d32, omd32)
            rp, rm, re, _, _ = reference_step(before["p"][i], gs[i], before["mom"][i], before["ema"][i], S, *hp)
            e_p, e_m, e_e = step_bounds(before["p"][i], gs[i], before["mom"][i], before["ema"][i], S, *hp, depth)
            for name, got, ref, bnd in (("p", g.p, rp, e_p), ("mom", g.mom, rm, e_m), ("ema", g.ema, re, e_e)):
                bad = ~((got.double() - ref).abs() <= bnd)
                assert not bool(bad.any()), f"step {t} group {i} {name}: {int(bad.sum())} elements outside the bound"
        for (e, src), e0 in zip(opt._buffers, before["bufs"]):
            ref = e0.double() * d32 + omd32 * src.double()
            assert bool(((e.double() - ref).abs() <= ema_bound(e0, src, d32, omd32)).all()), f"step {t} buffer EMA"
        # the same step in torch, fp32
        torch.nn.utils.clip_grad_norm_(t_all, 10.0)
        topt.step()
        with torch.no_grad():
            for v, q in zip(t_ema, t_all):
                v.mul_(d).add_(omd * q)
            for v, b in zip(t_bufs, [b for b in twin.buffers() if b.dtype.is_floating_point]):
                v.mul_(d).add_(omd * b)
        for g in opt.groups:
            assert not bool(g.g.any())
    assert any(clipped) and not all(clipped)
    ours_p = [q.detach() for q in list(model.trainingwrapper["backbone"].parameters()) +
              list(model.trainingwrapper["head"].parameters())]
    ours_e = [q.detach() for q in list(ema.trainingwrapper["backbone"].parameters()) +
              list(ema.trainingwrapper["head"].parameters())]
    torch.testing.assert_close(torch.cat([q.reshape(-1) for q in ours_p]), torch.cat([q.reshape(-1) for q in t_all]).detach(),
                               rtol=3e-5, atol=3e-6)
    torch.testing.assert_close(torch.cat([q.reshape(-1) for q in ours_e]), torch.cat([q.reshape(-1) for q in t_ema]),
                               rtol=3e-5, atol=3e-6)
    ema_bufs = [b for b in ema.buffers() if b.dtype.is_floating_point]
    for a, b in zip(ema_bufs, t_bufs):
        torch.testing.assert_close(a, b, rtol=3e-5, atol=3e-6)


def test_resume_from_state_dict_is_bitwise_an_uninterrupted_run(lib):
    _, _, ref = _small()
    for t in range(6):
        _grads(ref, 200 + t)
        ref.step()
    _, _, a = _small()
    for t in range(3):
        _grads(a, 200 + t)
        a.step()
    state = a.state_dict()
    model_b, ema_b, b = _small(seed=1)                          # different initial values: everything must come from `a`
    for gb, ga in zip(b.groups, a.groups):
        gb.p.copy_(ga.p)
        gb.ema.copy_(ga.ema)
    for (eb, sb), (ea, sa) in zip(b._buffers, a._buffers):
        eb.copy_(ea)
        sb.copy_(sa)
    b.load_state_dict(state)
    for t in range(3, 6):
        _grads(b, 200 + t)
        b.step()
    sr, sb_ = _snapshot(ref), _snapshot(b)
    for k in ("p", "mom", "ema", "bufs"):
        assert _equal_bits(sr[k], sb_[k]), k
    assert b.updates == ref.updates == 6


def test_one_group_or_two_groups_give_the_same_bits(lib):
    _, _, one = _small(groups=1, max_norm=1e6)
    _, _, two = _small(groups=2, max_norm=1e6, lr=0.05)
    for pg in two.param_groups:
        pg["lr"] = 0.05
    for t in range(4):
        _grads(two, 300 + t)
        one.groups[0].g.copy_(torch.cat([g.g for g in two.groups]))
        one.step()
        two.step()
        for k in ("p", "mom", "ema"):
            assert torch.equal(one.groups[0].__dict__[k].view(torch.int32),
                               torch.cat([g.__dict__[k] for g in two.groups]).view(torch.int32)), (t, k)


def test_step_does_not_synchronise(lib):
    _, _, opt = _small()
    _grads(opt, 400)
    opt.step()                                                  # first call loads the library
    _grads(opt, 401)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_ema_model_embed_sees_the_stepped_weights(lib):
    from visiondk_b200.train import FaceTrainingModel, layer_wise_groups
    cfg = {"backbone": {"timm-toy": {"pretrained": False, "image_size": 64, "feat_dim": 64, "depths": (1, 1, 2, 1),
                                     "dims": (64, 128, 128, 256)}},
           "head": {"arcface": {"feat_dim": 64, "num_class": 51, "margin_arc": 0.35, "margin_am": 0.0, "scale": 32}}}
    torch.manual_seed(31)
    model = FaceTrainingModel(cfg).cuda()
    ema = copy.deepcopy(model).eval()
    for q in ema.parameters():
        q.requires_grad_(False)
    opt = FusedSGDClipEMA(layer_wise_groups(model, True, 0.05), lr=0.05, momentum=0.9, weight_decay=5e-4, model=model,
                          ema_model=ema)
    x = torch.randn(2, 3, 64, 64, device="cuda")
    eb = ema.trainingwrapper["backbone"]
    before = eb.embed(x)
    _grads(opt, 500, 0.1)
    opt.step()
    after = eb.embed(x)
    eb.invalidate_pack()                                        # a pack built now holds the current EMA weights
    assert torch.equal(after, eb.embed(x))
    assert not torch.equal(after, before)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("group", [0, 1])
@pytest.mark.parametrize("when", ["first", "later"])
def test_nonfinite_gradient_skips_the_step(lib, bad, group, when):
    """GradScaler.step's rule: parameters and momentum unchanged bit for bit in every group, gradients zeroed, the EMA moved
    towards the unchanged parameters with `updates` counted, grad_norm() not finite.  The next finite step then starts the
    momentum buffer (a skipped first step) or continues exactly as a run that never saw the bad step."""
    _, _, opt = _small()
    _, _, clean = _small()
    bad_at = 0 if when == "first" else 2
    for t in range(bad_at):
        for o in (opt, clean):
            _grads(o, 600 + t)
            o.step()
    _grads(opt, 999)
    opt.groups[group].g[opt.groups[group].n // 3] = bad
    before = _snapshot(opt)
    opt.step()
    after = _snapshot(opt)
    assert _equal_bits(after["p"], before["p"]), "parameters moved on a skipped step"
    assert _equal_bits(after["mom"], before["mom"]), "momentum moved on a skipped step"
    assert all(not bool(g.g.any()) for g in opt.groups)
    assert not math.isfinite(opt.grad_norm())
    assert opt.updates == bad_at + 1
    d, omd = ema_decay(opt.updates)
    for e0, e1, p in zip(before["ema"], after["ema"], before["p"]):
        _assert_bits(e1.cpu().numpy(), kernel_ema(e0.cpu().numpy(), p.cpu().numpy(), d, omd), "EMA on a skipped step")
    for (e, src), e0 in zip(opt._buffers, before["bufs"]):
        _assert_bits(e.cpu().numpy(), kernel_ema(e0.cpu().numpy(), src.cpu().numpy(), d, omd), "buffer EMA on a skipped step")
    # the next, finite step
    _grads(opt, 600 + bad_at)
    _grads(clean, 600 + bad_at)
    gs = [g.g.cpu().numpy() for g in opt.groups]
    S = float(sum(exact_sumsq(x) for x in gs))
    opt.step()
    clean.step()
    if when == "first":
        for g, pg, gh, p0 in zip(opt.groups, opt.param_groups, gs, before["p"]):
            want = kernel_step(p0.cpu().numpy(), gh, np.full(g.n, np.nan, F32), None, float(opt._sumsq.item()), 10.0,
                               pg["lr"], 0.9, 5e-4, 1, 0, 0, 1)
            _assert_bits(g.mom.cpu().numpy(), want[2], "momentum after a skipped first step (torch's clone)")
            _assert_bits(g.p.cpu().numpy(), want[0], "parameters after a skipped first step")
        assert abs(opt.grad_norm() ** 2 - S) <= 1e-12 * S
    assert _equal_bits(_snapshot(opt)["p"], _snapshot(clean)["p"])
    assert _equal_bits(_snapshot(opt)["mom"], _snapshot(clean)["mom"])
