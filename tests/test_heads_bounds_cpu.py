"""CPU self-tests of the margin-head references and bounds in heads_ref.py.

* The stage-2 restatement, run at fp64 cosines, reproduces oracle/heads.py run in fp64 (the oracle is pinned to the reference's
  own modules by tests/test_oracle_heads_cpu.py), for every head kind.
* An fp32 emulation of heads.cu (3-way bf16 split, exact bf16 x bf16 products accumulated in fp32 one k16 step at a time, the
  fused stage 2 and the normalisation backward in fp32) passes every check of heads_ref.check_head.
* Plausible defects fail them, on inputs the GPU test (test_heads_fp64_gpu.py) also runs: a 2-part split, bf16 only, each
  5-of-6 product layout, grad_out ignored, label smoothing dropped from the backward target, the label column off by one, a
  padded class leaking into the softmax, and the clamp derivative taken as a product (inf * 0 = NaN at cos > 1).
"""
import math

import pytest
import torch

import heads_ref as R
from oracle import heads as H

SIX = [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]
LOG2E = float(torch.tensor(1.4426950408889634, dtype=torch.float32))

# the self-test cases, also run on the GPU by test_heads_fp64_gpu.py::test_self_test_case_on_gpu: the face config's
# feat_dim for the stage-2 defects, and D = 16 for the product layouts, where the measured kernel RMS (kappa_cos) sits furthest
# below the defects' (a dropped product's error averages over D terms, the accumulator's grows with them)
CASE = dict(B=96, D=128, Cn=257, seed=11)
CASE_RMS = dict(B=96, D=16, Cn=257, seed=12)
HEAD = dict(kind="arcface", margin_arc=0.35, margin_am=0.0, scale=32.0, label_smooth=0.1)


def parts(x):
    p0 = x.to(torch.bfloat16).float()
    r1 = x - p0
    p1 = r1.to(torch.bfloat16).float()
    p2 = (r1 - p1).to(torch.bfloat16).float()
    return p0, p1, p2


def round_toward_zero(x):
    """fp64 -> fp32, truncated: a model of the wgmma fp32 accumulator, which does not round to nearest.  With it the emulated
    cos RMS is 1.2 / 2.7 / 3.9 / 7.9 at D = 16 / 64 / 128 / 512; an H100 measures 1.0 / 2.1 / 3.0 / 6.2 (heads_ref.kappa_cos)."""
    r = x.float()
    return torch.where(r.double().abs() > x.abs(), torch.nextafter(r, torch.zeros_like(r)), r)


def emu_gemm(a, b, layout=SIX, truncate=False, kblocks_per_slab=None):
    """split_gemm: D[M, N] = sum over the layout's products of a_i . b_j^T, K padded to a multiple of 8 per product, each k16 step
    summed exactly (bf16 x bf16 products are exact in fp64) and added to the fp32 accumulator with one rounding (to nearest,
    or toward zero with `truncate`).  `kblocks_per_slab`: split-K slabs of that many 64-wide K blocks, each accumulated on its
    own and the slabs added in order in fp32 (heads.cu dfn_splits + the fixed-order slab reduction)."""
    M, K = a.shape
    Kp = R.pad8(K)
    pa = [torch.nn.functional.pad(p, (0, Kp - K)).double() for p in parts(a)]
    pb = [torch.nn.functional.pad(p, (0, Kp - K)).double() for p in parts(b)]
    A6 = torch.cat([pa[i] for i, _ in layout], 1)
    B6 = torch.cat([pb[j] for _, j in layout], 1)
    rnd = round_toward_zero if truncate else (lambda x: x.float())
    slab = 64 * kblocks_per_slab if kblocks_per_slab else A6.shape[1]
    out = torch.zeros(M, b.shape[0], dtype=torch.float32)
    for k0 in range(0, A6.shape[1], slab):
        acc = torch.zeros(M, b.shape[0], dtype=torch.float32)
        for k in range(k0, min(k0 + slab, A6.shape[1]), 16):
            acc = rnd(acc.double() + A6[:, k:k + 16] @ B6[:, k:k + 16].t())
        out = out + acc
    return out


def dfn_kblocks_per_slab(Cp):
    """heads.cu dfn_splits: min(256, ceil(kbt / 16)) slabs over kbt = ceil(6 Cp / 64) K blocks, evened out."""
    kbt = -(-6 * Cp // 64)
    want = min(256, -(-kbt // 16))
    return -(-kbt // want)


def fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def emu_row_inv(x):
    R_, K = x.shape
    J = -(-K // 32)
    xp = torch.nn.functional.pad(x, (0, J * 32 - K)).view(R_, J, 32)
    s = torch.zeros(R_, 32)
    for j in range(J):
        s = fma32(xp[:, j], xp[:, j], s)
    lane = torch.arange(32)
    for off in (16, 8, 4, 2, 1):
        s = s + s[:, lane ^ off]
    return 1.0 / torch.clamp_min(torch.sqrt(s[:, 0]), R.eps32())


def emu_col_inv(w):
    s = torch.zeros(w.shape[1])
    for d in range(w.shape[0]):
        s = fma32(w[d], w[d], s)
    return 1.0 / torch.clamp_min(torch.sqrt(s), R.eps32())


def expf(x):
    return torch.exp2((x * LOG2E).float())


def emu_logit(h, cosv, is_label, gt, defect):
    """head_logit for one column of every row (fp32)."""
    c = cosv.clamp(-1.0, 1.0)
    live = (cosv >= -1) & (cosv <= 1)
    sc, cm, sm = (torch.tensor(h[k], dtype=torch.float32) for k in ("scale", "cos_m", "sin_m"))
    if h["kind"] == "arcface":
        s = torch.sqrt(1.0 - c * c)
        arc = c > h["min_cos"]
        z_l = torch.where(arc, (c * cm - s * sm) * sc, (c - h["margin_am"]) * sc)
        d_l = torch.where(arc, (cm + (c / s) * sm) * sc, sc.expand_as(c))
        z = torch.where(is_label, z_l, c * sc)
        d = torch.where(is_label, d_l, sc.expand_as(c))
        dz = d * live.float() if defect == "clamp_product" else torch.where(live, d, torch.zeros_like(d))
        return z, dz
    raise NotImplementedError(h["kind"])


def emulate(feats, w, labels, h, grad_out, layout=SIX, defect=None, dlogits=None, truncate=False, dfn_slabs=True):
    """fp32 emulation of vdk_head_forward (with logits) + vdk_head_backward (fused, or un-fused with `dlogits`).
    `truncate` models the H100's accumulator; `dfn_slabs=False` runs dF~ as one chain over K = 6 Cp."""
    B, D = feats.shape
    Cn = w.shape[1]
    Cp = R.pad8(Cn)
    y = labels.clone()
    if defect == "label_off_by_one":
        y = (y + 1) % Cn
    inv_f, inv_w = emu_row_inv(feats), emu_col_inv(w)
    fn = feats * inv_f[:, None]
    wn = (w * inv_w[None, :]).t()
    wn = torch.nn.functional.pad(wn, (0, 0, 0, Cp - Cn))
    cos = emu_gemm(fn, wn, layout, truncate)                         # [B, Cp]
    ncls = Cp if defect == "padded_leak" else Cn
    cols = torch.arange(ncls)
    is_label = cols[None, :] == y[:, None]
    z, dz = emu_logit(h, cos[:, :ncls], is_label, None, defect)
    # online softmax: thread t takes classes t, t + 256, ...
    J = -(-ncls // 256)
    zp = torch.nn.functional.pad(z, (0, J * 256 - ncls), value=-math.inf).view(B, J, 256)
    mx = torch.full((B, 256), -3.4028234663852886e38)
    se = torch.zeros(B, 256)
    for j in range(J):
        zj = zp[:, j]
        valid = torch.isfinite(zj)
        up = valid & (zj > mx)
        se_up = se * expf(mx - zj) + 1.0
        se_keep = se + torch.where(valid, expf(zj - mx), torch.zeros_like(se))
        se = torch.where(up, se_up, se_keep)
        mx = torch.where(up, zj, mx)
    wm = mx.view(B, 8, 32).max(-1).values
    sew = (se.view(B, 8, 32) * expf(mx.view(B, 8, 32) - wm[..., None])).sum(-1)
    M = wm.max(-1).values
    S = torch.zeros(B)
    for k in range(8):
        S = S + sew[:, k] * expf(wm[:, k] - M)
    lse = M + torch.log(S)
    eps = h["label_smooth"]
    Z = z.sum(1)
    zy = z[torch.arange(B), y]
    row = (1 - eps) * (lse - zy) + eps * (lse - Z / Cn)
    loss = row.mean()
    # backward
    g = (1.0 if defect == "grad_out_ignored" else grad_out) / B
    p = expf(z - lse[:, None])
    t_off = 0.0 if defect == "smoothing_dropped" else eps / Cn
    tgt = torch.where(is_label, torch.tensor(1.0 - (0.0 if defect == "smoothing_dropped" else eps)), torch.tensor(0.0)) + t_off
    v = g * (p - tgt) * dz if dlogits is None else dlogits * dz
    v = torch.nn.functional.pad(v, (0, Cp - ncls))
    iw = torch.nn.functional.pad(inv_w, (0, Cp - Cn))
    vs = v * iw
    wT = torch.nn.functional.pad(w, (0, Cp - Cn))                   # [D, Cp]
    dfn = emu_gemm(vs, wT, layout, truncate, dfn_kblocks_per_slab(Cp) if dfn_slabs else None)  # [B, D]
    dot = (fn * dfn).sum(1, keepdim=True)
    df = (dfn - fn * dot) * inv_f[:, None]
    dwn = emu_gemm(fn.t().contiguous(), v.t().contiguous(), layout, truncate)  # [D, Cp]
    wt = w * inv_w[None, :]
    dotw = (wt * dwn[:, :Cn]).sum(0, keepdim=True)
    dW = (dwn[:, :Cn] - wt * dotw) * inv_w[None, :]
    return dict(cos=cos[:, :Cn], logits=z[:, :Cn], row_lse=lse, loss=loss, dfeats=df, dweight=dW)


@pytest.fixture(scope="module")
def case():
    feats, w, labels = R.make_case(**CASE)
    h = R.head_consts(**HEAD)
    return feats, w, labels, h


GRAD_OUT = R.f32(0.37)  # the fp32 value the kernel reads


def run_checks(case, layout=SIX, defect=None, rms=True):
    feats, w, labels, h = case
    out = emulate(feats, w, labels, h, GRAD_OUT, layout, defect)
    return R.check_head(out, feats, w, labels, h, grad_out=GRAD_OUT, rms=rms)


@pytest.fixture(scope="module")
def case_rms():
    feats, w, labels = R.make_case(**CASE_RMS)
    return feats, w, labels, R.head_consts(**HEAD)


@pytest.mark.parametrize("which", ["case", "case_rms"])
def test_emulated_kernel_is_inside_every_bound(which, request):
    c = request.getfixturevalue(which)
    info = run_checks(c)
    assert info["cos_gt_1"] > 0, "the crafted parallel rows should push some label cosines past 1"
    assert info["rms_cos"] < R.kappa_cos(c[0].shape[1]) / 2


LAYOUTS = {"2-part": SIX[:4], "bf16": SIX[:1], **{f"drop{SIX[i]}": SIX[:i] + SIX[i + 1:] for i in range(6)}}


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_defective_split_layout_is_rejected(case_rms, name):
    feats, w, labels, h = case_rms
    out = emulate(feats, w, labels, h, GRAD_OUT, LAYOUTS[name])
    cr = R.cos_reference(feats, w)
    rms = R.rms_factor(out["cos"], cr["cos"], cr["mag"])
    print(f"{name}: cos RMS {rms:.3f}")
    assert rms > 2 * R.kappa_cos(feats.shape[1])
    with pytest.raises(AssertionError):
        run_checks(case_rms, LAYOUTS[name])


@pytest.mark.parametrize("defect", ["grad_out_ignored", "smoothing_dropped", "label_off_by_one", "padded_leak", "clamp_product"])
def test_defective_stage2_is_rejected(case, defect):
    with pytest.raises(AssertionError):
        run_checks(case, defect=defect, rms=False)


def test_long_k_contraction_needs_the_slabs():
    """With a truncating accumulator (the H100 model), dF~ as one wgmma chain over K = 6 Cp drifts: the un-fused dfeats RMS
    (random dlogits, so nothing in stage 2 cancels) leaves KAPPA_DFEATS far behind, growing with C (17 at C = 5000, 59 at the
    face config's 58 671).  The fixed-order split-K slabs of heads.cu bring it back under a round-to-nearest single chain."""
    B, D, Cn = 160, 128, 5000
    feats, w, labels = R.make_case(B, D, Cn, seed=5)
    h = R.head_consts(**HEAD)
    dl = torch.randn(B, Cn, generator=torch.Generator().manual_seed(1))
    rms = {}
    for name, slabs in (("one chain", False), ("slabs", True)):
        out = emulate(feats, w, labels, h, 1.0, dlogits=dl, truncate=True, dfn_slabs=slabs)
        rms[name] = R.check_head(out, feats, w, labels, h, dlogits=dl, rms=False)["rms_dfeats"]
    print(rms)
    assert rms["one chain"] > 2 * R.KAPPA_DFEATS
    assert rms["slabs"] < R.KAPPA_DFEATS / 2


KINDS = [dict(kind="arcface", margin_arc=0.35, margin_am=0.0, scale=32.0),
         dict(kind="arcface", margin_arc=0.5, margin_am=0.2, scale=64.0),
         dict(kind="circleloss", margin=0.25, gamma=256.0),
         dict(kind="circleloss", margin=0.25, gamma=64.0),
         dict(kind="mv_softmax", is_am=False, margin=0.35, mv_weight=1.12, scale=32.0),
         dict(kind="mv_softmax", is_am=True, margin=0.35, mv_weight=1.12, scale=32.0)]


@pytest.mark.parametrize("smooth", [0.0, 0.1])
@pytest.mark.parametrize("k", range(len(KINDS)))
def test_restatement_matches_the_oracle_in_fp64(k, smooth):
    """stage2_reference + grad_reference at fp64 cosines give oracle/heads.py's logits, loss and autograd gradients, both run
    in fp64 on the same inputs (random rows: no cosine near a threshold or near +-1 at D = 16)."""
    B, D, Cn = 24, 16, 37
    feats, w, labels = R.make_case(B, D, Cn, seed=100 + k, craft=False)
    h = R.head_consts(**KINDS[k], label_smooth=R.f32(smooth), fp32=False)  # an fp32 value either way
    f64, w64 = feats.double().requires_grad_(True), w.double().requires_grad_(True)
    kind = h["kind"]
    loss, logits = H.head_loss(kind, f64, w64, labels, label_smooth=h["label_smooth"], **R.oracle_kwargs(h))
    (loss * GRAD_OUT).backward()
    cr = R.cos_reference(feats.double(), w.double())
    s2 = R.stage2_reference(cr["cos"], labels, h, grad_out=GRAD_OUT)
    assert int(s2["ambiguous"].sum()) == 0 and int(s2["bad_one"].sum()) == 0
    gr = R.grad_reference(cr, s2, labels)
    assert torch.allclose(s2["z"], logits.detach(), rtol=1e-12, atol=1e-11)
    assert abs(float(s2["loss"]) - float(loss)) <= 1e-12 * abs(float(loss))
    # torch's fp64 cross-entropy backward with label smoothing is itself off by ~3e-9 relative (it carries the smoothing
    # factor in fp32); without smoothing the two agree to fp64 rounding
    tol = 1e-7 if smooth else 1e-12
    assert torch.allclose(gr["df"], f64.grad, rtol=0, atol=tol * float(f64.grad.abs().max()))
    assert torch.allclose(gr["dW"], w64.grad, rtol=0, atol=tol * float(w64.grad.abs().max()))
