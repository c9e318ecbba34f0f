"""fp64 references and rounding bounds of the margin-softmax heads fused with cross-entropy (csrc/heads.cu).

Three layers, each checked elementwise (|got - ref| <= bound) and, for the contractions, by an RMS accuracy criterion:

  cos_reference      cos = normalize(f) . normalize(W, dim 0) in fp64 from the fp32 inputs, the magnitude
                     mag = sum_k |f~_k| |w~_k| and the bound of the kernel's 3-way-split contraction.
  stage2_reference   logits, row log-sum-exp, row loss, dz/dcos and dcos evaluated at the KERNEL's own cosines (cast to fp64),
                     so that every branch (ArcFace fallback, clamp, CircleLoss hinges, MV-Softmax hard negatives) is decided
                     on the values the kernel saw; thresholds use the kernel's fp32 constants.
  grad_reference     dfeats and dweight from the fp64 dcos through the two contractions and the normalisation backward.

Units: A = 2^-24 (fp32 unit roundoff).  The wgmma GEMM model is (ceil(K/16) + 17) 2^-23 relative to sum |a| |b| over the K
products (tests/test_gemm_gpu.py::acc_reference).  The split x = p0 + p1 + p2 (three bf16 parts) leaves |x - sum p| <= 2^-27 |x|,
and the three products it drops (p1 q2, p2 q1, p2 q2) are <= 2^-26 |x| |y|: 2^-25 |x| |y| per product in all.

RMS criterion: rms((got - ref) / (A * mag)) over all elements, with mag the sum of |terms| of the contraction (propagated through
the normalisation backward for the gradients).  It is what separates the six-product layout from a 2-part split or a layout
missing one product, which the elementwise (worst-case) GEMM model cannot; see kappa_cos for its measured values.
"""
import math

import torch

A = 2.0 ** -24
U32 = 2.0 ** -23
EX2 = 2.0 ** -22          # relative error of ex2.approx.ftz.f32 (__expf)
SPLIT = 2.0 ** -25        # split residual and dropped products, relative to |x| |y| per product
KIND = {"arcface": 0, "circleloss": 1, "mv_softmax": 2}

TINY = 2.0 ** -126        # fp32's smallest normal: __expf and the products below it may flush to zero
RMS_MIN_ELEMENTS = 4096   # the RMS criterion is applied where it is a statistic, not a handful of crafted rows


# RMS factor of dfeats (units of A * mag_df) in the un-fused backward with random dlogits, i.e. of the dF~ = dcos' . W^T
# contraction over K = 6 Cp and the normalisation backward (test_heads_fp64_gpu.py::test_long_k_contraction).  Measured on an
# H100 SXM (700 W) at C = 58 671: 31 with dF~ as one wgmma chain, 0.09 with heads.cu's fixed-order split-K slabs.
KAPPA_DFEATS = 1.0


def kappa_cos(D):
    """RMS factor (units of A * mag) the cos contraction must stay under at feat_dim D.

    Measured on an H100 SXM (700 W): 0.83-1.0 at D = 8 and 16, 2.1 at 64, 3.0 at 128, 6.2 at 512.  It grows like sqrt(D): the
    wgmma fp32 accumulator does not round to nearest (an exactly-rounded accumulator, emulated on the CPU, gives 0.43 at D = 128),
    so every k16 step after the p0 q0 block adds a biased error relative to the running sum.  kappa = 0.45 sqrt(Dp) sits 1.5x
    above the measurements; at D = 16 it sits 4x below the RMS of every defective product layout (test_heads_bounds_cpu.py)."""
    return 0.45 * math.sqrt(pad8(D))


def f32(x):
    return float(torch.tensor(float(x), dtype=torch.float32))


def eps32():
    return f32(1e-12)


def head_consts(kind, margin_arc=0.0, margin_am=0.0, scale=1.0, margin=0.0, gamma=1.0, mv_weight=1.0, is_am=False,
                label_smooth=0.0, fp32=True):
    """The fp32 constants make_cfg derives from the descriptor (cosf / sinf of an fp32 margin, fp32(pi) - m in fp32), or with
    fp32=False the oracle's fp64 ones."""
    f32 = globals()["f32"] if fp32 else float
    h = dict(kind=kind, scale=f32(scale), margin=f32(margin), gamma=f32(gamma), mv_weight=f32(mv_weight), is_am=bool(is_am),
             margin_am=f32(margin_am), margin_arc=f32(margin_arc), label_smooth=f32(label_smooth))
    m = h["margin"] if kind == "mv_softmax" else h["margin_arc"]
    h["cos_m"], h["sin_m"] = f32(math.cos(m)), f32(math.sin(m))
    h["min_cos"] = f32(math.cos(f32(f32(math.pi) - h["margin_arc"])))
    return h


def oracle_kwargs(h):
    if h["kind"] == "arcface":
        return dict(margin_arc=h["margin_arc"], margin_am=h["margin_am"], scale=h["scale"])
    if h["kind"] == "circleloss":
        return dict(margin=h["margin"], gamma=h["gamma"])
    return dict(is_am=h["is_am"], margin=h["margin"], mv_weight=h["mv_weight"], scale=h["scale"])


def ulp32(x):
    ax = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(ax)) - 23)


def _rnd32(x):
    return x.float().double()


# ------------------------------------------------------------------------------------------------------------------------------
# contraction: cos = f~ . W~

def gemm_rel(K):
    return (-(-K // 16) + 17) * U32


def pad8(n):
    return (n + 7) // 8 * 8


def norm_errors(feats, weight):
    """Relative error bounds of the kernel's fp32 f~ = f * inv_f and W~ = W * inv_w elements.
    row_inv_norm_kernel: a lane chains ceil(D/32) FMAs of positive terms, 5 shuffle adds, sqrtf, 1/x;
    col_inv_norm_kernel: D chained FMAs, sqrtf, 1/x;  then one rounding of the product."""
    D = feats.shape[1]
    e_f = ((-(-D // 32) + 5) / 2 + 2) * A * 1.01
    e_w = (D / 2 + 2) * A * 1.01
    return e_f, e_w


def cos_reference(feats, weight):
    f, w = feats.double(), weight.double()
    nf = f.norm(dim=1).clamp_min(eps32())
    nw = w.norm(dim=0).clamp_min(eps32())
    fh, wh = f / nf[:, None], w / nw[None, :]
    cos = fh @ wh
    mag = fh.abs() @ wh.abs()
    B, D = f.shape
    e_f, e_w = norm_errors(feats, weight)
    bound = mag * (gemm_rel(6 * pad8(D)) * 1.01 + SPLIT + e_f + e_w + 2 * A) * 1.01
    return dict(f=f, w=w, nf=nf, nw=nw, fh=fh, wh=wh, cos=cos, mag=mag, bound=bound, e_f=e_f, e_w=e_w)


def rms_factor(got, ref, mag):
    """rms((got - ref) / (A mag)) over elements with mag > 0."""
    m = mag > 0
    e = (got.double() - ref)[m] / (A * mag[m])
    return float(e.pow(2).mean().sqrt()) if e.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------------------------
# stage 2: margins, softmax, loss and dcos at the kernel's cosines

def _sqrt_term(c):
    """s = sqrtf(1 - c c) of an fp32 c, with |s~ - s|.  u = 1 - c^2 is rounded once (fused) or twice (c c, then 1 - that);
    both roundings are evaluated exactly and the larger taken.  |sqrt(u~) - sqrt(u)| <= |u~ - u| / sqrt(u), then sqrtf's own
    half ulp.  Returns (s, e_s); e_s = inf where u = 0 and u~ may differ from it."""
    c2 = c * c
    u = 1.0 - c2
    c2r = _rnd32(c2)
    e_unfused = (c2r - c2).abs() + (_rnd32(1.0 - c2r) - (1.0 - c2r)).abs()
    e_fused = (_rnd32(u) - u).abs()
    eu = torch.maximum(e_unfused, e_fused)
    s = u.clamp_min(0).sqrt()
    es = torch.where(s > 0, eu / s.clamp_min(1e-300), torch.where(eu > 0, math.inf, 0.0)) + A * s
    return s, es


def _quot_term(c, s, es):
    """t = c / s~ and |t~ - c/s| (inf where s <= e_s)."""
    t = c / s
    den = s * (s - es)
    et = torch.where(den > 0, c.abs() * es / den.clamp_min(1e-300), math.inf) + A * t.abs()
    return t, et


def stage2_reference(cosk, labels, h, grad_out=1.0, dlogits=None, logits_hint=None):
    """fp64 logits z, dz/dcos, row lse and loss, batch loss and dcos at the kernel's fp32 cosines `cosk` [B, C], with bounds.

    Kernel order (heads.cu head_logit / margin_ce_fwd_kernel / margin_ce_bwd_kernel) and the bound of each step:
      ArcFace: c = clamp(cos); non-label z = c s (A|z|); label c > min_cos: z = (c cos_m - s sin_m) scale with s = sqrtf(1 - c^2)
        (sin_m scale e_s + 4A scale (|c cos_m| + s sin_m)), dz = (cos_m + (c/s) sin_m) scale (e_t = |c| e_s / (s (s - e_s)): the
        1/(2s) amplification near c = 1); label fallback z = (c - m_am) scale; dz = 0 outside [-1, 1] (torch.clamp's select)
      CircleLoss: ap = max(fp32(1+m) - c, 0), an = max(c + m, 0) (exact hinge decisions: rounding keeps the sign);
        z = (a (c - o)) gamma, dz = a gamma: one rounding per operation
      MV-Softmax: gt = cos[y] (not clamped); thr = gt - m or gt cos_m - s sin_m; hard negatives cos > thr are ambiguous within
        |e_thr| of the threshold: the branch of an ambiguous element follows the kernel's logit when `logits_hint` is given,
        and the element is left out of the logit check
      softmax: __expf(z - M) = ex2.approx((z - M) log2e): relative 3A|z - M| + 2^-22 per term; per-thread chains of
        ceil(C/256) adds, 5 shuffles, 8 block adds; every online rescale (records of the running max along a thread's classes,
        plus the warp and block combines) another A (max z - min z) + 2^-22 + A; logf 1 ulp; M + log S one rounding;
        and lse's sensitivity to the logits' own errors, exp(2 max e_z) sum p e_z
      loss = (1-e)(lse - z_y) + e (lse - sum z / C): sum z over ceil(C/256) + 13 roundings; mean over B rows:
        ceil(B/32) + 6 roundings
      dcos = g (p - t) dz with g = gout / B, p = __expf(z - lse), t = (1-e) [c = y] + e/C; un-fused: dcos = dlogits dz.

    Returns a dict of fp64 tensors; `bad_one` marks elements where the reference itself is not finite (cos exactly 1 with a
    live sqrt derivative, or s within its error of 0), `ambiguous` the MV-Softmax threshold elements."""
    cosk = cosk.double()
    B, Cn = cosk.shape
    dev = cosk.device
    rows = torch.arange(B, device=dev)
    onehot = torch.zeros(B, Cn, dtype=torch.bool, device=dev)
    onehot[rows, labels] = True
    kind = h["kind"]
    bad_one = torch.zeros(B, Cn, dtype=torch.bool, device=dev)
    ambiguous = torch.zeros_like(bad_one)
    nan_row = torch.zeros(B, dtype=torch.bool, device=dev)
    if kind in ("arcface", "circleloss"):
        c = cosk.clamp(-1.0, 1.0)
        live = (cosk >= -1.0) & (cosk <= 1.0)
        if kind == "arcface":
            sc, cm, sm = h["scale"], h["cos_m"], h["sin_m"]
            z = c * sc
            ez = A * z.abs()
            d = torch.full_like(c, sc)
            ed = torch.zeros_like(c)
            s, es = _sqrt_term(c)
            t, et = _quot_term(c, s, es)
            arc = c > h["min_cos"]
            z_arc = (c * cm - s * sm) * sc
            ez_arc = sc * (sm * es + 4 * A * ((c * cm).abs() + s * sm))
            d_arc = (cm + t * sm) * sc
            ed_arc = sc * (sm * et + 3 * A * (cm + t.abs() * sm))
            z_fb = (c - h["margin_am"]) * sc
            ez_fb = 2 * A * sc * (c.abs() + abs(h["margin_am"]))
            lab_arc, lab_fb = onehot & arc, onehot & ~arc
            z = torch.where(lab_arc, z_arc, torch.where(lab_fb, z_fb, z))
            ez = torch.where(lab_arc, ez_arc, torch.where(lab_fb, ez_fb, ez))
            d = torch.where(lab_arc, d_arc, d)
            ed = torch.where(lab_arc, ed_arc, ed)
            bad_one = lab_arc & live & ~torch.isfinite(ed)
        else:
            g, m = h["gamma"], h["margin"]
            op, om = f32(1.0 + m), f32(1.0 - m)
            a_lab = (op - c).clamp_min(0.0)
            a_non = (c + m).clamp_min(0.0)
            a = torch.where(onehot, a_lab, a_non)
            ea = A * a
            x = torch.where(onehot, c - om, c - m)
            ex = A * x.abs()
            z = a * x * g
            ez = (g * (ea * x.abs() + a * ex) + 2 * A * z.abs()) * 1.01
            d = a * g
            ed = g * ea + A * d.abs()
        d = torch.where(live, d, torch.zeros_like(d))
        ed = torch.where(live, ed, torch.zeros_like(ed))
    else:
        sc, cm, sm, m, w = h["scale"], h["cos_m"], h["sin_m"], h["margin"], h["mv_weight"]
        gt = cosk[rows, labels]
        if h["is_am"]:
            thr = gt - m
            e_thr = A * thr.abs()
            final = torch.where(gt > m, gt - m, gt)
            e_final = torch.where(gt > m, A * (gt - m).abs(), torch.zeros_like(gt))
            dfin, e_dfin = torch.ones_like(gt), torch.zeros_like(gt)
        else:
            nan_row = gt.abs() > 1.0
            gs = gt.clamp(-1.0, 1.0)
            s, es = _sqrt_term(gs)
            t, et = _quot_term(gs, s, es)
            thr = gs * cm - s * sm
            e_thr = sm * es + 3 * A * ((gs * cm).abs() + s * sm)
            pos = gs > 0
            final = torch.where(pos, thr, gs)
            e_final = torch.where(pos, e_thr, torch.zeros_like(gs))
            dfin = torch.where(pos, cm + t * sm, torch.ones_like(gs))
            e_dfin = torch.where(pos, sm * et + 3 * A * (cm + t.abs() * sm), torch.zeros_like(gs))
        hard = cosk > thr[:, None]
        ambiguous = ~onehot & ((cosk - thr[:, None]).abs() <= e_thr[:, None] * 1.01 + 1e-300)
        z_hard = (w * cosk + w - 1.0) * sc
        if logits_hint is not None:
            hint = logits_hint.double()
            hard = torch.where(ambiguous, (hint - z_hard).abs() < (hint - cosk * sc).abs(), hard)
        z = torch.where(hard, z_hard, cosk * sc)
        ez = torch.where(hard, 4 * A * sc * ((w * cosk).abs() + abs(w) + 1.0) + A * z_hard.abs(), A * (cosk * sc).abs())
        d = torch.where(hard, torch.full_like(cosk, w * sc), torch.full_like(cosk, sc))
        ed = torch.where(hard, A * d.abs(), torch.zeros_like(d))
        z = torch.where(onehot, (final * sc)[:, None].expand_as(z), z)
        ez = torch.where(onehot, (sc * e_final + A * (final * sc).abs())[:, None].expand_as(z), ez)
        d = torch.where(onehot, (dfin * sc)[:, None].expand_as(d), d)
        ed = torch.where(onehot, (sc * e_dfin + A * (dfin * sc).abs())[:, None].expand_as(d), ed)
        bad_one = onehot & (pos[:, None] if not h["is_am"] else torch.zeros_like(onehot)) & ~torch.isfinite(ed)
        if not h["is_am"]:
            bad_one = bad_one & ~nan_row[:, None]

    # ---- row softmax / loss ----
    ok_row = ~nan_row
    zf = torch.where(ok_row[:, None], z, torch.zeros_like(z))
    ezf = torch.where(torch.isfinite(ez) & ok_row[:, None], ez, torch.zeros_like(ez))
    lse = torch.logsumexp(zf, dim=1)
    p = torch.exp(zf - lse[:, None])
    M = zf.max(1).values
    rng = M - zf.min(1).values
    J = -(-Cn // 256)
    zp = torch.nn.functional.pad(zf, (0, J * 256 - Cn), value=-math.inf).view(B, J, 256)
    prev = torch.cat([torch.full_like(zp[:, :1], -math.inf), zp.cummax(1).values[:, :-1]], 1)
    records = (zp > prev).sum(1).max(1).values.double()
    n_resc = records + 4
    e_S = (p * (3 * A * (zf - M[:, None]).abs() + EX2)).sum(1) + (J + 13) * A + n_resc * (A * rng + EX2 + A)
    e_shift = torch.exp(2 * ezf.max(1).values) * (p * ezf).sum(1)
    logS = lse - M
    e_lse = (e_shift + e_S * 1.01 + 2 * A * logS.abs() + A * lse.abs() + A * M.abs()) * 1.01
    eps = h["label_smooth"]
    zy = zf[rows, labels]
    Z = zf.sum(1)
    e_Z = (J + 13) * A * zf.abs().sum(1) + ezf.sum(1)
    t1, t2 = lse - zy, lse - Z / Cn
    loss_row = (1 - eps) * t1 + eps * t2
    e_loss_row = ((1 - eps) * (e_lse + ezf[rows, labels] + A * t1.abs()) + eps * (e_lse + e_Z / Cn + 2 * A * (Z / Cn).abs()
                  + A * t2.abs()) + 3 * A * ((1 - eps) * t1.abs() + eps * t2.abs()) + A * (1 - eps) * t1.abs()) * 1.01
    nb = -(-B // 32) + 6
    loss = loss_row[ok_row].sum() / B if bool(ok_row.all()) else torch.tensor(math.nan, dtype=torch.float64, device=dev)
    e_loss = e_loss_row[ok_row].sum() / B + nb * A * loss_row[ok_row].abs().mean() if bool(ok_row.any()) else torch.tensor(0.0)

    # ---- dcos ----
    if dlogits is None:
        g = f32(grad_out) / B
        tgt = torch.where(onehot, 1.0 - eps, 0.0) + eps / Cn
        dpt = p - tgt
        delta = ezf + e_lse[:, None] + 3 * A * (zf - lse[:, None]).abs()
        e_p = p * (torch.expm1(delta) + EX2 * torch.exp(delta)) + torch.where(p < 2 * TINY, p, torch.zeros_like(p))
        e_t = 3 * A * tgt
        dcos = g * dpt * d
        e_dcos = (abs(g) * ((e_p + e_t) * d.abs() + dpt.abs() * ed + 3 * A * (dpt * d).abs()) + A * (dcos).abs()
                  + 2 * TINY * (1 + abs(g) * d.abs())) * 1.01
    else:
        dl = dlogits.double()
        dcos = dl * d
        e_dcos = dl.abs() * ed + A * dcos.abs() + 2 * TINY
    dcos = torch.where(bad_one, torch.zeros_like(dcos), dcos)
    # a NaN row (MV-Softmax arc, gt > 1) is NaN everywhere in the fused backward (through its lse); in the un-fused one only
    # its label column is
    unbounded = bad_one | (~torch.isfinite(dcos) if dlogits is not None else ~ok_row[:, None])
    dcos = torch.where(unbounded, torch.zeros_like(dcos), dcos)
    e_dcos = torch.where(unbounded, torch.full_like(e_dcos, math.inf), e_dcos)
    return dict(z=z, ez=ez, d=d, ed=ed, lse=lse, e_lse=e_lse, loss_row=loss_row, e_loss_row=e_loss_row, loss=loss,
                e_loss=e_loss, dcos=dcos, e_dcos=e_dcos, bad_one=bad_one, ambiguous=ambiguous, nan_row=nan_row, p=p)


# ------------------------------------------------------------------------------------------------------------------------------
# backward contractions and the normalisation backward

def grad_reference(cr, s2, labels):
    """dfeats, dweight in fp64 from s2['dcos'] with bounds and RMS magnitudes.

      dcos' = dcos inv_w (fp32: + e_w + A relative);  dF~ = dcos' . W^T on the split GEMM over K = 6 Cp:
        e_dF = sum_c e_dcos' |W| + (gemm(6 Cp) + 2^-25) sum_c |dcos'| |W|
      df = (dF~ - f~ (f~ . dF~)) inv_f: the dot chains ceil(D/32) FMAs + 5 shuffles; the subtraction cancels when dF~ is nearly
        parallel to f~, which the bound carries as |f~_k| e_dot + 2A |f~_k dot|
      dW~ = f~^T . dcos on the split GEMM over K = 6 Bp:  e_dWt = sum_b (|f~| e_dcos + |f~ dcos| (e_f + A)) + (gemm(6 Bp) + 2^-25)
        sum_b |f~| |dcos|
      dW = (dW~ - W~ (W~ . dW~)) inv_w: 8 warps chain ceil(D/8) FMAs, 8 shared adds.
    Rows / columns holding an element whose dcos is unbounded (cos exactly 1, MV gt > 1) get an infinite bound (left out)."""
    f, w, fh, wh, nf, nw = cr["f"], cr["w"], cr["fh"], cr["wh"], cr["nf"], cr["nw"]
    e_f, e_w = cr["e_f"], cr["e_w"]
    B, D = f.shape
    Cn = w.shape[1]
    Cp, Bp = pad8(Cn), pad8(B)
    dcos, e_dcos = s2["dcos"], s2["e_dcos"]
    inf_el = ~torch.isfinite(e_dcos)
    e_dcos = torch.where(inf_el, torch.zeros_like(e_dcos), e_dcos)
    iw = 1.0 / nw
    dcs = dcos * iw
    e_dcs = e_dcos * iw + dcs.abs() * (e_w + A)
    wabs = w.abs()
    dF = dcs @ w.t()
    magF = dcs.abs() @ wabs.t()
    e_dF = e_dcs @ wabs.t() + (gemm_rel(6 * Cp) * 1.01 + SPLIT) * magF
    fabs = fh.abs()
    dot = (fh * dF).sum(1, keepdim=True)
    e_dot = (fabs * e_dF).sum(1, keepdim=True) + (fabs * dF.abs()).sum(1, keepdim=True) * (e_f + A + (-(-D // 32) + 5) * A)
    inner = dF - fh * dot
    e_inner = e_dF + fabs * e_dot + (fh * dot).abs() * (e_f + A) + 2 * A * ((fh * dot).abs() + inner.abs())
    inv_f = 1.0 / nf[:, None]
    df = inner * inv_f
    e_df = (e_inner * inv_f + inner.abs() * inv_f * e_f + A * df.abs()) * 1.01
    mag_df = inv_f * (magF + fabs * (fabs * magF).sum(1, keepdim=True))
    bad_rows = inf_el.any(1)
    e_df[bad_rows] = math.inf

    dWt = fh.t() @ dcos
    magW = fabs.t() @ dcos.abs()
    e_dWt = fabs.t() @ e_dcos + (fabs.t() @ dcos.abs()) * (e_f + A) + (gemm_rel(6 * Bp) * 1.01 + SPLIT) * magW
    whabs = wh.abs()
    dotw = (wh * dWt).sum(0, keepdim=True)
    e_dotw = (whabs * e_dWt).sum(0, keepdim=True) + (whabs * dWt.abs()).sum(0, keepdim=True) * (e_w + 2 * A + (-(-D // 8) + 8) * A)
    innw = dWt - wh * dotw
    e_innw = e_dWt + whabs * e_dotw + (wh * dotw).abs() * (e_w + 2 * A) + 2 * A * ((wh * dotw).abs() + innw.abs())
    dW = innw * iw
    e_dW = (e_innw * iw + innw.abs() * iw * e_w + A * dW.abs()) * 1.01
    mag_dW = iw * (magW + whabs * (whabs * magW).sum(0, keepdim=True))
    bad_cols = inf_el.any(0)
    e_dW[:, bad_cols] = math.inf
    return dict(df=df, e_df=e_df, mag_df=mag_df, dW=dW, e_dW=e_dW, mag_dW=mag_dW, bad_rows=bad_rows, bad_cols=bad_cols)


# ------------------------------------------------------------------------------------------------------------------------------
# inputs

def make_case(B, D, Cn, seed, craft=True, same_label=False, spread=1.0, label_cos_max=None):
    """Seeded fp32 inputs (generated on the CPU so every device sees the same values).  Labels include 0 and C - 1, and
    classes with no sample when C > B.  `craft` adds rows that hit every branch:
      up to 16 rows parallel to their class column at scalings from 0.05 to 1e3 (the kernel's own label cos lands
        on both sides of 1), one anti-parallel row (ArcFace fallback), one row parallel and one anti-parallel to a non-label
        column (non-label clamp, CircleLoss alpha_n = 0), rows with the label column at cos +-0.2, +-0.5 and a non-label
        column near each side of the MV threshold, a zero feature row and a zero weight column.
    `label_cos_max` turns the parallel rows into rows at that cosine to their class column (for MV-Softmax arc, whose
    loss is NaN where the label cos exceeds 1, exactly as in the reference)."""
    g = torch.Generator().manual_seed(seed)
    feats = torch.randn(B, D, generator=g) * 2.0
    w = torch.empty(D, Cn).uniform_(-1, 1, generator=g)
    w = w.renorm(2, 1, 1e-5).mul(1e5) * spread
    if same_label:
        labels = torch.full((B,), Cn // 2, dtype=torch.long)
    else:
        labels = torch.randint(0, Cn, (B,), generator=g)
        labels[0], labels[-1] = 0, Cn - 1
    if not craft or B < 4:
        return feats, w, labels
    r = 0

    def put(vec):
        nonlocal r
        if r < B:
            feats[r] = vec
        r += 1

    for sc in (1.0, 0.125, 3.7, 1e3, 0.3, 7.0, 1.1, 0.9, 13.0, 0.05, 2.5, 50.0, 0.77, 1.3, 9.0, 0.6)[:max(4, B // 6)]:
        col = w[:, labels[min(r, B - 1)]]
        if label_cos_max is not None:
            n = torch.randn(D, generator=g)
            n = n - (n @ col) / (col @ col) * col
            col = label_cos_max * col + math.sqrt(1 - label_cos_max ** 2) * n / n.norm() * col.norm()
        put(col * sc)
    put(-w[:, labels[min(r, B - 1)]] * 2.0)                        # anti-parallel: ArcFace fallback
    if Cn > 2:
        other = lambda row: (int(labels[min(row, B - 1)]) + 1) % Cn
        put(w[:, other(r)] * 1.5)                                   # parallel to a non-label column
        put(-w[:, other(r)] * 0.7)                                  # anti-parallel to a non-label column
    for cy in (0.2, -0.2, 0.5, -0.5, 0.9):                          # MV gt on both sides of 0 and of m
        if r >= B:
            break
        y = int(labels[r])
        u = w[:, y] / w[:, y].norm()
        n = torch.randn(D, generator=g)
        n = n - (n @ u) * u
        n = n / n.norm().clamp_min(1e-30)
        put(cy * u + math.sqrt(1 - cy * cy) * n)
    if r < B:
        feats[r] = 0.0                                              # zero feature row
        r += 1
    if Cn > 3:
        w[:, Cn - 2] = 0.0                                          # zero weight column (a class with no sample unless labelled)
    return feats, w, labels


# ------------------------------------------------------------------------------------------------------------------------------
# one check of every output of a forward + backward

def check_head(out, feats, weight, labels, h, grad_out=1.0, dlogits=None, stats=None, tag="", rms=None, rms_dfeats=False):
    """Checks the kernel outputs `out` (dict of tensors: cos [B, C], logits [B, C] or None, row_lse [B] or None, loss (scalar
    or None), dfeats [B, D], dweight [D, C]) against the fp64 references with kernel_ref.check_within, and the cos RMS factor
    against kappa_cos.  With `rms_dfeats` (un-fused backward with random dlogits, where dcos = dlogits dz carries a couple of
    roundings and nothing cancels) the dfeats RMS factor is held to KAPPA_DFEATS: that is the dF~ contraction's own accuracy.
    In the fused backward the gradients' RMS factors are only reported: there p - t cancels where a row is confidently right,
    and the fp32 stage 2 (__expf's 2^-22) adds to them, which their elementwise bounds carry.  Returns the exclusion counts
    and RMS factors."""
    from kernel_ref import check_within
    dev = out["cos"].device
    f, w, y = feats.to(dev), weight.to(dev), labels.to(dev)
    dlogits = dlogits.to(dev) if dlogits is not None else None
    none = lambda bad: f"{int(bad.sum())} elements"
    cr = cos_reference(f, w)
    cosk = out["cos"].double()
    check_within(cosk, cr["cos"], cr["bound"], f"cos{tag}", none, stats)
    info = dict(rms_cos=rms_factor(cosk, cr["cos"], cr["mag"]))
    s2 = stage2_reference(cosk, y, h, grad_out, dlogits, out.get("logits"))
    ok_row = ~s2["nan_row"]
    info.update(ambiguous=int(s2["ambiguous"].sum()), at_one=int(s2["bad_one"].sum()), nan_rows=int(s2["nan_row"].sum()),
                cos_gt_1=int((cosk[torch.arange(len(y), device=dev), y] > 1).sum()))
    if out.get("logits") is not None:
        keep = ~s2["ambiguous"] & ok_row[:, None]
        zb = torch.where(keep, s2["ez"], torch.full_like(s2["ez"], math.inf))
        zr = torch.where(keep, s2["z"], torch.zeros_like(s2["z"]))
        got = torch.where(keep, out["logits"].double(), torch.zeros_like(zr))
        check_within(got, zr, torch.where(keep, zb, torch.zeros_like(zb)), f"logits{tag}", none, stats)
    if out.get("row_lse") is not None:
        lg = out["row_lse"].double()[ok_row]
        check_within(lg, s2["lse"][ok_row], s2["e_lse"][ok_row], f"row_lse{tag}", none, stats)
    if out.get("loss") is not None and bool(ok_row.all()):
        lv = torch.as_tensor(out["loss"], dtype=torch.float64, device=dev).reshape(1)
        check_within(lv, s2["loss"].reshape(1), s2["e_loss"].reshape(1).to(dev), f"loss{tag}", none, stats)
    if out.get("dfeats") is not None:
        gr = grad_reference(cr, s2, y)
        rows, cols = ~gr["bad_rows"], ~gr["bad_cols"]
        check_within(out["dfeats"][rows], gr["df"][rows], gr["e_df"][rows], f"dfeats{tag}", none, stats)
        check_within(out["dweight"][:, cols], gr["dW"][:, cols], gr["e_dW"][:, cols], f"dweight{tag}", none, stats)
        info.update(rms_dfeats=rms_factor(out["dfeats"][rows], gr["df"][rows], gr["mag_df"][rows]),
                    rms_dweight=rms_factor(out["dweight"][:, cols], gr["dW"][:, cols], gr["mag_dW"][:, cols]),
                    excluded_rows=int(gr["bad_rows"].sum()), excluded_cols=int(gr["bad_cols"].sum()))
    print(f"HEADS{tag}: {info}")
    if rms is not False and cosk.numel() >= RMS_MIN_ELEMENTS:
        kap = kappa_cos(f.shape[1])
        assert info["rms_cos"] <= kap, f"cos{tag}: RMS {info['rms_cos']:.3f} > {kap:.3f} (units of 2^-24 mag)"
    if rms_dfeats:
        assert info["rms_dfeats"] <= KAPPA_DFEATS, f"dfeats{tag}: RMS {info['rms_dfeats']:.3f} > {KAPPA_DFEATS} (units of 2^-24 mag)"
    return info
