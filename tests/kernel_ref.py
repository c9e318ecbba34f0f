"""Shared pieces of the kernel parity tests: fp64 references, rounding bounds, NaN-guarded outputs and failure reports.

Every comparison here is elementwise, |got - ref| <= bound, with the bound derived from the kernel's roundings (the derivation
sits in each test's docstring).  Outputs live inside buffers filled with a NaN bit pattern, so a store past the last row,
past N into the padding of a pitched row, or past the end of the output shows up as a changed guard element.
"""
import math

import torch

U32 = 2.0 ** -23   # one fp32 ulp at 1 (twice fp32's unit roundoff)
LOG2E = 1.4426950408889634

# precision p (bits, implicit one included) and the smallest normal exponent of each output type
_FORMAT = {torch.bfloat16: (8, -126), torch.float16: (11, -14), torch.float32: (24, -126)}
_BITS = {2: torch.int16, 4: torch.int32}
# quiet NaNs with a payload no arithmetic produces: a guard element that still holds it was never written
_GUARD = {torch.bfloat16: 0x7FA5, torch.float16: 0x7E5A, torch.float32: 0x7FA5A5A5}


def ulp(x, dtype):
    """One unit in the last place of `dtype` at |x| (fp64 tensor in, fp64 out; subnormal spacing below the normal range)."""
    p, emin = _FORMAT[dtype]
    ax = x.abs().clamp_min(2.0 ** emin)
    return torch.exp2(torch.floor(torch.log2(ax)) - (p - 1))


def unit_roundoff(dtype):
    """Largest relative error of one round-to-nearest into `dtype` (normal range)."""
    return 2.0 ** -_FORMAT[dtype][0]


class Guarded:
    """A [rows, cols] view with row pitch `ld` inside a buffer of `rows + extra_rows` pitched rows and a `tail` of elements
    after them, every element outside the view holding a NaN guard pattern."""

    def __init__(self, rows, cols, ld, dtype, extra_rows=3, tail=64, device="cuda"):
        assert ld >= cols
        self.dtype = dtype
        self.buf = torch.empty((rows + extra_rows) * ld + tail, dtype=dtype, device=device)
        self.bits = self.buf.view(_BITS[self.buf.element_size()])
        self.bits.fill_(_GUARD[dtype])
        self.view = self.buf[:rows * ld].view(rows, ld)[:, :cols]
        self.inside = torch.zeros(self.buf.numel(), dtype=torch.bool, device=device)
        self.inside[:rows * ld].view(rows, ld)[:, :cols] = True

    def fill_(self, values):
        self.view.copy_(values)
        return self

    def ptr(self):
        return self.view.data_ptr()

    def guard_errors(self):
        """Message naming the guard elements that were written, or '' when every one still holds the pattern."""
        changed = (~self.inside) & (self.bits != _GUARD[self.dtype])
        if not bool(changed.any()):
            return ""
        idx = changed.nonzero().flatten()
        return f"{idx.numel()} guard elements written, first flat offsets {idx[:8].tolist()}"


def check_within(got, ref, bound, name, describe, stats=None):
    """Asserts |got - ref| <= bound elementwise (a NaN anywhere fails).  `describe(bad_mask)` names the work items holding
    the failures.  Records max |got - ref| / bound under `name` in `stats` and returns it."""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    used = float((err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max()) if err.numel() else 0.0
    if stats is not None:
        stats[name] = max(stats.get(name, 0.0), used)
    print(f"BOUND {name}: worst error {used:.4f} of the bound")
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} outside the bound (worst {used:.3g}x); first at {i}: got "
                             f"{float(got[tuple(i)])} ref {float(ref[tuple(i)])} bound {float(bound[tuple(i)])}\n{describe(bad)}")
    return used


# ------------------------------------------------------------------------------------------------------------------------------
# attention: softmax(q k^T / 8) v per (image, head) on qkv [B, N, 3, H, 64]

ATT_QTILE, ATT_KVTILE = 128, 64


def attention_items(B, N, H, sm_count):
    n_pairs = (-(-N // ATT_QTILE) + 1) // 2
    items = n_pairs * H * B
    return items, min(items, sm_count)


def describe_attention(bad_tokens, N, H, sm_count):
    """bad_tokens: bool [B, H, N] -> the (b, h, tile pair) items and CTA rounds holding failures."""
    B = bad_tokens.shape[0]
    n_pairs = (-(-N // ATT_QTILE) + 1) // 2
    items_total, grid = attention_items(B, N, H, sm_count)
    padded = torch.nn.functional.pad(bad_tokens, (0, n_pairs * 2 * ATT_QTILE - N))
    bad_bhp = padded.view(B, H, n_pairs, 2 * ATT_QTILE).any(-1)
    idx = bad_bhp.nonzero()
    item = (idx[:, 0] * H + idx[:, 1]) * n_pairs + idx[:, 2]
    rounds = torch.bincount(item // grid).tolist()
    return (f"{idx.shape[0]}/{items_total} items wrong (grid {grid}); wrong items per CTA round {rounds}; first (b, h, pair) "
            f"{idx[:6].tolist()} on CTAs {(item[:6] % grid).tolist()}")


def attention_reference(qkv):
    """fp64 softmax(q k^T / 8) v of the bf16 inputs, with elementwise error bounds of the kernel's output and log2-domain
    log-sum-exp.  Returns (out [B, N, H*64], out_bound, lse2 [B, H, N], lse2_bound), all fp64.

    Kernel arithmetic (attention_tc.cu) and the bound of each step, for row i, key j, feature d:
      S_ij = q_i . k_j in fp32 on wgmma (64 = 4 k16 steps): |dS_ij| <= (4 + 17) 2^-23 (|q_i| . |k_j|)  (DESIGN.md §3 model)
      x_ij = fma(S_ij, c, -m_ref), c = fp32(log2 e) / 8: one rounding, 2^-24 |x| <= 2^-24 c (|S_ij| + max_j |S_ij|), and
             c's own 2^-24 relative on c |S_ij|, so |dx_ij| <= c 21 2^-23 (|q||k|)_ij + 2^-23 c (|S_ij| + max_j |S_ij|)
      P~_ij = ex2.approx(x_ij): relative 2^-22 on top, so P~_ij = P_ij (1 + a_ij), a_ij = ln 2 |dx_ij| + 2^-22
      (m_ref is common to every key of a tile, and a rescale multiplies O and l by the same alpha: both cancel in O / l)
      O = sum_j bf16(P~_ij) v_j on wgmma: bf16 rounding of P (2^-8 relative) and the fp32 chain over ceil(N/16) k16 steps
             plus one alpha multiply per key tile: e_acc = (ceil(64 J / 16) + 17 + J) 2^-23 relative to (P |V|)
      l = sum_j P~_ij in fp32 on each thread (16 J adds) + 2 shuffles: e_l = (16 J + 2) 2^-24 relative
      out = bf16(O / l): 2^-22 for 1/l and the product, 2^-8 for the rounding
    => |out - R| <= (P (2^-8 + a)) |V| + e_acc (P |V|) + |R| (sum_j P_ij a_ij + e_l + 2^-8 + 2^-22)
      lse2 = m_ref + log2(l): log2 of l's relative error (sum_j P a + e_l + (J - 1) 2^-22 for the rescales' alphas) and the
             fp32 roundings of m_ref, log2f and the add: |d lse2| <= log2(e) (sum_j P a + e_l + (J - 1) 2^-22)
             + 2^-22 (|lse2| + log2(l_max) + 1)
    """
    B, N, _, H, D = qkv.shape
    J = -(-N // ATT_KVTILE)
    c = float(torch.tensor(LOG2E, dtype=torch.float32)) / 8.0
    e_acc = (4 * J + 17 + J) * U32
    e_l = (16 * J + 2) * 2.0 ** -24
    q, k, v = qkv.double().permute(2, 0, 3, 1, 4).unbind(0)  # [B, H, N, 64]
    out = torch.empty(B, H, N, D, dtype=torch.float64, device=qkv.device)
    out_b = torch.empty_like(out)
    lse = torch.empty(B, H, N, dtype=torch.float64, device=qkv.device)
    lse_b = torch.empty_like(lse)
    qf, kf, vf = q.reshape(B * H, N, D), k.reshape(B * H, N, D), v.reshape(B * H, N, D)
    of, obf, lf, lbf = out.view(B * H, N, D), out_b.view(B * H, N, D), lse.view(B * H, N), lse_b.view(B * H, N)
    step = max(1, (1 << 24) // (N * N))
    for s0 in range(0, B * H, step):
        sl = slice(s0, min(B * H, s0 + step))
        S = qf[sl] @ kf[sl].transpose(-1, -2)
        absqk = qf[sl].abs() @ kf[sl].abs().transpose(-1, -2)
        a = math.log(2.0) * (c * 21 * U32 * absqk + U32 * c * (S.abs() + S.abs().amax(-1, keepdim=True))) + 2.0 ** -22
        del absqk
        lse_nat = torch.logsumexp(S * 0.125, dim=-1)
        P = torch.exp(S * 0.125 - lse_nat[..., None])
        del S
        absv = vf[sl].abs()
        R = P @ vf[sl]
        pa = (P * a).sum(-1, keepdim=True)
        of[sl] = R
        obf[sl] = (P * (2.0 ** -8 + a)) @ absv + e_acc * (P @ absv) + R.abs() * (pa + e_l + 2.0 ** -8 + 2.0 ** -22)
        lf[sl] = lse_nat * LOG2E
        l_max = 256.0 * N
        lbf[sl] = LOG2E * (pa[..., 0] + e_l + (J - 1) * 2.0 ** -22) + 2.0 ** -22 * (lf[sl].abs() + math.log2(l_max) + 1)
        del P, a
    out = out.transpose(1, 2).reshape(B, N, H * D)
    out_b = out_b.transpose(1, 2).reshape(B, N, H * D)
    return out, out_b, lse, lse_b


def run_attention(lib, qkv, with_lse=True):
    """Runs vdk_attention_fwd(_lse) into NaN-guarded outputs: returns (out [B, N, H*64] Guarded, lse2 [B, H, N] Guarded)."""
    from visiondk_b200 import _lib
    B, N, _, H, D = qkv.shape
    out = Guarded(B * N, H * D, H * D, torch.bfloat16, extra_rows=0, tail=4096)
    lse = Guarded(B * H, N, N, torch.float32, extra_rows=0, tail=1024) if with_lse else None
    if with_lse:
        rc = lib.vdk_attention_fwd_lse(qkv.data_ptr(), B, N, H, D, out.ptr(), lse.ptr(), _lib.stream_ptr())
    else:
        rc = lib.vdk_attention_fwd(qkv.data_ptr(), B, N, H, D, out.ptr(), _lib.stream_ptr())
    _lib.check(rc, "attention forward")
    torch.cuda.synchronize()
    return out, lse


def check_attention(lib, qkv, stats=None, with_lse=True):
    """Runs the forward on qkv and checks out and lse2 against attention_reference elementwise, and every guard element."""
    B, N, _, H, D = qkv.shape
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    out, lse = run_attention(lib, qkv, with_lse)
    ref, ref_b, lse_ref, lse_b = attention_reference(qkv)
    got = out.view.view(B, N, H * D)

    def describe_out(bad):
        return describe_attention(bad.view(B, N, H, D).any(-1).permute(0, 2, 1), N, H, sm)

    check_within(got, ref, ref_b, "attention out", describe_out, stats)
    assert not out.guard_errors(), "out: " + out.guard_errors()
    if with_lse:
        check_within(lse.view.view(B, H, N), lse_ref, lse_b, "attention lse2", lambda bad: describe_attention(bad, N, H, sm), stats)
        assert not lse.guard_errors(), "lse2: " + lse.guard_errors()
    return got


def crafted_qkv(B, N, H, alphas, beta, seed, dense=False, device="cuda"):
    """q_i = alphas[i % len] e_0, k_j = beta[j] e_0, so every raw score q_i . k_j = alpha * beta is an exact product of two bf16
    values: the test chooses each row's score sequence.  Neighbouring rows take different alphas, so the rows of one 16-row
    warp slice mix rows that rescale with rows that do not.  dense=True adds random q components in dimensions 1-31 and random k
    components in dimensions 32-63: the scores stay exact (the two sets of dimensions are disjoint), and the backward's dQ = dS K
    and dK = dS^T Q are dense rows instead of multiples of e_0."""
    torch.manual_seed(seed)
    qkv = torch.zeros(B, N, 3, H, 64, device=device)
    a = torch.tensor(alphas, device=device)[torch.arange(N, device=device) % len(alphas)]
    qkv[:, :, 0, :, 0] = a[None, :, None]
    qkv[:, :, 1, :, 0] = beta[None, :, None]
    qkv[:, :, 2] = torch.randn(B, N, H, 64, device=device).to(torch.bfloat16).float()
    if dense:
        qkv[:, :, 0, :, 1:32] = torch.randn(B, N, H, 31, device=device).to(torch.bfloat16).float()
        qkv[:, :, 1, :, 32:] = torch.randn(B, N, H, 32, device=device).to(torch.bfloat16).float()
    out = qkv.to(torch.bfloat16)
    assert torch.equal(out.float(), qkv)  # alphas and betas are bf16 values
    return out


def _store(ref, e32):
    """Bound after the bf16 store of an fp32 value within e32 of ref; 0 where both are 0 (an exact fp32 zero stores exactly)."""
    return torch.where(ref.abs() + e32 > 0, bf16_store_bound(ref, e32), torch.zeros_like(e32))


def attention_bwd_reference(qkv, out, dout, lse2, out_bound=None, lse2_bound=None):
    """fp64 dq, dk, dv of softmax(q k^T / 8) v per (image, head), with an elementwise bound of attention_bwd_kernel's result.
    Returns (dqkv [B, N, 3, H, 64], bound of the same shape), both fp64.

    The reference differentiates with P_ij = 2^(S_ij log2(e) / 8 - lse2_i) and D_i = sum_d dO_id out_id, taking `out`
    [B, N, H*64] and `lse2` [B, H, N] as given:
      isolated: out and lse2 are the kernel's own operands (bf16 and fp32 of the fp64 forward), out_bound = lse2_bound = None.
                This is exactly the kernel's contract, and P is whatever that lse2 makes of the scores.
      chained:  out and lse2 are the exact fp64 forward (attention_reference), so P is the exact softmax and the result is the
                exact gradient; out_bound and lse2_bound bound how far the forward kernel's out and lse2, which the backward
                kernel is then given, lie from them, and enter D's and x's errors below.

    Kernel arithmetic (vit.cu attention_bwd_kernel) and the bound of each step, for query row i, key j, feature d, with
    u = 2^-24 (fp32 unit roundoff), U = 2^-23 and n = ceil(N / 16) k16 steps over the (zero-padded) token dimension.
    An fp32 chain of k16 mma.sync steps is within (steps + 17) U of the product of magnitudes (DESIGN.md §3 model).
      S_ij = q_i . k_j, 4 k16 steps: |dS_ij| <= 21 U A_ij, A_ij = |q_i| . |k_j|
      x_ij = S_ij c - lse2_i, c = 0.125 fp32(log2 e): c's own rounding u c |S|, the fp32 multiply and subtract (or one fma)
             u c |S| + u |x|, and the input's error lse2_bound_i (chained):
             |dx_ij| <= c 21 U A_ij + U c |S_ij| + U |x_ij| + lse2_bound_i   (U, not u, on |x| covers |x~| > |x|)
      P~_ij = ex2.approx.ftz(x~_ij): 2 ulp (2^-22) relative on top of 2^dx, and an absolute 2^-126 where ftz flushes to 0:
             |P~ - P| <= P a + 2^-126,  a_ij = (2^|dx_ij| - 1)(1 + 2^-22) + 2^-22
      P^ = bf16(P~) (0 for padded rows and columns): |P^ - P| <= eP = P (a + 2^-8 (1 + a)) + 2^-126
      D~_i: two lanes each run a 32-term fp32 fma chain of exact bf16 products, then one add, over the bf16 out (chained: out
             lies within out_bound of the exact O): |dD_i| <= 33 u sum_d |dO_id| (|out_id| + ob_id) + sum_d |dO_id| ob_id
      dP~_ij = dO_i . v_j, 4 k16 steps: |ddP_ij| <= 21 U B_ij, B_ij = |dO_i| . |v_j|;  E_ij = 21 U B_ij + |dD_i|
      dS~_ij = bf16(fp32(0.125 P^_ij) fp32(dP~_ij - D~_i)): 0.125 P^ is exact; with G_ij = |dP_ij - D_i|, |dP~ - D~| <= G + E,
             so before the store |dS~ - dS| <= 0.125 (eP (G + E) + P E + (P + eP)(G + E)(2u + u^2)) + 2^-149 (an fp32
             subnormal product), then half a bf16 ulp.  The bound scales with |dP| + |D|, not with |dP - D|: where a peaked
             row makes dP_ij - D_i cancel, the error of each term does not.
      dV_j = sum_i P^_ij dO_i (A = P^T), n steps: (n + 17) U sum_i (P + eP)_ij |dO_i| + sum_i eP_ij |dO_i|, then the bf16 store
      dQ_i = sum_j dS^_ij k_j, n steps: (n + 17) U sum_j (|dS| + eS)_ij |k_j| + sum_j eS_ij |k_j|, then the bf16 store
      dK_j = sum_i dS^_ij q_i (A = dS^T), n steps: likewise with |q_i|
    A row of dO that is exactly 0 has D = 0 and dP = 0 exactly, so its dS and dQ rows are exact zeros; their bound is 0 too.
    The work is chunked over (image, head) slices so that no [slices, N, N] fp64 temporary exceeds 2^24 elements.
    """
    B, N, _, H, D = qkv.shape
    assert D == 64
    dev = qkv.device
    n = -(-N // 16)
    u, c = 2.0 ** -24, float(torch.tensor(LOG2E, dtype=torch.float32)) / 8.0
    e_chain = (n + 17) * U32

    def heads(t):  # [B, N, H*64] -> [B*H, N, 64]
        return t.double().reshape(B, N, H, D).transpose(1, 2).reshape(B * H, N, D)

    q, k, v = (t.reshape(B * H, N, D) for t in qkv.double().permute(2, 0, 3, 1, 4).unbind(0))
    o, do = heads(out), heads(dout)
    ob = heads(out_bound) if out_bound is not None else torch.zeros_like(o)
    l = lse2.double().reshape(B * H, N)
    lb = lse2_bound.double().reshape(B * H, N) if lse2_bound is not None else torch.zeros_like(l)
    grads = torch.empty(3, B * H, N, D, dtype=torch.float64, device=dev)
    bounds = torch.empty_like(grads)
    step = max(1, (1 << 24) // (N * N))
    for s0 in range(0, B * H, step):
        sl = slice(s0, min(B * H, s0 + step))
        qs, ks, vs, os_, dos = q[sl], k[sl], v[sl], o[sl], do[sl]
        aq, ak, av, ado = qs.abs(), ks.abs(), vs.abs(), dos.abs()
        S = qs @ ks.transpose(-1, -2)
        x = S * (LOG2E / 8.0) - l[sl, :, None]
        P = torch.exp2(x)
        dx = c * 21 * U32 * (aq @ ak.transpose(-1, -2)) + U32 * c * S.abs() + U32 * x.abs() + lb[sl, :, None]
        del S, x
        a = torch.expm1(math.log(2.0) * dx) * (1 + 2.0 ** -22) + 2.0 ** -22
        del dx
        eP = P * (a + 2.0 ** -8 * (1 + a)) + 2.0 ** -126
        del a
        Dv = (dos * os_).sum(-1)
        eD = 33 * u * (ado * (os_.abs() + ob[sl])).sum(-1) + (ado * ob[sl]).sum(-1)
        dP = dos @ vs.transpose(-1, -2)
        E = 21 * U32 * (ado @ av.transpose(-1, -2)) + eD[..., None]
        Gm = dP - Dv[..., None]
        dS = 0.125 * P * Gm
        G = Gm.abs()
        del dP, Gm
        eS32 = 0.125 * (eP * (G + E) + P * E + (P + eP) * (G + E) * (2 * u + u * u))
        eS = _store(dS, eS32 + (G + E > 0).double() * 2.0 ** -149)
        del G, E, eS32
        grads[2, sl] = P.transpose(-1, -2) @ dos
        bounds[2, sl] = _store(grads[2, sl], (e_chain * (P + eP) + eP).transpose(-1, -2) @ ado)
        del P, eP
        W = e_chain * (dS.abs() + eS) + eS
        grads[0, sl] = dS @ ks
        bounds[0, sl] = _store(grads[0, sl], W @ ak)
        grads[1, sl] = dS.transpose(-1, -2) @ qs
        bounds[1, sl] = _store(grads[1, sl], W.transpose(-1, -2) @ aq)
        del dS, eS, W
    # [3, B*H, N, 64] -> [B, N, 3, H, 64]
    grads = grads.view(3, B, H, N, D).permute(1, 3, 0, 2, 4).contiguous()
    bounds = bounds.view(3, B, H, N, D).permute(1, 3, 0, 2, 4).contiguous()
    return grads, bounds


# ------------------------------------------------------------------------------------------------------------------------------
# ConvNeXt HBM-bound kernels (csrc/convnext.cu, csrc/train_ops.cu): launch arithmetic, fp64 references and bounds.
# Every reference takes the kernel's own bf16 / fp32 inputs and is computed in fp64 on the device.

A32 = 2.0 ** -24   # fp32 unit roundoff
WG_T, WG_C = 14, 64


def wgrad_launch(B, H, W, C, sm_count):
    """launch_dwconv7_wgrad: tile edge T, strips per tile row nh, images per CTA ipc, image groups, tiles per image, chunks."""
    T = min(WG_T, max(H, W))
    tiles = -(-H // T) * -(-W // T)
    chunks = -(-C // WG_C)
    ipc = max(1, min(16, tiles * chunks * B // (sm_count * 4)))
    return dict(T=T, nh=-(-T // 7), ipc=ipc, groups=-(-B // ipc), tiles=tiles, chunks=chunks)


def ln_bwd_launch(npix, C, sm_count):
    """launch_ln_bwd: (LPP, IT, U), blocks, pixels per warp trip, and the fewest trips any warp makes."""
    vecs = C // 8
    lpp, it, u = next(cfg for lim, cfg in ((8, (8, 1, 4)), (16, (16, 1, 4)), (32, (32, 1, 4)), (64, (32, 2, 2)),
                                          (96, (32, 3, 1)), (128, (32, 4, 1)), (192, (32, 6, 1))) if vecs <= lim)
    ppt = (32 // lpp) * u
    blocks = max(1, min(-(-npix // (8 * ppt)), sm_count * (1 if it >= 4 else 2)))
    nwarps = 8 * blocks
    last = npix - (nwarps - 1) * ppt  # pixels left to the last warp after its first base
    return dict(lpp=lpp, it=it, u=u, blocks=blocks, ppt=ppt, nwarps=nwarps,
                min_trips=max(0, -(-last // (nwarps * ppt))) if last > 0 else 0,
                max_trips=-(-npix // (nwarps * ppt)))


def dwconv7_reference(x, w49):
    """fp64 correlation out[b, y, x, c] = sum_{dy, dx} w49[7 dy + dx, c] x[b, y + dy - 3, x + dx - 3, c] (zero padding)
    of NHWC x with [49, C] taps, and sum |w x| over the same 49 products."""
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 3, 3, 3, 3))
    w = w49.double()
    out = torch.zeros(B, H, W, C, dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(out)
    for t in range(49):
        dy, dx = divmod(t, 7)
        p = xp[:, dy:dy + H, dx:dx + W, :] * w[t]
        out += p
        mag += p.abs()
    return out, mag


def dwconv7_bwd_data_bound(ref, mag, addend):
    """Bound of mode 1 (vdk_dwconv7(1, ...): out = bf16(sum_49 w x + addend)), whatever the order of its fp32 operations:
      49 FMAs and one add of the addend, each one rounding of a partial sum bounded by sum |w x| + |addend|:
        |fp32 result - exact| <= 50 * 2^-24 * (mag + |addend|)
      bf16 store: half an ulp of the fp32 result, <= ulp_bf16(|ref| + e32) / 2."""
    a = addend.double().abs() if addend is not None else 0.0
    e32 = 50 * A32 * (mag + a) * 1.001
    return e32 + 0.5 * ulp(ref.abs() + e32, torch.bfloat16)


def wgrad_reference(x, g):
    """fp64 dw49 [49, C] = sum_{b,y,x} g[b,y,x,c] x[b,y+dy-3,x+dx-3,c], dbias [C] = sum g, and their sums of |terms|."""
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 3, 3, 3, 3))
    gd = g.double()
    dw = torch.empty(49, C, dtype=torch.float64, device=x.device)
    dw_mag = torch.empty_like(dw)
    for t in range(49):
        dy, dx = divmod(t, 7)
        p = gd * xp[:, dy:dy + H, dx:dx + W, :]
        dw[t] = p.sum((0, 1, 2))
        dw_mag[t] = p.abs().sum((0, 1, 2))
    return dw, dw_mag, gd.sum((0, 1, 2)), gd.abs().sum((0, 1, 2))


def wgrad_bound(mag, init, launch):
    """Bound of vdk_dwconv7_wgrad (dw49 += ..., dbias += ...) for one output element.
    Kernel order (train_ops.cu): bf16 x bf16 products are exact in fp32.  A thread chains ipc x T x 7 FMAs (its images,
    tile rows, strip pixels); nh strip partials are added in shared memory; every CTA (image group x tile) adds its
    partial to the output with one fp32 atomic, starting from the output's initial value.  Each rounding is at most
    2^-24 of a partial sum bounded by sum |terms| + |init|, and no term passes more than
        n = ipc * T * 7 + nh + groups * tiles
    roundings:  |got - (init + exact)| <= n 2^-24 (sum |terms| + |init|)."""
    n = launch["ipc"] * launch["T"] * 7 + launch["nh"] + launch["groups"] * launch["tiles"]
    return n * A32 * (mag + init.double().abs()) * 1.001


def layernorm_bwd_reference(xhat, rstd64, gamma, dy, addend, patch):
    """fp64 LayerNorm backward from the exact normalised input xhat [P, C] (pixel rows of NHWC order) and exact rstd64 [P]:
    dx = rstd (g - mean_c g - xhat mean_c(g xhat)) + addend with g = dy gamma; dgamma = sum_p dy xhat; dbeta = sum_p dy.
    dy [P, C] is given in pixel order (the caller undoes the patch layout)."""
    g = dy.double() * gamma.double()
    m1 = g.mean(-1, keepdim=True)
    m2 = (g * xhat).mean(-1, keepdim=True)
    dx = rstd64[:, None] * (g - m1 - xhat * m2)
    if addend is not None:
        dx = dx + addend.double()
    return dx, (dy.double() * xhat).sum(0), dy.double().sum(0), m1, m2


def layernorm_bwd_bound(xhat, rstd64, gamma, beta, y, dy, addend, m1, m2, launch, dg_init, db_init):
    """Elementwise bounds of vdk_layernorm_bwd (dx, dgamma, dbeta), all fp64; a = 2^-24, n1 = 8 IT + log2(LPP).

    Kernel order (train_ops.cu) per pixel, channel:
      h = (y - beta) * fl(1/gamma): y is the SAVED bf16 output, e_y = |y - (gamma xhat + beta)| <= ulp(y) / 2, so
          |h - xhat| <= dh = e_y / |gamma| + 3 a |y - beta| / |gamma|          (gamma = 0: h = 0, dh = |xhat|)
          -- the recovered xhat loses |beta / gamma| / |xhat| times more than bf16 precision when beta dominates y --
      g = fl(dy gamma): a |dy gamma|
      s1 = sum_c g, s2 = sum_c g h: 8 IT sequential adds per lane + log2(LPP) shuffles, then x fl(1/C):
          |m1 - M1| <= (n1 + 3) a mean|g|,  |m2 - M2| <= (n1 + 3) a mean(|g| (|xhat| + dh)) + mean(|g| dh)
      o = fl(rstd) * (g - m1 - h m2) (+ addend), bf16 store:
          |inner - INNER| <= a |g| + dm1 + dh |M2| + (|xhat| + dh) dm2 + 3 a (|g| + |M1| + |xhat M2|)
          |o - dx| <= rstd |inner - INNER| + 3 a rstd (|g| + |M1| + |xhat M2|) + a |dx|, then half a bf16 ulp.
      dgamma, dbeta: a lane chains U x trips pixels, then log2(32 / LPP) shuffles, 8 warps' shared atomics and one global
          atomic per block onto the initial value: n = U trips + log2(32/LPP) + 8 + blocks + 1 roundings of partial sums
          bounded by sum_p |dy| (|xhat| + dh) + |init| (dgamma; plus sum_p |dy| dh from h itself), sum_p |dy| + |init| (dbeta)."""
    a = A32
    gm = gamma.double()
    zero = gm == 0
    ag = gm.abs().masked_fill(zero, 1.0)
    e_y = (y.double() - (gm * xhat + beta.double())).abs()
    dh = torch.where(zero, xhat.abs(), e_y / ag + 3 * a * (y.double() - beta.double()).abs() / ag)
    gabs = (dy.double() * gm).abs()
    n1 = 8 * launch["it"] + int(math.log2(launch["lpp"]))
    dm1 = (n1 + 3) * a * gabs.mean(-1, keepdim=True)
    dm2 = (n1 + 3) * a * (gabs * (xhat.abs() + dh)).mean(-1, keepdim=True) + (gabs * dh).mean(-1, keepdim=True)
    mag = gabs + m1.abs() + (xhat * m2).abs()
    inner = a * gabs + dm1 + dh * m2.abs() + (xhat.abs() + dh) * dm2 + 3 * a * mag
    dx_ref_abs = rstd64[:, None] * (gabs + m1.abs() + (xhat * m2).abs())
    if addend is not None:
        dx_ref_abs = dx_ref_abs + addend.double().abs()
    e32 = (rstd64[:, None] * inner + 3 * a * rstd64[:, None] * mag + a * dx_ref_abs) * 1.01
    dyd = dy.double().abs()
    n = launch["u"] * launch["max_trips"] + int(math.log2(32 // launch["lpp"])) + 8 + launch["blocks"] + 1
    dg_b = (n * a * ((dyd * (xhat.abs() + dh)).sum(0) + dg_init.double().abs()) + (dyd * dh).sum(0)) * 1.01
    db_b = n * a * (dyd.sum(0) + db_init.double().abs()) * 1.01
    return e32, dg_b, db_b


def bf16_store_bound(ref, e32):
    """e32 plus half a bf16 ulp of the (fp32) value that was rounded."""
    return e32 + 0.5 * ulp(ref.abs() + e32, torch.bfloat16)


def describe_pixels(bad_pix, npix, launch):
    """bad_pix: bool [npix] -> the ln_bwd warps and grid-stride trips that wrote them."""
    idx = bad_pix.nonzero().flatten()
    slot = idx // launch["ppt"]
    warp, trip = slot % launch["nwarps"], slot // launch["nwarps"]
    return (f"{idx.numel()}/{npix} pixels wrong; first pixels {idx[:6].tolist()} on warps {warp[:6].tolist()} (blocks "
            f"{(warp[:6] // 8).tolist()}) in trips {trip[:6].tolist()}; wrong pixels per trip {torch.bincount(trip).tolist()}")


def describe_wgrad(bad, launch):
    """bad: bool [49 or 1, C] -> the taps and 64-channel chunks whose atomics were wrong."""
    idx = bad.nonzero()
    chunks = torch.unique(idx[:, 1] // WG_C).tolist()
    return (f"{idx.shape[0]} outputs wrong in 64-channel chunks {chunks[:8]} (launch {launch}); first (tap, channel) "
            f"{idx[:6].tolist()}")


# ---- depthwise forward / backward-data dispatch (launch_dwconv7) ----
DW_TW = 7        # kDwTW: output columns of a persistent / chunk-kernel tile
LN_NS = 32       # deepest fp32 reduction tree of a LayerNorm statistic in the three depthwise kernels (see dwconv7_ln_bound)


def dwconv_launch(B, H, W, C, sm_count, pipe=True):
    """The kernel launch_dwconv7 picks and its tiling.  Persistent kernel: CHUNK, nchunks, TH (14 unless H <= 7), tiles,
    the most co-resident groups sm_count * (2 if TH == 7 else 1) // nchunks (the occupancy query can only give fewer),
    and the fewest tiles any group then runs.  `pipe=False` is VDK_DWCONV_PIPE=0 (the round-1 chunk kernel, one tile per
    CTA).  Otherwise the all-channel fallback with tile edge T = 7 / 4 / 2."""
    chunk = next((c for c in (128, 96, 64) if C % c == 0), 0)
    if chunk and C // chunk <= 16:
        n = C // chunk
        if pipe:
            TH = 14 if H > 7 else 7
            tiles = B * -(-H // TH) * -(-W // DW_TW)
            gmax = max(1, min(tiles, sm_count * (2 if TH == 7 else 1) // n))
            return dict(kind="pipe", chunk=chunk, nchunks=n, TH=TH, TW=DW_TW, tiles=tiles, groups_max=gmax,
                        min_tiles_per_group=tiles // gmax)
        TH = min(7, H)
        return dict(kind="chunk", chunk=chunk, nchunks=n, TH=TH, TW=DW_TW, tiles=B * -(-H // TH) * -(-W // DW_TW))
    T = 7
    while T > 2 and (T + 6) ** 2 * C * 2 > 200 * 1024:
        T = 4 if T == 7 else 2
    return dict(kind="fallback", chunk=0, nchunks=1, T=T, TH=min(T, H), TW=T, tiles=B * -(-H // min(T, H)) * -(-W // T))


def describe_dw_tiles(bad, launch):
    """bad: bool [B, H, W, C] -> the tiles holding failures, and for the persistent kernel the group (CTA or cluster) and
    round that ran them (tile t runs on group t % groups in round t // groups, at the largest possible grid)."""
    B, H, W, _ = bad.shape
    th, tw = launch["TH"], launch["TW"]
    tiles_h, tiles_w = -(-H // th), -(-W // tw)
    idx = bad.any(-1).nonzero()
    t = torch.unique((idx[:, 0] * tiles_h + idx[:, 1] // th) * tiles_w + idx[:, 2] // tw)
    msg = f"{int(bad.any(-1).sum())} pixels wrong in {t.numel()}/{launch['tiles']} {th}x{tw} tiles {t[:6].tolist()}"
    if launch["kind"] == "pipe":
        g = launch["groups_max"]
        msg += f"; groups {(t[:6] % g).tolist()}, rounds {(t[:6] // g).tolist()}; wrong tiles per round {torch.bincount(t // g).tolist()}"
    if launch.get("chunk"):
        ch = torch.unique(bad.nonzero()[:, 3] // launch["chunk"]).tolist()
        msg += f"; channel chunks {ch[:8]}"
    return msg + f" ({launch['kind']})"


def dwconv7_ln_reference(x, w49, bias, gamma, beta, eps):
    """fp64 mode-0 forward: z = conv + bias, y = LayerNorm_C(z) gamma + beta and rstd = 1 / sqrt(var_C(z) + eps), plus
    what dwconv7_ln_bound needs."""
    conv, mag = dwconv7_reference(x, w49)
    z = conv + bias.double()
    mu = z.mean(-1, keepdim=True)
    d = z - mu
    var = d.pow(2).mean(-1)
    r = (var + eps).rsqrt()
    y = d * r[..., None] * gamma.double() + beta.double()
    return dict(z=z, mag=mag + bias.double().abs(), mu=mu, d=d, var=var, rstd=r, y=y)


def dwconv7_ln_bound(ref, gamma, beta, eps, chunk):
    """Bounds of vdk_dwconv7 mode 0 (y = bf16(LayerNorm_C(conv + bias) gamma + beta)) and of rstd_out; a = 2^-24.

    Kernel order (convnext.cu): z~ = bias + 49 FMAs in fp32:  |z~ - z| <= ez = 50 a mag.
      Statistics, two-pass per channel chunk and Chan's combination across the chunks of a pixel (persistent and chunk
      kernels), or two-pass over all of C (fallback).  Every sum is a tree of at most NS = 32 fp32 roundings (4 channels
      per thread, 5 shuffle levels, <= 16 partials across warps or chunks, x 1/n and its rounding):
        mean:  |mu~ - mu| <= e_mu = NS a mean|z| + mean(ez)
        centred sum of squares Q = sum (z - mu)^2: the computed one differs by at most
               (NS + 2) a Q + 2 sum |z - mu| ez + sum ez^2 + C e_mu^2     (a wrong mean adds C (mu~ - mu)^2 only)
               + 2 CHUNK sum_k |m_k - mu| e_mu_k                           (Chan: d_k = m~_k - mu~ carries the chunk mean error)
        rstd = rsqrtf(Q / C + eps): relative error e_r = e_Q / (2 (Q + C eps)) + 2^-22 + 2a   -> rstd_out's bound
      y = (z~ - mu~) rstd gamma + beta: |dxhat| <= rstd (ez + e_mu) + |xhat| e_r, then 4 fp32 roundings on
      |gamma xhat| + |beta| and half a bf16 ulp."""
    a = A32
    z, d, r = ref["z"], ref["d"], ref["rstd"]
    C = z.shape[-1]
    ez = 50 * a * ref["mag"]
    e_mu = LN_NS * a * z.abs().mean(-1, keepdim=True) + ez.mean(-1, keepdim=True)
    Q = d.pow(2).sum(-1)
    eQ = (LN_NS + 2) * a * Q + 2 * (d.abs() * ez).sum(-1) + ez.pow(2).sum(-1) + C * e_mu[..., 0] ** 2
    if chunk and C > chunk:
        zk = z.unflatten(-1, (C // chunk, chunk))
        e_mu_k = LN_NS * a * zk.abs().mean(-1) + ez.unflatten(-1, (C // chunk, chunk)).mean(-1)
        eQ = eQ + 2 * chunk * ((zk.mean(-1) - ref["mu"]).abs() * e_mu_k).sum(-1)
    e_r = (eQ / (2 * (Q + C * eps)) + 2.0 ** -22 + 2 * a) * 1.01
    xhat = d * r[..., None]
    dxh = r[..., None] * (ez + e_mu) + xhat.abs() * e_r[..., None]
    g = gamma.double().abs()
    e32 = (g * dxh + 4 * a * (g * xhat.abs() + beta.double().abs())) * 1.01
    return e32 + 0.5 * ulp(ref["y"].abs() + e32, torch.bfloat16), r * e_r


def layernorm_bwd_dgamma(y, beta, gamma, dy, launch, dg_init):
    """dgamma of vdk_layernorm_bwd against the xhat the kernel can see, xh = (y - beta) / gamma in fp64 from the saved y
    (channels with gamma = 0 excluded by the caller).  The kernel's h = (y - beta) * fl(1 / gamma) carries 3 a |xh|;
    dy * h is chained over U x trips pixels per lane, log2(32 / LPP) shuffles, 8 shared and one global atomic per block:
        |dgamma - init - sum dy xh| <= n a (sum |dy xh| + |init|) + 3 a sum |dy xh|,  n as in layernorm_bwd_bound."""
    a = A32
    gm = gamma.double()
    xh = (y.double() - beta.double()) / gm.masked_fill(gm == 0, 1.0)
    t = dy.double() * xh
    n = launch["u"] * launch["max_trips"] + int(math.log2(32 // launch["lpp"])) + 8 + launch["blocks"] + 1
    return dg_init.double() + t.sum(0), ((n * a) * (t.abs().sum(0) + dg_init.double().abs()) + 3 * a * t.abs().sum(0)) * 1.01


# ---- BatchNorm with batch statistics over the rows of [R, C] (train_ops.cu) ----
def bn_rows_depth(R):
    """Roundings of a column sum: a thread chains ceil(R / 8) rows (generic kernels: 8 warps stride the rows; the vector
    kernel's 256 threads chain fewer), then <= 5 shuffles and 8 per-warp partials."""
    return -(-R // 8) + 16


def batchnorm_fwd_reference(x, weight, bias, eps, momentum, rm, rv):
    xd = x.double()
    R = xd.shape[0]
    mu = xd.mean(0)
    d = xd - mu
    var = d.pow(2).mean(0)
    r = (var + eps).rsqrt()
    y = d * r * weight.double() + bias.double()
    return dict(x=xd, mu=mu, d=d, var=var, rstd=r, y=y, rm=(1 - momentum) * rm.double() + momentum * mu,
                rv=(1 - momentum) * rv.double() + momentum * var * R / (R - 1))


def batchnorm_fwd_bound(ref, weight, bias, eps, momentum, rm, rv, out_dtype):
    """Bounds of vdk_batchnorm_train_fwd; a = 2^-24, n = bn_rows_depth(R).
      mean: e_mu = (n + 2) a mean|x|;  Q = sum (x - mu)^2: e_Q = (n + 3) a Q + R e_mu^2 (a wrong mean adds R e_mu^2 only)
      rstd = rsqrtf(Q / R + eps): e_r = e_Q / (2 (Q + R eps)) + 2^-22 + 2a relative
      y: the generic kernels form (x - mu) rstd w + b; the vector kernel fma(x, rstd w, b - mu rstd w), which cancels
      when |mu| >> std: |dy| <= |w| (rstd e_mu + |xhat| e_r) + 4 a (|x| + |mu|) rstd |w| + 4 a |b|, then the output
      rounding (half a bf16 ulp, or a |y| in fp32)
      running_mean: 3 a (|(1-m) rm| + |m mu|) + m e_mu;  running_var: 4 a (|(1-m) rv| + |m var_unbiased|) + m var_u e_Q / Q."""
    a = A32
    x, d, r = ref["x"], ref["d"], ref["rstd"]
    R = x.shape[0]
    n = bn_rows_depth(R)
    e_mu = (n + 2) * a * x.abs().mean(0)
    Q = d.pow(2).sum(0)
    eQ = (n + 3) * a * Q + R * e_mu ** 2
    e_r = (eQ / (2 * (Q + R * eps)) + 2.0 ** -22 + 2 * a) * 1.01
    w, b = weight.double().abs(), bias.double().abs()
    xhat = d * r
    e32 = (w * (r * e_mu + xhat.abs() * e_r) + 4 * a * (x.abs() + ref["mu"].abs()) * r * w + 4 * a * b) * 1.01
    yb = e32 + (0.5 * ulp(ref["y"].abs() + e32, torch.bfloat16) if out_dtype == torch.bfloat16 else a * (ref["y"].abs() + e32))
    m = momentum
    rm_b = 3 * a * ((1 - m) * rm.double().abs() + m * ref["mu"].abs()) + m * e_mu
    vu = ref["var"] * R / (R - 1)
    rv_b = 4 * a * ((1 - m) * rv.double().abs() + m * vu) + m * vu * eQ / Q.clamp_min(1e-300)
    return yb, r * e_r, e_mu * 1.01, rm_b * 1.01, rv_b * 1.01


def batchnorm_bwd_reference(x, dy, weight, save_mean, save_rstd):
    """fp64 backward at the forward's saved fp32 statistics: xhat = (x - mean) rstd, dx = w rstd (dy - mean dy -
    xhat mean(dy xhat)), dweight = sum dy xhat, dbias = sum dy."""
    xhat = (x.double() - save_mean.double()) * save_rstd.double()
    g = dy.double()
    m1, m2 = g.mean(0), (g * xhat).mean(0)
    dx = weight.double() * save_rstd.double() * (g - m1 - xhat * m2)
    return dict(xhat=xhat, g=g, m1=m1, m2=m2, dx=dx, dw=(g * xhat).sum(0), db=g.sum(0))


def batchnorm_bwd_bound(ref, weight, save_rstd, dw_init, db_init, out_dtype):
    """Bounds of vdk_batchnorm_train_bwd; a = 2^-24, n = bn_rows_depth(R).  xh = (x - mean) rstd in fp32: 2a |xhat|
    (the subtraction of a mean far from 0 included: it is relative to |x - mean|).
      dbias += sum dy: n a (sum |dy| + |init|);  dweight += sum dy xh: n a (sum |dy xhat| + |init|) + 3 a sum |dy xhat|
      m1 = s1 / R, m2 = s2 / R: (n + 2) a mean|dy|, (n + 2) a mean|dy xhat| + 3 a mean|dy xhat|
      dx = w rstd (dy - m1 - xh m2): |w rstd| (dm1 + |xhat| dm2 + 2 a |xhat m2| + 3 a (|dy| + |m1| + |xhat m2|))
           + 3 a |dx|, then the output rounding."""
    a = A32
    xhat, g = ref["xhat"], ref["g"]
    R = g.shape[0]
    n = bn_rows_depth(R)
    t = (g * xhat).abs()
    db_b = n * a * (g.abs().sum(0) + db_init.double().abs()) * 1.01
    dw_b = (n * a * (t.sum(0) + dw_init.double().abs()) + 3 * a * t.sum(0)) * 1.01
    dm1 = (n + 2) * a * g.abs().mean(0)
    dm2 = (n + 5) * a * t.mean(0)
    wr = (weight.double() * save_rstd.double()).abs()
    inner = dm1 + xhat.abs() * dm2 + 2 * a * (xhat * ref["m2"]).abs() + 3 * a * (g.abs() + ref["m1"].abs() + (xhat * ref["m2"]).abs())
    e32 = (wr * inner + 3 * a * ref["dx"].abs()) * 1.01
    dxb = e32 + (0.5 * ulp(ref["dx"].abs() + e32, torch.bfloat16) if out_dtype == torch.bfloat16 else a * (ref["dx"].abs() + e32))
    return dxb, dw_b, db_b


# ------------------------------------------------------------------------------------------------------------------------------
# wgmma GEMM (csrc/gemm.cu): accumulator, epilogues, split-K and the fused LayerNorm-backward epilogue

# Documented accuracy of the fp16x2 activations (gemm.cu, include/vdk_b200.h).  test_gemm_gpu.py's sweeps run every finite
# 16-bit pre-activation through them: on an H100 the worst GELU error was 4.3e-4 |x|, the worst GELU' error 7.6e-3 (near
# |x| = 3, where the error of tanh.approx.f16 in 1 - tanh^2 is multiplied by x (c1 + 3 c3 x^2) ~ 5)
GELU_REL_ERR = 6e-4     # |gelu~(x) - gelu(x)| <= GELU_REL_ERR |x|
GELU_GRAD_ERR = 8e-3    # |gelu~'(x) - gelu'(x)| <= GELU_GRAD_ERR
GELU_GRAD_MAX = 1.13    # max |gelu'(x)| = 1.1289...


def gelu64(x):
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.special.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def out_rounding(ref, dtype):
    return torch.zeros_like(ref) if dtype == torch.float32 else ulp(ref, dtype)


def acc_reference(a, b):
    """fp64 A . B^T of the 16-bit operands and the fp32 accumulation bound (ceil(K/16) + 17) 2^-23 (|A| |B|^T)."""
    A, Bm = a.double(), b.double()
    K = A.shape[1]
    return A @ Bm.t(), (-(-K // 16) + 17) * U32 * (A.abs() @ Bm.abs().t())


def epilogue_reference(a, b, epilogue, out_dtype, bias=None, gamma=None, beta=None, residual=None, aux=None, ln_eps=1e-6):
    """fp64 epilogue of the exact accumulator A . B^T (a [M, K], b [N, K]) and the elementwise bound of vdk_gemm's D.
    Returns a dict with ref and bound, and with aux_ref / aux_bound when `aux` (the kernel's saved pre-activation of a
    GELU epilogue) is given.

      x = acc + bias in fp32:         |x~ - x| <= ex = e_acc + 2^-24 |x|  (no rounding without a bias)
      NONE                            ref = x, bound ex
      GELU                            ref = gelu(x), bound max|gelu'| ex + GELU_REL_ERR |x| + 2^-24 |ref|
      GELU + aux_out                  aux: ref x, bound ex + ulp(x); out: ref gelu(aux), bound GELU_REL_ERR |aux| + 2^-24 |ref|
      SCALE_RESIDUAL                  ref = res + gamma x, bound |gamma| ex + 2^-24 (|gamma x| + |ref|)
      MUL_GELU_GRAD                   ref = acc gelu'(pre), bound (|gelu'(pre)| + GELU_GRAD_ERR) e_acc + GELU_GRAD_ERR |acc|
                                      + 2^-24 |ref|
      LAYERNORM (row of n = N values, E = max_j ex_j, r = 1/sqrt(var + eps), d_i = x_i - mean):
        mean: ~n/4 sequential fp32 adds per thread, 2 shuffles, a divide: |dmean| <= E + (n/4 + 3) 2^-24 mean|x| = dm
        d~_i off by D_i = ex_i + dm + 2^-24 |d_i|; the two-pass variance off by the relative
        rho = (2 max D sqrt(var) + max D^2) / (var + eps) + (n/4 + 4) 2^-24, rsqrtf adds 2^-22:
        bound |g_i| r D_i + |g_i d_i| r (rho / 2 + 2^-22) + 2^-24 (3 |g_i d_i| r + |ref|)
    plus one ulp of a 16-bit output type at |ref| everywhere.
    """
    from visiondk_b200 import _lib
    acc, e = acc_reference(a, b)
    N = acc.shape[1]
    x = acc + bias.double() if bias is not None else acc
    ex = e + 2.0 ** -24 * x.abs() if bias is not None else e
    out = {}
    if epilogue == _lib.EPI_NONE:
        ref, bound = x, ex
    elif epilogue == _lib.EPI_GELU and aux is not None:
        out["aux_ref"], out["aux_bound"] = x, ex + ulp(x, out_dtype)
        pre = aux.double()
        ref = gelu64(pre)
        bound = GELU_REL_ERR * pre.abs() + 2.0 ** -24 * ref.abs()
    elif epilogue == _lib.EPI_GELU:
        ref = gelu64(x)
        bound = GELU_GRAD_MAX * ex + GELU_REL_ERR * x.abs() + 2.0 ** -24 * ref.abs()
    elif epilogue == _lib.EPI_SCALE_RESIDUAL:
        g = gamma.double()
        ref = residual.double() + g * x
        bound = g.abs() * ex + 2.0 ** -24 * ((g * x).abs() + ref.abs())
    elif epilogue == _lib.EPI_MUL_GELU_GRAD:
        gp = gelu_grad64(residual.double())
        ref = acc * gp
        bound = (gp.abs() + GELU_GRAD_ERR) * e + GELU_GRAD_ERR * acc.abs() + 2.0 ** -24 * ref.abs()
    elif epilogue == _lib.EPI_LAYERNORM:
        mean = x.mean(1, keepdim=True)
        dv = x - mean
        var = (dv * dv).mean(1, keepdim=True)
        r = 1.0 / torch.sqrt(var + ln_eps)
        g, bt = gamma.double(), beta.double()
        ref = dv * r * g + bt
        E = ex.amax(1, keepdim=True)
        dm = E + (N / 4 + 3) * 2.0 ** -24 * x.abs().mean(1, keepdim=True)
        Di = ex + dm + 2.0 ** -24 * dv.abs()
        Dmax = Di.amax(1, keepdim=True)
        rho = (2 * Dmax * var.sqrt() + Dmax * Dmax) / (var + ln_eps) + (N / 4 + 4) * 2.0 ** -24
        gd = (g * dv).abs()
        bound = g.abs() * r * Di + gd * r * (rho / 2 + 2.0 ** -22) + 2.0 ** -24 * (3 * gd * r + ref.abs())
    else:
        raise ValueError(epilogue)
    out["ref"], out["bound"] = ref, bound + out_rounding(ref, out_dtype)
    return out


def split_k_bound(a, b, n_split):
    """Each split's partial is one wgmma chain over its K range; adding n_split partials (atomics or the slab sum) adds at most
    n_split more roundings, each 2^-23 of the running |sum|: (ceil(K/16) + 17 + n_split) 2^-23 (|A| |B|^T).  At K = 12544 and
    50176 the measured error is a few 1e-4 of this bound: the bound takes every one of the ~800 / ~3200 roundings at its maximum
    and of one sign, and |A| |B|^T of random-sign operands exceeds |A B^T| by ~sqrt(K), while the rounding errors of the real
    sums cancel like a random walk.  It stays the worst-case model; a lost or doubled split (one partial, ~sqrt(K / n_split)
    times the operand scales) is still several times larger than it."""
    A, Bm = a.double(), b.double()
    return A @ Bm.t(), (-(-A.shape[1] // 16) + 17 + n_split) * U32 * (A.abs() @ Bm.abs().t())


def fused_launch(M, N, G, sm):
    """Summation depths of the fused LayerNorm-backward epilogue (VDK_EPI_LN_BWD) in ln_bwd_launch's terms
    (layernorm_bwd_bound): a row group's sums chain 16 adds per 64-column box, G / 64 boxes and 2 shuffles (n1 = 8 IT +
    log2 LPP with IT = G / 64, LPP = 4 covers it); a column sum chains 6 roundings per tile over a CTA's tiles, 8 warps and
    the slab reduction's partials (8 groups)."""
    BN = 256 if N % 256 == 0 else 128
    num_n = N // BN
    tiles = -(-M // 128) * num_n
    # clusters (G > BN): at least half the SMs hold a co-resident cluster; fewer CTAs only lengthen the chains
    slots = sm if G <= BN else sm // 2
    grid = min(tiles, slots - slots % num_n)
    per_cta = -(-tiles // grid)
    parts = (grid // num_n) * (N // G)
    return dict(lpp=4, it=G // 64, u=1, max_trips=6 * per_cta + 8 + -(-parts // 8) + 8, blocks=0, per_cta=per_cta)
