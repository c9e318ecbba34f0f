"""References for the fused clip + SGD + EMA step (csrc/optim.cu): torch's semantics in fp64, a bit-exact numpy restatement of the
kernel's fp32 operation sequence, an exact sum of squares and an elementwise bound on the kernel's roundings.

What one step means (Trainer.update: GradScaler.unscale_ -> clip_grad_norm_ -> GradScaler.step(SGD) -> zero_grad ->
ModelEMA.update), restated from torch's definitions, not from the kernel:
  S = sum over every group of g^2;  if S is not finite the SGD step is skipped (p and momentum unchanged);
  coef = min(max_norm / (sqrt(S) + 1e-6), 1)                                   (clip_grad_norm_)
  d = g*coef + wd*p;  buf = d on the first applied step (torch clones it), else m*buf + d;  no buffer at m == 0 (buf = d)
  p -= lr*buf                                                                  (torch.optim.SGD)
  ema = ema*dk + (1 - dk)*p,  dk = 0.9999 * (1 - exp(-updates / 2000))        (ModelEMA.update, on every step)
The hyper-parameters are the fp32 values the kernel receives: torch too casts a Python scalar to the tensor's type.

Rounding bound of the kernel (u = 2^-24, fp32's unit roundoff; every bound is on |kernel - fp64 reference| per element):
  * S: every fp32 square is exact in fp64 and all terms are >= 0, so L sequential fp64 additions give a relative error
    <= L * 2^-53 (plus one rounding when the exact value is itself rounded for the comparison).  `sumsq_depth(n)` counts L.
  * coef: fp64 sqrt (rel. 2^-53, plus half of S's error), rounded to fp32 (u), + 1e-6f (u; and 1e-6f differs from 1e-6 by
    <= u relative), divided in fp32 (u): |coef_k - coef| <= coef * e_c, e_c = 4u + (L/2 + 2) * 2^-53.  The clamp at 1 does
    not add to it: it only moves coef towards the reference's value when the reference is also clamped near 1.
  * g*coef rounded once: e_gc = |g| e_c coef + u |g| coef (1 + e_c).
  * d = fmaf(wd, p, g*coef), one rounding of a bounded magnitude: e_d = e_gc + u * D,   D = |wd p| + |g| coef (1+e_c)(1+u).
  * buf = fmaf(m, mom, d) (exact product, one rounding): e_b = e_d + u * (|m mom| + D + e_d)   (|m mom| = 0 without history).
  * p = fmaf(-lr, buf, p): e_p = lr e_b + u * (|p| + lr (|m mom| + D + e_b)).
  * ema = fl(fl(ema*dk) + fl(omd*p)), three roundings: e_e = omd e_p + u |ema dk| + u omd (|p'| + e_p)
                                                             + u (|ema dk| (1+u) + omd (|p'| + e_p)(1+u)).
  A skipped step has e_p = e_b = 0: only the EMA's three roundings remain.

Bit-exact restatement: the kernel's operations are all specified (IEEE fp32 multiply, divide, add, `fmaf`, `__fmul_rn`,
`__fadd_rn`; no fast-math, denormals kept), so `kernel_step` reproduces its bits.  `fmaf` is emulated exactly: the product of
two fp32 values is exact in fp64, the fp64 sum with the third operand is rounded but its TwoSum residual is exact, and the
one case where rounding that fp64 sum to fp32 differs from rounding the exact value, an fp64 sum exactly on an fp32 midpoint
with a non-zero residual, is corrected towards the residual.
"""
import math
from fractions import Fraction

import numpy as np
import torch

from kernel_ref import _GUARD

U = 2.0 ** -24          # fp32 unit roundoff
U64 = 2.0 ** -53        # fp64 unit roundoff
RED_THREADS, RED_BLOCKS_MAX = 256, 1184   # csrc/optim.cu kRedThreads, kRedBlocksMax
STEP_THREADS, STEP_BLOCKS_MAX = 256, 132 * 16
F32 = np.float32


# ---- exact fp32 fused multiply-add --------------------------------------------------------------------------------------
def fmaf(a, b, c):
    """Correctly rounded fp32 a*b + c (numpy arrays or scalars of fp32), as CUDA's fmaf."""
    a, b, c = (np.asarray(x, dtype=F32) for x in (a, b, c))
    prod = a.astype(np.float64) * b.astype(np.float64)   # exact: 24 + 24 significant bits
    cd = c.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        s = prod + cd
        bb = s - prod
        res = (prod - (s - bb)) + (cd - bb)               # TwoSum: s + res == prod + c exactly
        r = s.astype(F32)
        up = np.nextafter(r, F32(np.inf))
        dn = np.nextafter(r, F32(-np.inf))
        below = r.astype(np.float64) <= s
        lo = np.where(below, r, dn)
        hi = np.where(below, up, r)
        mid = (lo.astype(np.float64) + hi.astype(np.float64)) * 0.5
        fix = np.isfinite(r) & (s == mid) & (res != 0)
        out = np.where(fix, np.where(res > 0, hi, lo), r)
    return out.astype(F32)


def round_fraction_to_f32(x: Fraction) -> np.float32:
    """Round-to-nearest-even of an exact rational into fp32 (subnormals and overflow included)."""
    if x == 0:
        return F32(0.0)
    sign = -1 if x < 0 else 1
    ax = abs(x)
    e = ax.numerator.bit_length() - ax.denominator.bit_length()
    if Fraction(2) ** e > ax:
        e -= 1
    q = max(e - 23, -149)                                 # quantum of the fp32 grid at |x|
    scaled = ax / Fraction(2) ** q
    n = scaled.numerator // scaled.denominator
    rem = scaled - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    val = Fraction(n) * Fraction(2) ** q
    if val >= Fraction(2) ** 128:
        return F32(sign * np.inf)
    return F32(sign * float(val))


def fmaf_exact(a, b, c) -> np.float32:
    """fmaf of three fp32 scalars through exact rational arithmetic."""
    return round_fraction_to_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


# ---- sum of squares ---------------------------------------------------------------------------------------------------
def exact_sumsq(g) -> Fraction:
    """The exact sum of squares of fp32 values: each v = M * 2^E with an integer M < 2^24, so v^2 = M^2 * 4^E and the
    per-exponent sums of M^2 are exact integers."""
    g = np.ascontiguousarray(np.asarray(g, dtype=F32).ravel())
    if not np.isfinite(g).all():
        raise ValueError("exact_sumsq needs finite values")
    mant, ex = np.frexp(g)
    m = np.abs(np.ldexp(mant.astype(np.float64), 24)).astype(np.int64)   # exact: |mant| < 1 has 24 bits
    e = ex.astype(np.int64) - 24
    total = Fraction(0)
    order = np.argsort(e, kind="stable")
    e_s, m_s = e[order], m[order]
    bounds = np.flatnonzero(np.diff(e_s)) + 1
    for seg_m, seg_e in zip(np.split(m_s, bounds), np.split(e_s, bounds)):
        if seg_m.size == 0:
            continue
        sq = seg_m * seg_m                                  # < 2^48
        pad = (-sq.size) % 8192
        chunks = np.concatenate([sq, np.zeros(pad, np.int64)]).reshape(-1, 8192).sum(axis=1)   # each < 2^61
        s = sum(int(c) for c in chunks)
        total += Fraction(s) * Fraction(2) ** (2 * int(seg_e[0]))
    return total


def sumsq_blocks(n: int) -> int:
    return max(1, min((n // 4 + RED_THREADS - 1) // RED_THREADS, RED_BLOCKS_MAX))


def sumsq_depth(n: int) -> int:
    """Longest chain of fp64 additions in vdk_grad_sumsq for n elements: a thread's float4 sweep (4 per float4, plus the tail),
    the in-block tree, the final kernel's per-thread sum of partials and its tree, and the accumulate add."""
    blocks = sumsq_blocks(n)
    per_thread = -(-(n // 4) // (blocks * RED_THREADS)) if n >= 4 else 0
    return 4 * per_thread + 1 + 8 + -(-blocks // RED_THREADS) + 8 + 1


# ---- the kernel's fp32 sequence, bit for bit ----------------------------------------------------------------------------
def kernel_coef(sumsq: float, max_norm) -> np.float32:
    total_norm = F32(np.sqrt(np.float64(sumsq)))
    with np.errstate(invalid="ignore", divide="ignore"):
        return F32(np.fmin(F32(max_norm) / (total_norm + F32(1e-6)), F32(1.0)))


def kernel_step(p, g, mom, ema, sumsq, max_norm, lr, momentum, weight_decay, first_step, ema_decay, ema_omd, zero_grad):
    """numpy restatement of sgd_clip_ema_kernel: returns (p, g, mom, ema) after one call (ema None when absent)."""
    p, g, mom = (np.array(x, dtype=F32, copy=True) for x in (p, g, mom))
    ema = None if ema is None else np.array(ema, dtype=F32, copy=True)
    lr, m, wd = F32(lr), F32(momentum), F32(weight_decay)
    if math.isfinite(sumsq):
        coef = kernel_coef(sumsq, max_norm)
        with np.errstate(invalid="ignore", over="ignore"):
            d = g * coef
        if wd != 0:
            d = fmaf(wd, p, d)
        if m == 0 or first_step:
            buf = d
        else:
            buf = fmaf(m, mom, d)
        p = fmaf(-lr, buf, p)
        if m != 0:
            mom = buf.astype(F32)
    if ema is not None:
        ema = kernel_ema(ema, p, ema_decay, ema_omd)
    if zero_grad:
        g = np.zeros_like(g)
    return p, g, mom, ema


def kernel_ema(ema, src, d, omd):
    """ema_only_kernel and the step's EMA: fl(fl(ema * d) + fl(omd * src))."""
    with np.errstate(over="ignore", invalid="ignore"):
        return (np.asarray(ema, F32) * F32(d)) + (F32(omd) * np.asarray(src, F32))


def ema_decay(updates: int, decay: float = 0.9999, tau: float = 2000.0):
    """models/ema.py:24, and the fp32 (d, 1 - d) pair the optimizer passes."""
    d = decay * (1 - math.exp(-updates / tau))
    return d, 1 - d


# ---- fp64 semantics and the bound ---------------------------------------------------------------------------------------
# These take numpy arrays or torch tensors (so full-size groups can be checked on the device in fp64) and compute in fp64.
def _f64(x):
    return x.double() if torch.is_tensor(x) else np.asarray(x, np.float64)


def reference_coef(sumsq: float, max_norm: float) -> float:
    return min(float(max_norm) / (math.sqrt(sumsq) + 1e-6), 1.0)


def reference_step(p, g, mom, ema, sumsq, max_norm, lr, momentum, weight_decay, has_buf, ema_d, ema_omd):
    """One reference update in fp64.  `has_buf`: torch holds a momentum buffer (a step with momentum != 0 has been applied
    before).  Returns (p, mom, ema, has_buf, applied)."""
    p, g, mom = _f64(p), _f64(g), _f64(mom)
    if not math.isfinite(sumsq):
        new_p, new_mom, applied = p, mom, False
    else:
        coef = reference_coef(sumsq, max_norm)
        d = g * coef + weight_decay * p
        if momentum == 0:
            buf, new_mom = d, mom
        else:
            buf = momentum * mom + d if has_buf else d
            new_mom, has_buf = buf, True
        new_p, applied = p - lr * buf, True
    new_ema = None if ema is None else _f64(ema) * ema_d + ema_omd * new_p
    return new_p, new_mom, new_ema, has_buf, applied


def step_bounds(p, g, mom, ema, sumsq, max_norm, lr, momentum, weight_decay, has_buf, ema_d, ema_omd, depth):
    """Elementwise bounds (e_p, e_mom, e_ema) on |kernel - reference_step| for one step from the same fp32 state; see the
    module docstring for the derivation."""
    p, g, mom = abs(_f64(p)), abs(_f64(g)), abs(_f64(mom))
    if not math.isfinite(sumsq):
        e_p = e_b = 0 * p
        p_new = p
    else:
        coef = reference_coef(sumsq, max_norm)
        e_c = 4 * U + (depth / 2 + 2) * U64
        e_gc = g * (coef * e_c) + g * (U * coef * (1 + e_c))
        D = weight_decay * p + g * (coef * (1 + e_c) * (1 + U))
        e_d = e_gc + U * D
        with_hist = momentum != 0 and has_buf
        hist = momentum * mom if with_hist else 0 * p
        e_b = e_d + U * (hist + D + e_d) if with_hist else e_d
        e_p = lr * e_b + U * (p + lr * (hist + D + e_b))
        p_new = p + lr * (hist + D)
        if momentum == 0:
            e_b = 0 * p
    e_e = None
    if ema is not None:
        ed = abs(_f64(ema)) * ema_d
        pe = p_new + e_p
        e_e = ema_omd * e_p + U * ed + U * ema_omd * pe + U * (ed * (1 + U) + ema_omd * pe * (1 + U))
    return e_p, e_b, e_e


def ema_bound(ema, src, d, omd):
    """|kernel_ema - (ema*d + omd*src)| for fp32 inputs: three roundings."""
    ed = abs(_f64(ema)) * d
    so = abs(_f64(src)) * omd
    return U * ed + U * so + U * (ed + so) * (1 + U) ** 2


# ---- NaN-guarded flat device buffers ------------------------------------------------------------------------------------
class GuardedVec:
    """A length-n fp32 view with `pad` guard elements on each side, every guard holding kernel_ref's NaN pattern (the
    `Guarded` pattern for a flat buffer).  `pad` is a multiple of 4, so the view keeps the buffer's 16-byte alignment."""

    def __init__(self, values, pad=64, device="cuda"):
        values = torch.as_tensor(values, dtype=torch.float32).reshape(-1)
        n = values.numel()
        self.buf = torch.empty(n + 2 * pad, dtype=torch.float32, device=device)
        self.bits = self.buf.view(torch.int32)
        self.bits.fill_(_GUARD[torch.float32])
        self.view = self.buf[pad:pad + n]
        self.view.copy_(values)
        self.pad, self.n = pad, n

    def ptr(self):
        return self.buf.data_ptr() + 4 * self.pad        # also for n == 0, where torch reports an empty view's pointer as 0

    def host(self):
        return self.view.cpu().numpy()

    def guard_errors(self):
        g = _GUARD[torch.float32]
        bad = int((self.bits[:self.pad] != g).sum()) + int((self.bits[self.pad + self.n:] != g).sum())
        return f"{bad} guard elements written" if bad else ""
