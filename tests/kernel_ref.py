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
