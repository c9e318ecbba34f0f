"""CPU self-tests of kernel_ref.attention_bwd_reference's bound: an fp32 emulation of attention_bwd_kernel (vit.cu), phase by
phase in the kernel's order, must stay inside the bound, on random and on crafted softmaxes; and each plausible defect of
the kernel must fall outside it."""
import math

import pytest
import torch

from kernel_ref import LOG2E, attention_bwd_reference, attention_reference, crafted_qkv

C_LOG2 = float(torch.tensor(LOG2E, dtype=torch.float32)) * 0.125   # scale * fp32(log2 e): 0.125 is exact


def chain(a, b):
    """a @ b as a chain of mma.sync k16 steps: each step's 16 exact products are summed and added to the fp32 accumulator
    with one rounding."""
    acc = torch.zeros(a.shape[:-1] + b.shape[-1:], dtype=torch.float32)
    for k0 in range(0, a.shape[-1], 16):
        acc = (acc.double() + a[..., k0:k0 + 16].double() @ b[..., k0:k0 + 16, :].double()).float()
    return acc


def bf16r(t):
    return t.to(torch.bfloat16).float()


def emulate_bwd(qkv, out, dout, lse2, defect=None):
    """attention_bwd_kernel in fp32 for every (image, head) at once: rows are zero-padded to Np = 16 ceil(N / 16).
    Returns dqkv [B, N, 3, H, 64] (fp32 holding bf16 values)."""
    B, N, _, H, D = qkv.shape
    Np = 16 * -(-N // 16)

    def pad(t):  # [B, N, H, 64] -> [B*H, Np, 64]
        t = t.float().transpose(1, 2).reshape(B * H, N, D)
        return torch.nn.functional.pad(t, (0, 0, 0, Np - N))
    q, k, v = (pad(qkv[:, :, i]) for i in range(3))
    o, do = pad(out.view(B, N, H, D)), pad(dout.view(B, N, H, D))
    lse = lse2.float().reshape(B * H, N)
    if defect == "next_row_lse":
        lse = lse.roll(-1, 1)
    lse = torch.nn.functional.pad(lse, (0, Np - N))
    real = torch.arange(Np) < N

    # D_i: lane `half` chains fma(o[c+1], do[c+1]) then fma(o[c], do[c]) over its 32 columns (exact bf16 products), then
    # the two lanes' sums are added
    prod = o * do
    lanes = []
    for half in range(2):
        acc = torch.zeros(B * H, Np)
        for col in range(half * 32, half * 32 + 32, 2):
            acc = acc + prod[..., col + 1]
            acc = acc + prod[..., col]
        lanes.append(acc)
    Dv = lanes[0] if defect == "D_half" else lanes[0] + lanes[1]
    if defect == "no_D":
        Dv = torch.zeros_like(Dv)

    # phase 1: P = ex2.approx.ftz(fma(S, c, -lse2)) for real rows and columns, stored bf16
    S = chain(q, k.transpose(-1, -2))
    x = (S.double() * C_LOG2 - lse[..., None].double()).float()
    P = torch.exp2(x.double()).float()
    P = torch.where(P < 2.0 ** -126, torch.zeros_like(P), P)
    keep = real[:, None] & (real[None, :] | (defect == "no_column_mask"))
    P = bf16r(torch.where(keep, P, torch.zeros_like(P)))
    # phase 2: dV = P^T dO
    dv = bf16r(chain(P if defect == "dV_from_P" else P.transpose(-1, -2), do))
    # phase 3: dS = bf16(0.125 P (dO V^T - D)), in place over P
    dP = chain(do, v.transpose(-1, -2))
    scale = 1.0 if defect == "no_scale" else 0.125
    dS = bf16r((scale * P) * (dP - Dv[..., None]))
    # phases 4 and 5: dQ = dS K, dK = dS^T Q
    dq = bf16r(chain(dS, k))
    dk = bf16r(chain(dS if defect == "dK_from_dS" else dS.transpose(-1, -2), q))
    g = torch.stack([dq, dk, dv])[:, :, :N].reshape(3, B, H, N, D)
    return g.permute(1, 3, 0, 2, 4)


def isolated(qkv):
    """The kernel's operands from the fp64 forward: out = bf16(O), lse2 = fp32(lse2)."""
    out, _, lse2, _ = attention_reference(qkv)
    return out.to(torch.bfloat16), lse2.float()


def within(got, ref, bound):
    return bool(((got.double() - ref).abs() <= bound).all())


def worst(got, ref, bound):
    return float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())


def random_case(B, N, H, seed, scale=1.5):
    gen = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(B, N, 3, H, 64, generator=gen) * scale).to(torch.bfloat16)
    dout = torch.randn(B, N, H * 64, generator=gen).to(torch.bfloat16)
    return qkv, dout


def one_hot_case(N, ks, seed):
    """Row i peaks on key 5 with P_peak close to 1 - 2^-k, k = ks[i % len]: every other score is 0 and the peak's is
    alpha = bf16(8 ln((N - 1)(2^k - 1)))."""
    alphas = [float(torch.tensor(8 * math.log((N - 1) * (2.0 ** k - 1))).to(torch.bfloat16)) for k in ks]
    beta = torch.zeros(N)
    beta[5] = 1.0
    qkv = crafted_qkv(1, N, 2, alphas, beta, seed, dense=True, device="cpu")
    return qkv, torch.randn(1, N, 2 * 64).to(torch.bfloat16)


def below_800_case(N, seed):
    """Every real score below -800 raw units: lse2 < -128, so exp2(0 - lse2) of a padded key overflows to inf."""
    beta = -800.0 - 4.0 * (torch.arange(N) % 8).float()
    qkv = crafted_qkv(1, N, 2, [1.0, 1.5], beta, seed, dense=True, device="cpu")
    return qkv, torch.randn(1, N, 2 * 64).to(torch.bfloat16)


CASES = {
    "random_37": lambda: random_case(2, 37, 2, 0),
    "random_208": lambda: random_case(1, 208, 2, 1),
    "random_1": lambda: random_case(3, 1, 2, 2),
    "one_hot_197": lambda: one_hot_case(197, [2, 6, 10, 16, 24], 3),
    "below_800_17": lambda: below_800_case(17, 4),
    "uniform_50": lambda: (crafted_qkv(1, 50, 2, [0.0], torch.ones(50), 5, dense=True, device="cpu"),
                           torch.randn(1, 50, 128).to(torch.bfloat16)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_emulated_kernel_stays_inside_the_bound(name):
    qkv, dout = CASES[name]()
    out, lse2 = isolated(qkv)
    ref, bound = attention_bwd_reference(qkv, out, dout, lse2)
    got = emulate_bwd(qkv, out, dout, lse2)
    for i, op in enumerate("qkv"):
        w = worst(got[:, :, i], ref[:, :, i], bound[:, :, i])
        print(f"{name} d{op}: worst {w:.4f} of the bound")
        assert w <= 1.0, (name, op, w)


def test_zero_dout_rows_have_exact_zero_dq_and_a_zero_bound():
    qkv, dout = random_case(1, 37, 2, 6)
    dout.view(1, 37, 2, 64)[:, ::5] = 0
    out, lse2 = isolated(qkv)
    ref, bound = attention_bwd_reference(qkv, out, dout, lse2)
    got = emulate_bwd(qkv, out, dout, lse2)
    zero = (dout.view(1, 37, 2, 64) == 0).all(-1)
    assert int(zero.sum()) == 2 * 8
    assert bool((got[:, :, 0][zero] == 0).all()) and bool((bound[:, :, 0][zero] == 0).all())
    assert within(got, ref, bound)


def test_one_token_dv_is_dout():
    qkv, dout = random_case(3, 1, 2, 7)
    out, lse2 = isolated(qkv)
    got = emulate_bwd(qkv, out, dout, lse2)
    assert torch.equal(got[:, :, 2].reshape(3, 1, 128), dout.float())


DEFECTS = ["no_D", "D_half", "no_scale", "next_row_lse", "dV_from_P", "dK_from_dS"]


@pytest.mark.parametrize("defect", DEFECTS)
def test_bound_rejects_a_defective_kernel(defect):
    qkv, dout = random_case(2, 37, 2, 8)
    out, lse2 = isolated(qkv)
    ref, bound = attention_bwd_reference(qkv, out, dout, lse2)
    assert within(emulate_bwd(qkv, out, dout, lse2), ref, bound)
    assert not within(emulate_bwd(qkv, out, dout, lse2, defect=defect), ref, bound)


@pytest.mark.parametrize("N", [17, 197])
def test_bound_rejects_an_unmasked_padded_column_when_lse2_is_below_minus_128(N):
    """A padded key has a zero K row, so its score is 0 and P = exp2(-lse2): finite, and invisible after the zero V and K rows,
    while lse2 > -128; past that it is inf, 0.125 inf (dP - D) is inf, and inf times the zero K row makes dQ NaN."""
    qkv, dout = below_800_case(N, 9)
    out, lse2 = isolated(qkv)
    assert float(lse2.max()) < -128
    ref, bound = attention_bwd_reference(qkv, out, dout, lse2)
    assert within(emulate_bwd(qkv, out, dout, lse2), ref, bound)
    bad = emulate_bwd(qkv, out, dout, lse2, defect="no_column_mask")
    assert not within(bad, ref, bound) and bool(bad[:, :, 0].isnan().any())
    # with scores near 0 the same defect changes nothing: the bound cannot see it there
    qkv0, dout0 = random_case(1, N, 2, 10)
    out0, lse0 = isolated(qkv0)
    assert torch.equal(emulate_bwd(qkv0, out0, dout0, lse0, defect="no_column_mask"), emulate_bwd(qkv0, out0, dout0, lse0))
