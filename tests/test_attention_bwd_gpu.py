"""Attention backward (vit.cu attention_bwd_kernel, N <= 208, one CTA of ceil(N/16) warps per (image, head)) against the fp64
reference of kernel_ref.attention_bwd_reference, elementwise within the bound derived there, with dqkv written into a
NaN-guarded buffer: every token count 1-208, the ViT-Ti/S/B/L training shapes, crafted softmaxes, and exact properties
(determinism, batch and head independence, read-only operands).

Isolated cases give the kernel out = bf16(O) and lse2 = fp32(lse2) of the fp64 forward, which is the kernel's whole
contract.  The chained case feeds it the wgmma forward's own out and lse2 (vdk_attention_fwd_lse, as training does) and
holds the result to the exact gradient, with the forward's bounds carried into the backward's."""
import math

import pytest
import torch

from kernel_ref import (Guarded, attention_bwd_reference, attention_reference, check_within, crafted_qkv, run_attention)
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu

MAX_N = 208


def run_bwd(lib, qkv, out, dout, lse2):
    """vdk_attention_bwd into a NaN-guarded dqkv [B*N, 3*H*64]; returns the Guarded buffer."""
    B, N, _, H, D = qkv.shape
    g = Guarded(B * N, 3 * H * D, 3 * H * D, torch.bfloat16, extra_rows=0, tail=4096)
    _lib.check(lib.vdk_attention_bwd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse2.data_ptr(), B, N, H, D, g.ptr(),
                                     _lib.stream_ptr()), "attention backward")
    torch.cuda.synchronize()
    return g


def isolated(qkv):
    """The backward's operands from the fp64 forward: out = bf16(O) [B, N, H*64], lse2 = fp32(lse2) [B, H, N]."""
    out, _, lse2, _ = attention_reference(qkv)
    return out.to(torch.bfloat16), lse2.float()


def describe(bad):
    """bad: bool [B, N, 3, H, 64] -> which operands, CTAs (image, head), warps and rows within a warp hold failures."""
    B, N, _, H, _ = bad.shape
    tok = bad.any(-1)                                   # [B, N, 3, H]
    idx = tok.nonzero()
    ops = {op: int(tok[:, :, i].sum()) for i, op in enumerate(("dq", "dk", "dv"))}
    ctas = tok.any(2).any(1).nonzero()[:6].tolist()
    return (f"wrong rows per operand {ops}; CTAs (b, h) {ctas}; first (b, token, operand, h) {idx[:6].tolist()}; "
            f"warps {sorted(set((idx[:, 1] // 16).tolist()))[:13]}, rows in warp {sorted(set((idx[:, 1] % 16).tolist()))}")


def check_bwd(lib, qkv, dout, out, lse2, name, stats=None, ref_operands=None):
    """Runs the backward on (qkv, out, dout, lse2) and checks dq, dk, dv against attention_bwd_reference of ref_operands
    (default: the kernel's own operands), and every guard element.  Returns (got [B, N, 3, H, 64] bf16, bound)."""
    B, N, _, H, D = qkv.shape
    g = run_bwd(lib, qkv, out, dout, lse2)
    got = g.view.view(B, N, 3, H, D)
    if ref_operands is None:
        ref, bound = attention_bwd_reference(qkv, out, dout, lse2)
    else:
        ref, bound = attention_bwd_reference(qkv, ref_operands[0], dout, ref_operands[1], *ref_operands[2:])
    for i, op in enumerate(("dQ", "dK", "dV")):
        def desc(bad, i=i):
            full = torch.zeros(B, N, 3, H, D, dtype=torch.bool, device=bad.device)
            full[:, :, i] = bad
            return describe(full)
        check_within(got[:, :, i], ref[:, :, i], bound[:, :, i], f"{name} {op}", desc, stats)
    assert not g.guard_errors(), "dqkv: " + g.guard_errors()
    return got, bound


def random_operands(B, N, H, seed, scale=1.5):
    torch.manual_seed(seed)
    qkv = (torch.randn(B, N, 3, H, 64, device="cuda") * scale).to(torch.bfloat16)
    dout = torch.randn(B, N, H * 64, device="cuda").to(torch.bfloat16)
    return qkv, dout


@pytest.mark.parametrize("warps", range(1, 14))
def test_every_token_count(lib, warps):
    """N = 16 (warps - 1) + 1 ... 16 warps: every padded-row count of the last warp's tile, at B = 2, H = 2."""
    stats = {}
    for N in range(16 * (warps - 1) + 1, 16 * warps + 1):
        qkv, dout = random_operands(2, N, 2, seed=N)
        out, lse2 = isolated(qkv)
        check_bwd(lib, qkv, dout, out, lse2, f"N={N}", stats)
    print(f"BOUND worst of warps={warps}: " + ", ".join(f"{op} {max(v for k, v in stats.items() if k.endswith(op)):.4f}"
                                                       for op in ("dQ", "dK", "dV")))


# (name, B, N, H): the training shapes at 224^2 / 16 (197 tokens), and smaller shapes with 1-3 heads
SHAPES = [
    ("vit_b16_train", 128, 197, 12),
    ("vit_l16", 32, 197, 16),
    ("vit_s16", 64, 197, 6),
    ("vit_ti16", 64, 197, 3),
    ("b2_n197_h3", 2, 197, 3),
    ("b1_n208_h2", 1, 208, 2),
    ("b3_n50_h2", 3, 50, 2),
    ("b2_n17_h1", 2, 17, 1),
]


@pytest.mark.parametrize("name,B,N,H", SHAPES, ids=[s[0] for s in SHAPES])
def test_shapes_isolated(lib, name, B, N, H):
    qkv, dout = random_operands(B, N, H, seed=B * 1000 + N + H)
    out, lse2 = isolated(qkv)
    check_bwd(lib, qkv, dout, out, lse2, name)


def test_vit_b16_chained_through_the_wgmma_forward(lib):
    """The forward kernel's out and lse2 go into the backward; the result is held to the exact gradient of softmax(q k^T/8) v,
    with the forward's out and lse2 bounds carried into D's and P's errors."""
    B, N, H = 128, 197, 12
    qkv, dout = random_operands(B, N, H, seed=3)
    fwd_out, fwd_lse = run_attention(lib, qkv)
    out64, out_b, lse64, lse_b = attention_reference(qkv)
    out_k, lse_k = fwd_out.view.view(B, N, H * 64), fwd_lse.view.view(B, H, N)
    check_within(out_k, out64, out_b, "chained: forward out", lambda bad: f"{int(bad.sum())} elements")
    check_within(lse_k, lse64, lse_b, "chained: forward lse2", lambda bad: f"{int(bad.sum())} rows")
    check_bwd(lib, qkv, dout, out_k, lse_k, "vit_b16_chained", ref_operands=(out64, lse64, out_b, lse_b))


def one_hot_alphas(N, ks):
    """alpha of a row whose single score alpha (others 0) gives P_peak = 1 / (1 + (N - 1) e^(-alpha/8)) ~ 1 - 2^-k."""
    return [float(torch.tensor(8 * math.log((N - 1) * (2.0 ** k - 1))).to(torch.bfloat16)) for k in ks]


def _beta(N, fn):
    return fn(torch.arange(N, device="cuda")).float()


# (name, N, alphas, beta(j), dense): exact scores alpha_i beta_j (crafted_qkv); dense adds random q / k components in disjoint
# dimensions, so dQ and dK are dense rows
CRAFTED = [
    # near-one-hot rows on key 5: P_peak ~ 1 - 2^-k, where dP - D cancels to ~2^-k of its terms
    ("one_hot_k2_to_24", 197, one_hot_alphas(197, [2, 6, 10, 16, 24]), lambda j: (j == 5).float(), True),
    ("one_hot_n64", 64, one_hot_alphas(64, [3, 8, 12, 20]), lambda j: (j == 5).float(), True),
    # every score 0: P = 1/N
    ("uniform", 197, [0.0], lambda j: torch.ones_like(j), True),
    # the maximum on token N - 1, the only real row of the last 16-row tile (113 = 7 * 16 + 1) or one of five (197)
    ("max_at_last_token_197", 197, [64.0, 16.0, 4.0, 0.0], lambda j: (j == 196).float(), True),
    ("max_at_last_token_113", 113, [64.0, 16.0, 4.0, 0.0], lambda j: (j == 112).float(), True),
    # every real score below -800 raw units: lse2 < -128, where an unmasked padded key would give exp2(-lse2) = inf
    ("below_minus_800_n17", 17, [1.0, 1.5], lambda j: -800.0 - 4.0 * (j % 8), True),
    ("below_minus_800_n197", 197, [1.0, 1.5], lambda j: -800.0 - 4.0 * (j % 8), True),
]


@pytest.mark.parametrize("name,N,alphas,beta,dense", CRAFTED, ids=[c[0] for c in CRAFTED])
def test_crafted_softmax(lib, name, N, alphas, beta, dense):
    B, H = 4, 2
    qkv = crafted_qkv(B, N, H, alphas, _beta(N, beta), seed=N, dense=dense)
    torch.manual_seed(N + 1)
    dout = torch.randn(B, N, H * 64, device="cuda").to(torch.bfloat16)
    out, lse2 = isolated(qkv)
    if name.startswith("below"):
        assert float(lse2.max()) < -128
    check_bwd(lib, qkv, dout, out, lse2, name)


def test_zero_dout_rows_give_exact_zero_dq(lib):
    """dO rows that are exactly 0 (every 5th token, in every warp and in the ragged last tile) have D = 0 and dP = 0, so the
    dS row and the dQ row are exact zeros, and the bound there is 0."""
    B, N, H = 2, 197, 3
    qkv, dout = random_operands(B, N, H, seed=11)
    dout.view(B, N, H, 64)[:, ::5] = 0
    dout.view(B, N, H, 64)[:, N - 1] = 0
    out, lse2 = isolated(qkv)
    got, bound = check_bwd(lib, qkv, dout, out, lse2, "zero dO rows")
    zero = (dout.view(B, N, H, 64) == 0).all(-1)
    assert int(zero.sum()) == B * H * (len(range(0, N, 5)) + 1)
    assert bool((got[:, :, 0][zero] == 0).all()) and bool((bound[:, :, 0][zero] == 0).all())


def test_one_token_dv_equals_dout(lib):
    """N = 1: P = 1 exactly after the bf16 rounding, so dV = dO bit for bit."""
    B, N, H = 8, 1, 4
    qkv, dout = random_operands(B, N, H, seed=12)
    out, lse2 = isolated(qkv)
    got, _ = check_bwd(lib, qkv, dout, out, lse2, "N=1")
    assert torch.equal(got[:, :, 2].reshape(B, N, H * 64).view(torch.int16), dout.view(torch.int16))


def bits(t):
    return t.contiguous().view(torch.int16)


def test_repeat_runs_are_bitwise_equal_and_operands_are_read_only(lib):
    B, N, H = 8, 197, 12
    qkv, dout = random_operands(B, N, H, seed=13)
    out, lse2 = isolated(qkv)
    before = [t.clone() for t in (qkv, out, dout, lse2)]
    a = run_bwd(lib, qkv, out, dout, lse2).view.clone()
    b = run_bwd(lib, qkv, out, dout, lse2).view.clone()
    assert torch.equal(bits(a), bits(b))
    for t, t0 in zip((qkv, out, dout, lse2), before):
        assert torch.equal(t.view(torch.int16 if t.element_size() == 2 else torch.int32),
                           t0.view(torch.int16 if t0.element_size() == 2 else torch.int32))


def test_one_image_alone_equals_its_slice_of_the_batch(lib):
    """At B = 128 (ViT-B training), images 0, 77 and 127 computed as B = 1 calls on contiguous slices are bit-identical to
    their slices of the batched result."""
    B, N, H = 128, 197, 12
    qkv, dout = random_operands(B, N, H, seed=14)
    out, lse2 = isolated(qkv)
    full = run_bwd(lib, qkv, out, dout, lse2).view.view(B, N, 3 * H * 64).clone()
    for b in (0, 77, 127):
        one = run_bwd(lib, qkv[b:b + 1].contiguous(), out[b:b + 1].contiguous(), dout[b:b + 1].contiguous(),
                      lse2[b:b + 1].contiguous()).view.view(1, N, 3 * H * 64)
        assert torch.equal(bits(one), bits(full[b:b + 1])), b


def test_other_heads_do_not_change_a_head(lib):
    """Changing every other head's q, k, v, dO, out and lse2 leaves head h's dq, dk, dv bitwise unchanged."""
    B, N, H, h = 2, 197, 12, 5
    qkv, dout = random_operands(B, N, H, seed=15)
    out, lse2 = isolated(qkv)
    a = run_bwd(lib, qkv, out, dout, lse2).view.view(B, N, 3, H, 64).clone()
    others = torch.arange(H, device="cuda") != h
    qkv2, dout2 = random_operands(B, N, H, seed=16)
    out2, lse22 = isolated(qkv2)
    qkv2[:, :, :, ~others] = qkv[:, :, :, ~others]
    dout2.view(B, N, H, 64)[:, :, ~others] = dout.view(B, N, H, 64)[:, :, ~others]
    out2.view(B, N, H, 64)[:, :, ~others] = out.view(B, N, H, 64)[:, :, ~others]
    lse22[:, ~others] = lse2[:, ~others]
    b = run_bwd(lib, qkv2, out2, dout2, lse22).view.view(B, N, 3, H, 64)
    assert torch.equal(bits(a[:, :, :, h]), bits(b[:, :, :, h]))
    assert not torch.equal(bits(a[:, :, :, others]), bits(b[:, :, :, others]))


def test_refusals(lib):
    """More than 208 tokens, a head dim other than 64 and a null operand are refused before any launch."""
    s = _lib.stream_ptr()
    qkv = torch.zeros(1, MAX_N + 1, 3, 1, 72, dtype=torch.bfloat16, device="cuda")
    o = torch.zeros(1, MAX_N + 1, 72, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(1, 1, MAX_N + 1, device="cuda")
    dq = torch.zeros_like(qkv)
    p = [t.data_ptr() for t in (qkv, o, o, lse)]
    assert lib.vdk_attention_bwd(*p, 1, MAX_N + 1, 1, 64, dq.data_ptr(), s) == _lib.VDK_ERR_INVALID
    assert "at most 208 tokens" in _lib.last_error()
    assert lib.vdk_attention_bwd(*p, 1, 16, 1, 72, dq.data_ptr(), s) == _lib.VDK_ERR_INVALID
    assert "head_dim must be 64" in _lib.last_error()
    for i in range(5):
        args = p + [dq.data_ptr()]
        args[i] = None
        assert lib.vdk_attention_bwd(*args[:4], 1, 16, 1, 64, args[4], s) == _lib.VDK_ERR_INVALID
        assert "null operand" in _lib.last_error()
    torch.cuda.synchronize()
    assert bool((dq == 0).all())
