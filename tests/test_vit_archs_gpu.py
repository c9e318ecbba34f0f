"""The CBIR configs' DINO ViT-B/8, DINOv2 ViT-L/14, SigLIP So400m/14 and CLIP ViT-H/14 towers on the H100: the wgmma attention
forward at head dims 72 and 80 (csrc/attention_tc.cu) against an fp64 reference with an elementwise bound derived for any head dim
(attention_reference_hd below), and full-size embeddings of each tower against the fp32 oracle (oracle/vit_archs.py, pinned
against HF transformers in tests/test_oracle_vit_archs_cpu.py)."""
import math

import pytest
import torch

from kernel_ref import ATT_KVTILE, LOG2E, U32, attention_items, check_within, describe_attention, run_attention
from oracle.vit_archs import VIT_IMAGE_SIZE, ViTWrapperOracle, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory

pytestmark = pytest.mark.gpu


def attention_reference_hd(qkv):
    """fp64 softmax(q k^T / sqrt(D)) v of the bf16 inputs, D = qkv.shape[-1], with elementwise bounds of the kernel's output and
    log2-domain log-sum-exp.  Returns (out [B, N, H*D], out_bound, lse2 [B, H, N], lse2_bound), all fp64.

    kernel_ref.attention_reference's derivation (D = 64) with the two steps that depend on D:
      S_ij = q_i . k_j in fp32 on wgmma over kd = ceil(D / 16) k16 steps (D = 72 pads the last one with zeros, which add nothing):
             |dS_ij| <= (kd + 17) 2^-23 (|q_i| . |k_j|)
      x_ij = fma(S_ij, c, -m_ref), c = fp32(log2 e) / sqrtf(D) in fp32: c is off log2(e) / sqrt(D) by up to 3 2^-24 relative
             (log2 e, sqrtf and the division each round once), on c |S_ij - m|; with the fma's own 2^-24:
             |dx_ij| <= c (kd + 17) 2^-23 (|q||k|)_ij + 2 2^-23 c (|S_ij| + max_j |S_ij|)
    The P.V chain runs over keys and does not depend on D: e_acc = (4 J + 17 + J) 2^-23, e_l = (16 J + 2) 2^-24, as there."""
    B, N, _, H, D = qkv.shape
    J = -(-N // ATT_KVTILE)
    kd = -(-D // 16)
    scale = D ** -0.5
    c = float(torch.tensor(LOG2E, dtype=torch.float32)) / math.sqrt(D)
    e_acc = (4 * J + 17 + J) * U32
    e_l = (16 * J + 2) * 2.0 ** -24
    q, k, v = qkv.double().permute(2, 0, 3, 1, 4).unbind(0)  # [B, H, N, D]
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
        a = math.log(2.0) * (c * (kd + 17) * U32 * absqk + 2 * U32 * c * (S.abs() + S.abs().amax(-1, keepdim=True))) + 2.0 ** -22
        del absqk
        lse_nat = torch.logsumexp(S * scale, dim=-1)
        P = torch.exp(S * scale - lse_nat[..., None])
        del S
        absv = vf[sl].abs()
        R = P @ vf[sl]
        pa = (P * a).sum(-1, keepdim=True)
        of[sl] = R
        obf[sl] = (P * (2.0 ** -8 + a)) @ absv + e_acc * (P @ absv) + R.abs() * (pa + e_l + 2.0 ** -8 + 2.0 ** -22)
        lf[sl] = lse_nat * LOG2E
        lbf[sl] = LOG2E * (pa[..., 0] + e_l + (J - 1) * 2.0 ** -22) + 2.0 ** -22 * (lf[sl].abs() + math.log2(256.0 * N) + 1)
        del P, a
    return (out.transpose(1, 2).reshape(B, N, H * D), out_b.transpose(1, 2).reshape(B, N, H * D), lse, lse_b)


def check_attention(lib, qkv):
    """Runs vdk_attention_fwd_lse on qkv into NaN-guarded outputs and checks out and lse2 against attention_reference_hd
    elementwise, and every guard element.  Returns out [B, N, H*D]."""
    B, N, _, H, D = qkv.shape
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    out, lse = run_attention(lib, qkv, with_lse=True)
    ref, ref_b, lse_ref, lse_b = attention_reference_hd(qkv)
    got = out.view.view(B, N, H * D)
    check_within(got, ref, ref_b, f"attention out (D={D})",
                 lambda bad: describe_attention(bad.view(B, N, H, D).any(-1).permute(0, 2, 1), N, H, sm))
    assert not out.guard_errors(), "out: " + out.guard_errors()
    check_within(lse.view.view(B, H, N), lse_ref, lse_b, f"attention lse2 (D={D})", lambda bad: describe_attention(bad, N, H, sm))
    assert not lse.guard_errors(), "lse2: " + lse.guard_errors()
    return got


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def n_pairs(N):
    return (-(-N // 128) + 1) // 2


@pytest.mark.parametrize("D", [72, 80])
@pytest.mark.parametrize("N", [1, 256, 257, 785, 1370, 2049])
def test_attention_head_dim_matches_fp64(lib, D, N):
    """Random q, k, v (1.5 randn, bf16) at the towers' token counts (SigLIP 256, ViT-H 257, DINO 785, DINOv2 1370) and the edges
    (one token; 2049 = 33 key tiles, eight wraps of the K/V ring, a one-key last tile); out and lse2 within the bound, guards
    untouched."""
    B, H = (2, 3) if N > 1 else (3, 2)
    torch.manual_seed(N * 13 + D)
    qkv = (torch.randn(B, N, 3, H, D, device="cuda") * 1.5).to(torch.bfloat16)
    check_attention(lib, qkv)


@pytest.mark.parametrize("D", [72, 80])
def test_attention_head_dim_persistent_regime(lib, D):
    """More items than 3 x the SM count (785 tokens, 16 heads: four tile pairs per (image, head), the last holding one tile), so
    every CTA carries barrier phases, the Q double buffer and the K/V ring across items."""
    N, H = 785, 16
    B = -(-3 * sm_count() // (n_pairs(N) * H)) + 1
    items, grid = attention_items(B, N, H, sm_count())
    assert items > 3 * grid and grid == sm_count()
    torch.manual_seed(D)
    qkv = (torch.randn(B, N, 3, H, D, device="cuda") * 1.5).to(torch.bfloat16)
    check_attention(lib, qkv)


@pytest.mark.parametrize("D", [72, 80])
def test_attention_scores_from_the_remainder_columns_only(lib, D):
    """q and k are zero except in columns 64..D-1 (the 32-byte-swizzled remainder box): a dropped or mis-swizzled remainder makes
    every score 0 (out = the mean of v) or mixes rows, and fails the bound.  v is random in every column, so the remainder's
    P.V columns are checked too."""
    B, N, H = 2, 257, 4
    torch.manual_seed(3 * D)
    qkv = torch.randn(B, N, 3, H, D, device="cuda") * 1.5
    qkv[:, :, 0:2, :, :64] = 0.0
    qkv = qkv.to(torch.bfloat16)
    got = check_attention(lib, qkv)
    mean_v = qkv[:, :, 2].float().mean(1, keepdim=True).expand(B, N, H, D).reshape(B, N, H * D)
    assert (got.float() - mean_v).abs().max().item() > 0.1  # the scores do move the output away from the uniform average


def test_attention_head_dim_72_never_reads_the_next_head(lib):
    """D = 72: the remainder box spans columns 64-79, and 72-79 lie past the head.  Head 1's first 8 columns (q, k and v) hold 1e4,
    so a load that ran into the next head instead of being zero-filled by TMA would put ~1e8 into head 0's scores (q, k) or 1e4
    into its output (v).  Head 0 is random; head 1 (constant rows: uniform softmax) is checked too."""
    B, N, H, D = 2, 197, 2, 72
    torch.manual_seed(72)
    qkv = torch.randn(B, N, 3, H, D, device="cuda")
    qkv[:, :, :, 1] = 0.0
    qkv[:, :, :, 1, :8] = 1e4
    qkv = qkv.to(torch.bfloat16)
    got = check_attention(lib, qkv).view(B, N, H, D)
    assert got[:, :, 0].float().abs().max().item() < 100.0


def crafted_qkv(B, N, H, D, alphas, beta, seed):
    """q_i = alphas[i % len] e_{D-1}, k_j = beta[j] e_{D-1}: every raw score is the exact product alpha * beta, and it comes from
    the last column, which lies in the remainder box."""
    torch.manual_seed(seed)
    qkv = torch.zeros(B, N, 3, H, D, device="cuda")
    a = torch.tensor(alphas, device="cuda")[torch.arange(N, device="cuda") % len(alphas)]
    qkv[:, :, 0, :, D - 1] = a[None, :, None]
    qkv[:, :, 1, :, D - 1] = beta[None, :, None]
    qkv[:, :, 2] = torch.randn(B, N, H, D, device="cuda").to(torch.bfloat16).float()
    out = qkv.to(torch.bfloat16)
    assert torch.equal(out.float(), qkv)
    return out


# A rescale happens when a row's maximum exceeds the reference by more than 8 log2 units: 8 sqrt(D) / log2(e) raw score units,
# 47.05 at D = 72 and 49.6 at D = 80.  A step of 56 per key tile: alpha 1 grows 56 (rescale every tile), 0.8125 grows 45.5 (the
# stale reference stands, P up to 2^7.7 at D = 72).
CRAFTED = [
    ("grow_below_and_above_8", 577, [0.8125, 1.0, 0.0, -0.5], lambda t, j: 56.0 * t),
    ("jump_1000_in_last_tile", 197, [1.0, 0.03125, 0.0, -1.0], lambda t, j: torch.where(t == 3, 1000.0, 0.0)),
    ("max_in_first_tile", 257, [1.0, 0.5, 0.0, 0.0078125], lambda t, j: torch.where(t == 0, 0.0, -1000.0)),
]


@pytest.mark.parametrize("D", [72, 80])
@pytest.mark.parametrize("name,N,alphas,beta", CRAFTED, ids=[c[0] for c in CRAFTED])
def test_attention_head_dim_crafted_softmax(lib, D, name, N, alphas, beta):
    """Exact crafted scores that do and do not trigger the lazy rescale, at >= 3 items per CTA; out and lse2 within the bound."""
    H = 2
    B = max(1, -(-3 * sm_count() // (n_pairs(N) * H)))
    items, grid = attention_items(B, N, H, sm_count())
    assert items >= 3 * grid and grid == sm_count()
    j = torch.arange(N, device="cuda")
    qkv = crafted_qkv(B, N, H, D, alphas, beta(j // 64, j).float(), seed=N + D)
    check_attention(lib, qkv)


def test_attention_rejects_other_head_dims(lib):
    qkv = torch.zeros(1, 4, 3, 1, 96, dtype=torch.bfloat16, device="cuda")
    out = torch.empty(1, 4, 96, dtype=torch.bfloat16, device="cuda")
    assert lib.vdk_attention_fwd(qkv.data_ptr(), 1, 4, 1, 96, out.data_ptr(), _lib.stream_ptr()) == _lib.VDK_ERR_INVALID
    assert "64, 72 or 80" in _lib.last_error()


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


# (reference config tag, seed)
TOWERS = {
    "vit_base_patch8_224": ("dino", 21),
    "vit_large_patch14_dinov2": ("lvd142m", 22),
    "vit_so400m_patch14_siglip_224": ("webli", 23),
    "vit_huge_patch14_clip_224": ("laion2b_ft_in12k_in1k", 24),
}


@pytest.mark.parametrize("name", sorted(TOWERS))
def test_tower_embeddings_match_oracle(lib, name):
    """Full-size tower + the reference's Transformer neck (feat_dim 128, the CBIR config's) at its image size, 2 images, built
    through BackboneFactory from the config's `timm-<name>.<tag>` and loaded strict=True from the oracle's state_dict.  bf16
    activations vs the fp32 oracle: relative L2 <= 3e-2 and cosine >= 0.999 per embedding, as for the other full-size backbones.
    Training is refused."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    tag, seed = TOWERS[name]
    size = VIT_IMAGE_SIZE.get(name, 224)
    oracle = randomize_(ViTWrapperOracle(name, 128, size), seed=seed).eval()
    ours = BackboneFactory({f"timm-{name}.{tag}": {"pretrained": False, "image_size": size, "feat_dim": 128}}).get_backbone()
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().eval()
    torch.manual_seed(seed)
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        ref = torch.nn.functional.normalize(oracle(x))
    got = ours.embed(x.cuda(), l2_normalize=True).cpu()
    cos = (got * ref).sum(dim=1)
    print(f"{name}: rel {rel(got, ref):.4g} min cos {cos.min().item():.6f}")
    assert rel(got, ref) <= 3e-2, rel(got, ref)
    assert cos.min().item() >= 0.999
    with pytest.raises(NotImplementedError):
        ours.train()(x.cuda())
