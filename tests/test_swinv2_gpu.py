"""GPU checks of the Swin V2 path (csrc/swin.cu): the fused shifted-window attention and the post-norm residual elementwise
against fp64 references of the same bf16 inputs, within bounds derived from the kernels' roundings; both towers' full-size
embeddings against the fp32 oracle (tests/swinv2_ref.py) at the project's embedding tolerance (relative L2 <= 3e-2, cosine
>= 0.999 per row); one valuate run with the base tower.

The attention reference is the literal form: torch.roll, window_partition / window_reverse, timm's attn_mask and the
relative_position_index gather, all from tests/swinv2_ref.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from swinv2_ref import WrapperOracle, attention_mask, position_index, randomize_, window_partition, window_reverse
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.swin import SwinV2Wrapper

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # fp32 unit roundoff


def window_attention_reference(qkv, heads, w, shift, scale, bias):
    """fp64 result and elementwise bound, both [B, H, W, heads*32], for the bf16 qkv [B, H, W, 3, heads, 32].

    The kernel's roundings, per score s_j of a row: the fp32 tensor-core dot (32 products, |err| <= 32 u sum|q||k|), the fp32
    norms (sum of 32 squares, sqrt, max with 1e-12) and the products scale/|q| * 1/|k| * dot, together <= 128 u * scale of
    the cosine term (|cos| <= 1), then the bias and mask additions, 2 u |s_j| each:  ds = 128 u scale + 4 u max|s|.
    exp2((s_j - m) log2 e) adds 2^-21 (ex2.approx) and 2^-23 |s_j - m| relative, so p_j carries e_j = 2 ds + 2^-21 +
    2^-23 |s_j - m|.  P is rounded to bf16 (unit roundoff 2^-8) for P V, whose fp32 accumulation over N keys adds N u; the row
    sum of the unrounded p carries the weighted mean of e_j; the output rounds to bf16 (half an ulp, 2^-8 of the fp32 value)."""
    B, H, W = qkv.shape[:3]
    N, C = w * w, heads * 32
    x = qkv.double().reshape(B, H, W, 3 * C)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    xw = window_partition(x, w).view(-1, N, 3, heads, 32).permute(2, 0, 3, 1, 4)  # [3, B*nW, heads, N, 32]
    q, k, v = xw.unbind(0)
    qn = q / q.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    kn = k / k.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    sc = scale.double().cpu().view(1, heads, 1, 1).to(qkv.device)
    s = (qn @ kn.transpose(-2, -1)) * sc
    s = s + bias.double()[:, position_index(w).view(-1).to(qkv.device)].view(1, heads, N, N)
    if shift:
        mask = attention_mask(H, W, w, shift).double().to(qkv.device)
        s = (s.view(B, -1, heads, N, N) + mask.view(1, -1, 1, N, N)).view(-1, heads, N, N)
    m = s.amax(dim=-1, keepdim=True)
    p = torch.exp(s - m)
    den = p.sum(-1, keepdim=True)
    o = (p @ v) / den
    ds = 128 * U * sc + 4 * U * s.abs().amax(dim=-1, keepdim=True)
    e = 2 * ds + 2.0 ** -21 + 2.0 ** -23 * (s - m).abs()
    a = (p @ v.abs()) / den
    pre = (p * (e + 2.0 ** -8)) @ v.abs() / den + a * ((p * e).sum(-1, keepdim=True) / den + N * U)
    bound = pre + 2.0 ** -8 * (o.abs() + pre)

    def back(t):
        t = window_reverse(t.transpose(1, 2).reshape(-1, w, w, C), w, H, W)
        return torch.roll(t, shifts=(shift, shift), dims=(1, 2)) if shift else t

    return back(o), back(bound)


def run_window_attention(lib, qkv, heads, w, shift, scale, bias):
    B, H, W = qkv.shape[:3]
    out = torch.full((B, H, W, heads * 32), float("nan"), device="cuda", dtype=torch.bfloat16)
    _lib.check(lib.vdk_window_attention_fwd(qkv.data_ptr(), B, H, W, heads, w, shift, scale.data_ptr(), bias.data_ptr(),
                                            out.data_ptr(), _lib.stream_ptr()), "vdk_window_attention_fwd")
    torch.cuda.synchronize()
    return out


def random_inputs(B, H, W, heads, w, seed, logit_scale_hi=5.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(B, H, W, 3, heads, 32, device="cuda", generator=g) * 1.5).to(torch.bfloat16)
    ls = torch.rand(heads, device="cuda", generator=g) * (logit_scale_hi - 0.5) + 0.5
    scale = torch.clamp(ls, max=math.log(100.0)).exp().float().contiguous()
    bias = (16 * torch.sigmoid(torch.randn(heads, (2 * w - 1) ** 2, device="cuda", generator=g) * 2)).float().contiguous()
    return qkv, scale, bias


def check(lib, qkv, heads, w, shift, scale, bias, valid_heads=None):
    got = run_window_attention(lib, qkv, heads, w, shift, scale, bias).double()
    ref, bound = window_attention_reference(qkv, heads, w, shift, scale, bias)
    if valid_heads is not None:
        cols = torch.cat([torch.arange(h * 32, h * 32 + 32) for h in valid_heads]).cuda()
        got, ref, bound = got[..., cols], ref[..., cols], bound[..., cols]
    assert torch.isfinite(got).all(), "unwritten (NaN-guarded) or non-finite outputs"
    err = (got - ref).abs()
    assert (err <= bound).all(), f"max err {err.max().item():.3e}, worst ratio {(err / bound).max().item():.3f}"
    return err.max().item()


CASES = [  # (name, B, H, W, heads, window, shift)
    ("w8", 2, 32, 32, 4, 8, 0),
    ("w8_shift", 2, 32, 32, 4, 8, 4),
    ("w8_shift_rect", 1, 16, 40, 3, 8, 4),         # H != W: the rolled windows wrap around both edges at different periods
    ("w16", 1, 32, 32, 6, 16, 0),
    ("w16_shift", 2, 64, 64, 6, 16, 8),
    ("w8_single_window", 3, 8, 8, 32, 8, 0),        # base stage 4: one unshifted window
    ("w16_single_window", 2, 16, 16, 24, 16, 0),    # large stage 3: one 256-token window
    ("w8_many_items", 4, 64, 64, 4, 8, 4),          # base stage 1: 1024 CTAs, several per SM
]


@pytest.mark.parametrize("name,B,H,W,heads,w,shift", CASES, ids=[c[0] for c in CASES])
def test_window_attention_matches_fp64(lib, name, B, H, W, heads, w, shift):
    qkv, scale, bias = random_inputs(B, H, W, heads, w, seed=len(name) * 7 + w, logit_scale_hi=6.0)
    if name == "w8_many_items":
        assert B * (H // w) * (W // w) * heads > 3 * torch.cuda.get_device_properties(0).multi_processor_count
    if shift:  # every (query region, key region) pair of timm's three slices per axis occurs
        labels = attention_mask(H, W, w, shift)
        assert (labels != 0).any() and (labels == 0).any()
    check(lib, qkv, heads, w, shift, scale, bias)


@pytest.mark.parametrize("w", [8, 16])
def test_window_attention_zero_rows_and_clamped_scales(lib, w):
    """All-zero q and k rows (F.normalize's 1e-12 floor: their cosines are 0), and logit scales far above the ln 100 clamp."""
    H = 2 * w
    qkv, scale, bias = random_inputs(2, H, H, 4, w, seed=11 + w, logit_scale_hi=9.0)
    assert (scale == 100.0).any()
    qkv[0, 1:5, :, 0] = 0   # q rows
    qkv[1, :, 3:6, 1] = 0   # k rows
    qkv[0, 0, 0, :2] = 0    # both
    check(lib, qkv, 4, w, w // 2, scale, bias)


@pytest.mark.parametrize("w", [8, 16])
def test_window_attention_masked_keys_that_would_dominate(lib, w):
    """The bottom-right window of a shifted map holds four shift regions, labelled 4, 5, 7, 8; every q is u, and k is +u in
    the odd-labelled regions, -u in the even ones.  A query of region 4 or 8 then has cosine -1 with its own keys and +1 with
    the masked ones, which would win without the mask; with timm's -100 (not -inf) they still carry weight when
    scale - 100 > -scale (head 0: scale 100)."""
    H, heads, s = 2 * w, 2, w // 2
    qkv, scale, bias = random_inputs(1, H, H, heads, w, seed=5 + w)
    scale = torch.tensor([100.0, 30.0], device="cuda")
    u = torch.randn(32, device="cuda")
    reg = lambda r: 0 if r < H - w else (1 if r < H - s else 2)  # noqa: E731  timm's slices on the rolled axis
    for ry in range(H - w, H):
        for rx in range(H - w, H):
            y, x = (ry + s) % H, (rx + s) % H  # natural position of rolled (ry, rx)
            own = reg(ry) * 3 + reg(rx)
            qkv[0, y, x, 0, :] = u.to(torch.bfloat16)
            qkv[0, y, x, 1, :] = (u * (1.0 if own % 2 else -1.0)).to(torch.bfloat16)
    check(lib, qkv, heads, w, s, scale, bias)


def test_window_attention_poisoned_neighbour_head(lib):
    qkv, scale, bias = random_inputs(2, 16, 16, 4, 8, seed=3)
    qkv[..., 2, :] = float("nan")  # head 2's q, k and v
    check(lib, qkv, 4, 8, 4, scale, bias, valid_heads=[0, 1, 3])


@pytest.mark.parametrize("C", [128, 192, 256, 384, 768, 1024, 1536])
def test_postnorm_residual_matches_fp64(lib, C):
    """x <- x + LayerNorm(y) * g + b with |mean(y)| >> std(y).  Bound: the fp32 mean (C/32 + 6) u mean|y| scaled by rstd, the
    two-pass variance and rsqrt 64 u relative of the normalised value, and one bf16 ulp of the result."""
    g = torch.Generator(device="cuda").manual_seed(C)
    M = 1000
    y = (torch.randn(M, C, device="cuda", generator=g) * 2 + torch.randn(M, 1, device="cuda", generator=g) * 60).to(torch.bfloat16)
    x = (torch.randn(M, C, device="cuda", generator=g) * 3).to(torch.bfloat16)
    w = (1 + 0.3 * torch.randn(C, device="cuda", generator=g)).float()
    b = (0.5 * torch.randn(C, device="cuda", generator=g)).float()
    yd = y.double()
    mean = yd.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(yd.var(-1, unbiased=False, keepdim=True) + 1e-5)
    yhat = (yd - mean) * rstd
    ref = x.double() + yhat * w.double() + b.double()
    bound = w.double().abs() * ((C / 32 + 6) * U * yd.abs().mean(-1, keepdim=True) * rstd + 64 * U * yhat.abs()) \
        + 4 * U * b.double().abs() + 2.0 ** -8 * ref.abs()
    got = x.clone()
    _lib.check(lib.vdk_postnorm_residual(got.data_ptr(), y.data_ptr(), M, C, w.data_ptr(), b.data_ptr(), 1e-5, _lib.stream_ptr()),
               "vdk_postnorm_residual")
    torch.cuda.synchronize()
    err = (got.double() - ref).abs()
    assert (err <= bound).all(), f"max err {err.max().item():.3e}, worst ratio {(err / bound).max().item():.3f}"


def embed_and_compare(name, feat, batch, depths=None, seed=0):
    oracle = randomize_(WrapperOracle(name, feat, depths=depths), seed=seed).eval()
    ours = SwinV2Wrapper(name, feat, 256, pretrained=False, depths=depths)
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().eval()
    torch.manual_seed(seed + 1)
    x = torch.randn(batch, 3, 256, 256)
    with torch.no_grad():
        ref = oracle(x)
    got = ours(x.cuda()).cpu()
    rel = ((got - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    cos = F.cosine_similarity(got, ref).min().item()
    print(f"{name}: rel L2 err {rel:.4f}, min cosine {cos:.6f}")
    assert rel <= 3e-2 and cos >= 0.999, f"{name}: rel L2 err {rel:.4f}, min cosine {cos:.5f}"
    got_n = ours.embed(x.cuda(), l2_normalize=True).cpu()
    assert torch.allclose(got_n.norm(dim=1), torch.ones(batch), atol=1e-5)
    assert F.cosine_similarity(got_n, F.normalize(ref)).min().item() >= 0.999
    return ours


@pytest.mark.parametrize("name", ["swinv2_base_window8_256", "swinv2_large_window12to16_192to256"])
def test_full_size_embeddings_match_oracle(lib, name):
    """Both towers at full depth, every parameter randomised (logit scales, CPB weights, the post-norms that timm's init
    zeroes; see randomize_ for why the scales stay below the clamp here)."""
    embed_and_compare(name, 512, 2, seed=3)


def test_refits_after_weight_update_and_refuses_training(lib):
    ours = embed_and_compare("swinv2_base_window8_256", 64, 2, depths=(2, 2, 2, 2), seed=9)
    x = torch.randn(2, 3, 256, 256, device="cuda")
    a = ours.embed(x)
    with torch.no_grad():
        ours.model.layers[1].blocks[1].attn.cpb_mlp[2].weight.mul_(3.0)  # a new weight version: the bias tables are rebuilt
    assert not torch.equal(a, ours.embed(x))
    ours.train()
    with pytest.raises(NotImplementedError):
        ours(x)


def test_valuate_with_a_swinv2_backbone(lib):
    from engine.cbir.evaluation import valuate
    model = BackboneFactory({"timm-swinv2_base_window8_256.ms_in1k": {"pretrained": False, "image_size": 256, "feat_dim": 64}}).get_backbone()
    randomize_(model, seed=2)
    model = model.cuda().eval()
    cfg = {"root": "synthetic://cbir?ids=8&per_id=4&queries=4", "nw": 0,
           "val": {"bs": 8, "augment": [], "metrics": {"metrics": ["mrr", "recall"], "cutoffs": [1, 5]}}}
    got = valuate(model, cfg, "cuda", image_size=256)
    assert got and all(0.0 <= v <= 1.0 for v in got.values())
