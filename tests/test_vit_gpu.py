"""GPU parity of the ViT extract path (csrc/vit.cu) against the oracle (oracle/vit.py: timm's VisionTransformer restated and
pinned against HF ViTModel on CPU).  bf16 activations vs the fp32 oracle: tolerances stated per test."""
import pytest
import torch

from oracle.vit import ViTWrapperOracle, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.vit import ViTWrapper

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize("B,N,H", [(2, 197, 12), (3, 64, 3), (1, 577, 4), (2, 50, 2), (2, 1, 1)])
def test_attention_forward_matches_torch(lib, B, N, H):
    """softmax(q k^T / 8) v per (image, head) on the qkv Linear's output layout [B, N, 3, H, 64]; reference in fp32 on the same
    bf16-rounded inputs.  P is rounded to bf16 before P.V: |err| <= 2^-8 relative to the largest |v| of the row."""
    torch.manual_seed(N * 7 + H)
    qkv = (torch.randn(B, N, 3, H, 64, device="cuda") * 1.5).to(torch.bfloat16)
    out = torch.full((B, N, H * 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.vdk_attention_fwd(qkv.data_ptr(), B, N, H, 64, out.data_ptr(), _lib.stream_ptr()), "attention")
    q, k, v = qkv.float().permute(2, 0, 3, 1, 4).unbind(0)  # [B, H, N, 64]
    ref = torch.softmax((q @ k.transpose(-2, -1)) * 0.125, dim=-1) @ v
    ref = ref.transpose(1, 2).reshape(B, N, H * 64)
    assert torch.isfinite(out.float()).all()
    assert (out.float() - ref).abs().max().item() <= 2e-2 * v.abs().max().item()
    assert rel(out, ref) <= 1e-2


def build(seed, **kw):
    oracle = randomize_(ViTWrapperOracle("x", **kw), seed=seed).eval()
    ours = ViTWrapper("x", kw["feat_dim"], kw["image_size"], pretrained=False, patch=kw["patch"], dim=kw["dim"], depth=kw["depth"],
                      heads=kw["heads"], pre_norm=kw.get("pre_norm", False))
    ours.load_state_dict(oracle.state_dict(), strict=True)
    return oracle, ours.cuda().eval()


@pytest.mark.parametrize("cfg", [dict(feat_dim=64, image_size=64, patch=16, dim=128, depth=2, heads=2),
                                 dict(feat_dim=128, image_size=112, patch=14, dim=192, depth=3, heads=3),
                                 # timm's pre_norm CLIP tower: norm_pre, bias-free patch embedding, eps 1e-5 (config 5 family)
                                 dict(feat_dim=64, image_size=56, patch=14, dim=128, depth=2, heads=2, pre_norm=True)])
def test_vit_toy_embeddings_match_oracle(lib, cfg):
    oracle, ours = build(3, **cfg)
    torch.manual_seed(1)
    x = torch.randn(5, 3, cfg["image_size"], cfg["image_size"])
    with torch.no_grad():
        ref = oracle(x)
    got = ours(x.cuda()).cpu()
    assert got.shape == ref.shape
    assert rel(got, ref) <= 2e-2, rel(got, ref)
    # the fused F.normalize (face_model.py:139)
    gn = ours.embed(x.cuda(), l2_normalize=True).cpu()
    assert rel(gn, torch.nn.functional.normalize(ref)) <= 2e-2
    assert (gn.norm(dim=1) - 1).abs().max().item() <= 1e-5


def test_vit_base_patch16_224_embeddings_match_oracle(lib):
    """BASELINE config 3/5 family at full size: ViT-B/16 224^2, 197 tokens, neck Linear(151296, 512)."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oracle = randomize_(ViTWrapperOracle("vit_base_patch16_224", 512, 224), seed=5).eval()
    ours = BackboneFactory({"timm-vit_base_patch16_224": {"pretrained": False, "image_size": 224, "feat_dim": 512}}).get_backbone()
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().eval()
    torch.manual_seed(2)
    x = torch.randn(3, 3, 224, 224)
    with torch.no_grad():
        ref = torch.nn.functional.normalize(oracle(x))
    got = ours.embed(x.cuda(), l2_normalize=True).cpu()
    cos = (got * ref).sum(dim=1)
    assert rel(got, ref) <= 3e-2, rel(got, ref)
    assert cos.min().item() >= 0.999


def test_vit_large_patch14_clip_336_embeddings_match_oracle(lib):
    """BASELINE config 5 at full size: timm's vit_large_patch14_clip_336 (CLIP ViT-L/14 tower: pre_norm, 577 tokens, width 1024,
    24 blocks, 16 heads) + the reference's Transformer neck Linear(590 848 -> 512), against the fp32 oracle (cross-checked vs HF
    CLIPVisionModel in tests/test_oracle_vit_cpu.py).  Tolerance as for the other full-size backbones: bf16 activations through
    24 blocks -> relative L2 <= 3e-2, cosine >= 0.999 per embedding.  Training of this variant is refused, not faked."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    name = "vit_large_patch14_clip_336"
    oracle = randomize_(ViTWrapperOracle(name, 512, 336), seed=7).eval()
    ours = BackboneFactory({f"timm-{name}.openai_ft_in12k_in1k": {"pretrained": False, "image_size": 336, "feat_dim": 512}}).get_backbone()
    assert ours.model.pre_norm and ours.model.patch_embed.proj.bias is None
    ours.load_state_dict(oracle.state_dict(), strict=True)  # the key set of timm's pre_norm tower (norm_pre.*, no patch bias)
    ours = ours.cuda().eval()
    torch.manual_seed(4)
    x = torch.randn(2, 3, 336, 336)
    with torch.no_grad():
        ref = torch.nn.functional.normalize(oracle(x))
    got = ours.embed(x.cuda(), l2_normalize=True).cpu()
    cos = (got * ref).sum(dim=1)
    assert rel(got, ref) <= 3e-2, rel(got, ref)
    assert cos.min().item() >= 0.999
    with pytest.raises(NotImplementedError):
        ours.train()(x.cuda())


@pytest.mark.parametrize("B,N,H", [(2, 197, 3), (1, 208, 2), (3, 50, 2), (2, 17, 1)])
def test_attention_backward_matches_torch_autograd(lib, B, N, H):
    """dqkv of softmax(q k^T / 8) v against fp32 autograd on the same bf16-rounded inputs (P and dS are rounded to bf16 inside
    the kernel: rel L2 <= 2e-2 per operand)."""
    import ctypes as C
    torch.manual_seed(N + H)
    qkv = (torch.randn(B, N, 3, H, 64, device="cuda")).to(torch.bfloat16)
    dout = torch.randn(B, N, H * 64, device="cuda").to(torch.bfloat16)
    out = torch.empty((B, N, H * 64), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((B, H, N), dtype=torch.float32, device="cuda")
    dqkv = torch.full_like(qkv, float("nan"))
    s = _lib.stream_ptr()
    _lib.check(lib.vdk_attention_fwd_lse(qkv.data_ptr(), B, N, H, 64, out.data_ptr(), lse.data_ptr(), s), "attention fwd+lse")
    _lib.check(lib.vdk_attention_bwd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), B, N, H, 64, dqkv.data_ptr(), s),
               "attention bwd")
    x = qkv.float().requires_grad_(True)
    q, k, v = x.permute(2, 0, 3, 1, 4).unbind(0)
    ref = (torch.softmax((q @ k.transpose(-2, -1)) * 0.125, dim=-1) @ v).transpose(1, 2).reshape(B, N, H * 64)
    ref.backward(dout.float())
    # the saved log-sum-exp (log2 domain) equals torch's logsumexp of the scaled scores
    lse_ref = torch.logsumexp((q @ k.transpose(-2, -1)) * 0.125, dim=-1) * 1.4426950408889634
    assert (lse - lse_ref.detach()).abs().max().item() <= 2e-2
    assert torch.isfinite(dqkv.float()).all()
    for i, name in enumerate("qkv"):
        assert rel(dqkv[:, :, i], x.grad[:, :, i]) <= 2e-2, (name, rel(dqkv[:, :, i], x.grad[:, :, i]))


def grads_match(ours, oracle, rel_tol, cos_tol, invariant, vec_rel_tol=None, vec_cos_tol=None):
    import torch.nn.functional as F
    ref = dict(oracle.named_parameters())
    bad, worst = [], []
    for n, p in ours.named_parameters():
        gr, g = ref[n].grad, p.grad.detach().cpu()
        assert torch.isfinite(g).all(), n
        if n in invariant or gr.norm() < 1e-7 * (1 + gr.numel() ** 0.5):
            continue
        r = rel(g, gr)
        c = F.cosine_similarity(g.flatten(), gr.flatten(), dim=0).item()
        worst.append((r, c, n))
        # 1-D parameters (biases, norm scales) are sums over every token of signed terms: cancellation amplifies the bf16 noise
        rt, ct = (rel_tol, cos_tol) if g.dim() >= 2 else (vec_rel_tol or rel_tol, vec_cos_tol or cos_tol)
        if not (r <= rt and c >= ct):
            bad.append(f"{n}: rel {r:.4f} cos {c:.5f}")
    for r, c, n in sorted(worst, reverse=True)[:8]:
        print(f"  rel {r:.4f} cos {c:.5f} {n}")
    assert not bad, "\n".join(bad[:20])


# exact gradient 0: a constant shift in front of a batch-statistics BatchNorm1d is normalised away (the Linear bias, and the neck
# LayerNorm's bias, which only shifts the Linear output by a per-feature constant)
VIT_INVARIANT = {"output_layer.2.bias", "output_layer.0.bias"}


def test_vit_toy_training_gradients_match_oracle_autograd(lib):
    cfg = dict(feat_dim=64, image_size=64, patch=16, dim=128, depth=2, heads=2)
    oracle, ours = build(7, **cfg)
    oracle.train()
    ours.train()
    torch.manual_seed(1)
    x = torch.randn(6, 3, 64, 64)
    wout = torch.randn(6, 64)
    out_ref = oracle(x)
    (out_ref * wout).sum().backward()
    out = ours(x.cuda())
    (out * wout.cuda()).sum().backward()
    assert rel(out.detach().cpu(), out_ref.detach()) <= 3e-2
    grads_match(ours, oracle, 6e-2, 0.995, VIT_INVARIANT)
    bn_o, bn = oracle.output_layer[3], ours.output_layer[3]
    assert rel(bn.running_mean.cpu(), bn_o.running_mean) <= 2e-2 and rel(bn.running_var.cpu(), bn_o.running_var) <= 2e-2
    assert int(bn.num_batches_tracked) == 1


def test_vit_base_patch16_224_training_gradients_match_oracle(lib):
    """BASELINE config 3 backbone at full size (ViT-B/16 224^2, 12 blocks, 197 tokens), batch 8 (BatchNorm1d on batch statistics
    is ill-conditioned for 3 samples): every parameter gradient vs fp32 autograd of the oracle (bf16 activations: weight
    matrices rel <= 0.15, cos >= 0.99; 1-D parameters, model.norm.bias the worst of them, rel <= 0.25, cos >= 0.97)."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oracle = randomize_(ViTWrapperOracle("vit_base_patch16_224", 512, 224), seed=5).train()
    ours = ViTWrapper("vit_base_patch16_224", 512, 224, pretrained=False)
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().train()
    torch.manual_seed(2)
    x = torch.randn(8, 3, 224, 224)
    wout = torch.randn(8, 512)
    (oracle(x) * wout).sum().backward()
    (ours(x.cuda()) * wout.cuda()).sum().backward()
    grads_match(ours, oracle, 0.15, 0.99, VIT_INVARIANT, vec_rel_tol=0.25, vec_cos_tol=0.97)


def test_vit_train_step_with_circleloss_and_fused_optimizer(lib):
    """One config-3 style step: ViT forward -> CircleLoss + CE -> backward -> clip + SGD + EMA; loss decreases over 8 steps."""
    from visiondk_b200.train import FaceTrainingModel, FaceTrainer
    cfg = {"backbone": {"timm-vit_toy": {"pretrained": False, "image_size": 64, "feat_dim": 64, "patch": 16, "dim": 128, "depth": 2,
                                         "heads": 2}},
           "head": {"circleloss": {"feat_dim": 64, "num_class": 10, "margin": 0.25, "gamma": 64}}}
    torch.manual_seed(0)
    model = FaceTrainingModel(cfg).cuda()
    trainer = FaceTrainer(model, lr0=0.02, momentum=0.9, weight_decay=5e-4, label_smooth=0.0, layer_wise=True, warm_steps=0,
                          total_steps=100, use_ema=True)
    x = torch.randn(16, 3, 64, 64, device="cuda")
    y = torch.randint(0, 10, (16,), device="cuda")
    losses = [float(trainer.step(x, y)) for _ in range(8)]
    assert all(l == l for l in losses) and losses[-1] < losses[0], losses


def test_vit_backward_in_unit_ranges_equals_single_call(lib):
    cfg = dict(feat_dim=64, image_size=64, patch=16, dim=128, depth=3, heads=2)
    _, ours = build(9, **cfg)
    ours.train()
    torch.manual_seed(3)
    x = torch.randn(6, 3, 64, 64, device="cuda")
    wout = torch.randn(6, 64, device="cuda")
    for p in ours.parameters():
        p.grad = torch.zeros_like(p)
    (ours(x) * wout).sum().backward()
    one_call = {n: p.grad.clone() for n, p in ours.named_parameters()}
    for p in ours.parameters():
        p.grad.zero_()
    seen = []
    ours.grad_section_hook = lambda names: seen.extend(names)
    (ours(x) * wout).sum().backward()
    ours.grad_section_hook = None
    assert sorted(seen) == sorted(n for n, _ in ours.named_parameters())
    for n, p in ours.named_parameters():
        a, b = p.grad, one_call[n]
        assert (a - b).abs().max().item() <= 1e-4 * (b.abs().max().item() + 1e-6) + 1e-6, n

