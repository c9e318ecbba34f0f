"""The CBIR configs' DINO, DINOv2, SigLIP and CLIP ViT-H towers as restated in oracle/vit_archs.py, cross-checked against HF transformers'
independent implementations of the same architectures at real widths and head counts (toy depth and image size), and the
state_dict key sets of the four timm entries.  timm itself is not installed: these pin the architectures, not timm."""
import pytest
import torch

from oracle.vit_archs import ViTWrapperOracle, randomize_
from visiondk_b200.vit import VIT_ARCHS, ViTWrapper


def close(got, ref):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = (got - ref).abs().max().item()
    assert err <= 2e-5 * ref.abs().max().item() + 1e-5, err


def qkv_split(b):
    return b.attn.qkv.weight.data.chunk(3, dim=0), b.attn.qkv.bias.data.chunk(3, dim=0)


def load(hf, sd, allowed_missing=()):
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and not [k for k in missing if not any(a in k for a in allowed_missing)], (missing, unexpected)


def vit_model_sd(m, prefix=""):
    """oracle VisionTransformer -> HF ViTModel / Dinov2Model keys (the two share the embedding and attention names)."""
    sd = {prefix + "embeddings.cls_token": m.cls_token.data, prefix + "embeddings.position_embeddings": m.pos_embed.data,
          prefix + "embeddings.patch_embeddings.projection.weight": m.patch_embed.proj.weight.data,
          prefix + "embeddings.patch_embeddings.projection.bias": m.patch_embed.proj.bias.data,
          prefix + "layernorm.weight": m.norm.weight.data, prefix + "layernorm.bias": m.norm.bias.data}
    for i, b in enumerate(m.blocks):
        pre = f"{prefix}encoder.layer.{i}."
        (qw, kw, vw), (qb, kb, vb) = qkv_split(b)
        for name, w, bb in (("query", qw, qb), ("key", kw, kb), ("value", vw, vb)):
            sd[pre + f"attention.attention.{name}.weight"], sd[pre + f"attention.attention.{name}.bias"] = w, bb
        sd[pre + "attention.output.dense.weight"] = b.attn.proj.weight.data
        sd[pre + "attention.output.dense.bias"] = b.attn.proj.bias.data
    return sd


def test_dino_vit_b8_matches_hf_vit_model():
    """vit_base_patch8_224 (DINO): the plain ViT at patch 8, width 768, 12 heads of 64."""
    transformers = pytest.importorskip("transformers")
    patch, dim, _, heads = VIT_ARCHS["vit_base_patch8_224"]
    depth, size = 2, 32
    o = randomize_(ViTWrapperOracle("x", 32, size, patch=patch, dim=dim, depth=depth, heads=heads), seed=11).eval()
    m = o.model
    cfg = transformers.ViTConfig(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=heads, intermediate_size=4 * dim,
                                 image_size=size, patch_size=patch, num_channels=3, qkv_bias=True, layer_norm_eps=1e-6,
                                 hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    hf = transformers.ViTModel(cfg, add_pooling_layer=False).eval()
    sd = vit_model_sd(m)
    for i, b in enumerate(m.blocks):
        pre = f"encoder.layer.{i}."
        sd[pre + "layernorm_before.weight"], sd[pre + "layernorm_before.bias"] = b.norm1.weight.data, b.norm1.bias.data
        sd[pre + "layernorm_after.weight"], sd[pre + "layernorm_after.bias"] = b.norm2.weight.data, b.norm2.bias.data
        sd[pre + "intermediate.dense.weight"], sd[pre + "intermediate.dense.bias"] = b.mlp.fc1.weight.data, b.mlp.fc1.bias.data
        sd[pre + "output.dense.weight"], sd[pre + "output.dense.bias"] = b.mlp.fc2.weight.data, b.mlp.fc2.bias.data
    load(hf, sd, ("pooler",))
    torch.manual_seed(0)
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        close(m(x), hf(pixel_values=x).last_hidden_state)
    assert m(x).shape[1] == (size // patch) ** 2 + 1


def test_dinov2_vit_l14_matches_hf_dinov2_model_with_layer_scale():
    """vit_large_patch14_dinov2: LayerScale after attention and MLP (random gammas, not the 1e-5 init, so that they matter)."""
    transformers = pytest.importorskip("transformers")
    patch, dim, _, heads = VIT_ARCHS["vit_large_patch14_dinov2"]
    depth, size = 2, 56
    o = randomize_(ViTWrapperOracle("vit_large_patch14_dinov2", 32, size, patch=patch, dim=dim, depth=depth, heads=heads,
                                    layer_scale=True), seed=12).eval()
    m = o.model
    gammas = torch.cat([torch.cat([b.ls1.gamma.data, b.ls2.gamma.data]) for b in m.blocks])
    assert gammas.std().item() > 0.1  # random layer-scale values
    cfg = transformers.Dinov2Config(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=heads, mlp_ratio=4,
                                    image_size=size, patch_size=patch, num_channels=3, qkv_bias=True, layer_norm_eps=1e-6,
                                    hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                    layerscale_value=1e-5, use_swiglu_ffn=False)
    hf = transformers.Dinov2Model(cfg).eval()
    sd = vit_model_sd(m)
    for i, b in enumerate(m.blocks):
        pre = f"encoder.layer.{i}."
        sd[pre + "norm1.weight"], sd[pre + "norm1.bias"] = b.norm1.weight.data, b.norm1.bias.data
        sd[pre + "norm2.weight"], sd[pre + "norm2.bias"] = b.norm2.weight.data, b.norm2.bias.data
        sd[pre + "mlp.fc1.weight"], sd[pre + "mlp.fc1.bias"] = b.mlp.fc1.weight.data, b.mlp.fc1.bias.data
        sd[pre + "mlp.fc2.weight"], sd[pre + "mlp.fc2.bias"] = b.mlp.fc2.weight.data, b.mlp.fc2.bias.data
        sd[pre + "layer_scale1.lambda1"], sd[pre + "layer_scale2.lambda1"] = b.ls1.gamma.data, b.ls2.gamma.data
    load(hf, sd, ("mask_token",))
    torch.manual_seed(1)
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        close(m(x), hf(pixel_values=x).last_hidden_state)


def test_siglip_so400m_matches_hf_siglip_vision_model():
    """vit_so400m_patch14_siglip_224: no class token, width 1152, 16 heads of 72, MLP 4304, erf GELU, no attention-pool head."""
    transformers = pytest.importorskip("transformers")
    name = "vit_so400m_patch14_siglip_224"
    patch, dim, _, heads = VIT_ARCHS[name]
    depth, size = 2, 56
    o = randomize_(ViTWrapperOracle(name, 32, size, patch=patch, dim=dim, depth=depth, heads=heads, mlp_dim=4304, class_token=False),
                   seed=13).eval()
    m = o.model
    assert m.cls_token is None and m.blocks[0].mlp.fc1.out_features == 4304
    cfg = transformers.SiglipVisionConfig(hidden_size=dim, intermediate_size=4304, num_hidden_layers=depth, num_attention_heads=heads,
                                          num_channels=3, image_size=size, patch_size=patch, hidden_act="gelu", layer_norm_eps=1e-6,
                                          attention_dropout=0.0, vision_use_head=False)
    hf = transformers.SiglipVisionModel(cfg).eval()
    v = "vision_model."
    sd = {v + "embeddings.patch_embedding.weight": m.patch_embed.proj.weight.data,
          v + "embeddings.patch_embedding.bias": m.patch_embed.proj.bias.data,
          v + "embeddings.position_embedding.weight": m.pos_embed.data[0],
          v + "post_layernorm.weight": m.norm.weight.data, v + "post_layernorm.bias": m.norm.bias.data}
    for i, b in enumerate(m.blocks):
        pre = f"{v}encoder.layers.{i}."
        (qw, kw, vw), (qb, kb, vb) = qkv_split(b)
        for nm, w, bb in (("q_proj", qw, qb), ("k_proj", kw, kb), ("v_proj", vw, vb)):
            sd[pre + f"self_attn.{nm}.weight"], sd[pre + f"self_attn.{nm}.bias"] = w, bb
        sd[pre + "self_attn.out_proj.weight"], sd[pre + "self_attn.out_proj.bias"] = b.attn.proj.weight.data, b.attn.proj.bias.data
        sd[pre + "layer_norm1.weight"], sd[pre + "layer_norm1.bias"] = b.norm1.weight.data, b.norm1.bias.data
        sd[pre + "layer_norm2.weight"], sd[pre + "layer_norm2.bias"] = b.norm2.weight.data, b.norm2.bias.data
        sd[pre + "mlp.fc1.weight"], sd[pre + "mlp.fc1.bias"] = b.mlp.fc1.weight.data, b.mlp.fc1.bias.data
        sd[pre + "mlp.fc2.weight"], sd[pre + "mlp.fc2.bias"] = b.mlp.fc2.weight.data, b.mlp.fc2.bias.data
    load(hf, sd, ("position_ids",))
    torch.manual_seed(2)
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        got = m(x)
        close(got, hf(pixel_values=x).last_hidden_state)
    assert got.shape[1] == (size // patch) ** 2


def test_clip_vit_h14_matches_hf_clip_vision_model():
    """vit_huge_patch14_clip_224: the pre_norm CLIP tower at width 1280, 16 heads of 80."""
    transformers = pytest.importorskip("transformers")
    name = "vit_huge_patch14_clip_224"
    patch, dim, _, heads = VIT_ARCHS[name]
    depth, size = 2, 56
    o = randomize_(ViTWrapperOracle(name, 32, size, patch=patch, dim=dim, depth=depth, heads=heads), seed=14).eval()
    m = o.model
    assert m.patch_embed.proj.bias is None and isinstance(m.norm_pre, torch.nn.LayerNorm) and m.norm.eps == 1e-5
    cfg = transformers.CLIPVisionConfig(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=heads, intermediate_size=4 * dim,
                                        image_size=size, patch_size=patch, num_channels=3, layer_norm_eps=1e-5, hidden_act="gelu",
                                        attention_dropout=0.0, projection_dim=16)
    hf = transformers.CLIPVisionModel(cfg).eval()
    v = "vision_model."
    sd = {v + "embeddings.class_embedding": m.cls_token.data.reshape(-1),
          v + "embeddings.position_embedding.weight": m.pos_embed.data[0],
          v + "embeddings.patch_embedding.weight": m.patch_embed.proj.weight.data,
          v + "pre_layrnorm.weight": m.norm_pre.weight.data, v + "pre_layrnorm.bias": m.norm_pre.bias.data,
          v + "post_layernorm.weight": m.norm.weight.data, v + "post_layernorm.bias": m.norm.bias.data}
    for i, b in enumerate(m.blocks):
        pre = f"{v}encoder.layers.{i}."
        (qw, kw, vw), (qb, kb, vb) = qkv_split(b)
        for nm, w, bb in (("q_proj", qw, qb), ("k_proj", kw, kb), ("v_proj", vw, vb)):
            sd[pre + f"self_attn.{nm}.weight"], sd[pre + f"self_attn.{nm}.bias"] = w, bb
        sd[pre + "self_attn.out_proj.weight"], sd[pre + "self_attn.out_proj.bias"] = b.attn.proj.weight.data, b.attn.proj.bias.data
        sd[pre + "layer_norm1.weight"], sd[pre + "layer_norm1.bias"] = b.norm1.weight.data, b.norm1.bias.data
        sd[pre + "layer_norm2.weight"], sd[pre + "layer_norm2.bias"] = b.norm2.weight.data, b.norm2.bias.data
        sd[pre + "mlp.fc1.weight"], sd[pre + "mlp.fc1.bias"] = b.mlp.fc1.weight.data, b.mlp.fc1.bias.data
        sd[pre + "mlp.fc2.weight"], sd[pre + "mlp.fc2.bias"] = b.mlp.fc2.weight.data, b.mlp.fc2.bias.data
    load(hf, sd, ("position_ids",))
    torch.manual_seed(3)
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        close(m.forward_tokens(x), hf(pixel_values=x).last_hidden_state)


# timm name -> (image size, tokens fed to the neck, MLP width, has cls_token, has LayerScale)
NEW_ARCHS = {
    "vit_base_patch8_224": (224, 785, 3072, True, False),
    "vit_large_patch14_dinov2": (518, 1370, 4096, True, True),
    "vit_so400m_patch14_siglip_224": (224, 256, 4304, False, False),
    "vit_huge_patch14_clip_224": (224, 257, 5120, True, False),
}


@pytest.mark.parametrize("name", sorted(NEW_ARCHS))
def test_new_arch_state_dict_keys_match_the_oracle(name):
    """ViTWrapper's key set (and every shape) equals the oracle's for each new arch, so a checkpoint of the reference's TimmWrapper
    loads with strict=True: no cls_token for SigLIP, ls1.gamma / ls2.gamma for DINOv2, fc1 / fc2 at the MLP width."""
    from oracle import vit_archs
    from visiondk_b200.vit import VIT_IMAGE_SIZE
    size, tokens, mlp, cls, ls = NEW_ARCHS[name]
    assert VIT_IMAGE_SIZE.get(name, 224) == vit_archs.VIT_IMAGE_SIZE.get(name, 224) == size
    assert VIT_ARCHS[name] == vit_archs.VIT_ARCHS[name]
    _, dim, depth, _ = VIT_ARCHS[name]
    torch.manual_seed(0)
    ours = ViTWrapper(name, 128, size, pretrained=False)
    sd = {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    oracle = {k: tuple(v.shape) for k, v in ViTWrapperOracle(name, 128, size).state_dict().items()}
    assert sd == oracle
    assert ("model.cls_token" in sd) == cls
    assert sd["model.pos_embed"] == (1, tokens, dim)
    assert sd["output_layer.2.weight"] == (128, tokens * dim)
    assert sd["model.blocks.0.mlp.fc1.weight"] == (mlp, dim) and sd[f"model.blocks.{depth - 1}.mlp.fc2.weight"] == (dim, mlp)
    for i in (0, depth - 1):
        assert (f"model.blocks.{i}.ls1.gamma" in sd) == ls and (f"model.blocks.{i}.ls2.gamma" in sd) == ls
    assert not [k for k in sd if "attn_pool" in k or "fc_norm" in k or k.startswith("model.head")]


@pytest.mark.parametrize("name", sorted(NEW_ARCHS))
def test_new_arch_training_is_refused_before_any_kernel(name):
    """Training these towers is not built: the train-mode forward raises NotImplementedError naming the feature, on the CPU
    already (before the CUDA check that any kernel call would make)."""
    size = NEW_ARCHS[name][0]
    m = ViTWrapper(name, 128, size, pretrained=False).train()
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, size, size))
