"""The Swin V2 oracle (tests/swinv2_ref.py) against two independent implementations with the weights mapped across, at
real widths and head counts and depths (2, 2, 2, 2), so that stages 1-2 hold shifted blocks: HF transformers' Swinv2Model
for both towers (window_size and pretrained_window_sizes configured), and torchvision's SwinTransformer V2 for the base
tower (torchvision's CPB table divides by window - 1, which is the base tower's case)."""
import pytest
import torch
from torchvision.models.swin_transformer import PatchMergingV2, SwinTransformer, SwinTransformerBlockV2
from transformers import Swinv2Config, Swinv2Model

from swinv2_ref import ARCHS, backbone, randomize_

DEPTHS = (2, 2, 2, 2)


def _hf_state(sd, depths):
    out = {
        "embeddings.patch_embeddings.projection.weight": sd["patch_embed.proj.weight"],
        "embeddings.patch_embeddings.projection.bias": sd["patch_embed.proj.bias"],
        "embeddings.norm.weight": sd["patch_embed.norm.weight"], "embeddings.norm.bias": sd["patch_embed.norm.bias"],
        "layernorm.weight": sd["norm.weight"], "layernorm.bias": sd["norm.bias"],
    }
    for i, d in enumerate(depths):
        if i > 0:
            for k in ("reduction.weight", "norm.weight", "norm.bias"):
                out[f"encoder.layers.{i - 1}.downsample.{k}"] = sd[f"layers.{i}.downsample.{k}"]
        for j in range(d):
            s, h = f"layers.{i}.blocks.{j}.", f"encoder.layers.{i}.blocks.{j}."
            q, k, v = sd[s + "attn.qkv.weight"].chunk(3, dim=0)
            out.update({
                h + "attention.self.logit_scale": sd[s + "attn.logit_scale"],
                h + "attention.self.continuous_position_bias_mlp.0.weight": sd[s + "attn.cpb_mlp.0.weight"],
                h + "attention.self.continuous_position_bias_mlp.0.bias": sd[s + "attn.cpb_mlp.0.bias"],
                h + "attention.self.continuous_position_bias_mlp.2.weight": sd[s + "attn.cpb_mlp.2.weight"],
                h + "attention.self.query.weight": q, h + "attention.self.query.bias": sd[s + "attn.q_bias"],
                h + "attention.self.key.weight": k,
                h + "attention.self.value.weight": v, h + "attention.self.value.bias": sd[s + "attn.v_bias"],
                h + "attention.output.dense.weight": sd[s + "attn.proj.weight"],
                h + "attention.output.dense.bias": sd[s + "attn.proj.bias"],
                h + "layernorm_before.weight": sd[s + "norm1.weight"], h + "layernorm_before.bias": sd[s + "norm1.bias"],
                h + "intermediate.dense.weight": sd[s + "mlp.fc1.weight"], h + "intermediate.dense.bias": sd[s + "mlp.fc1.bias"],
                h + "output.dense.weight": sd[s + "mlp.fc2.weight"], h + "output.dense.bias": sd[s + "mlp.fc2.bias"],
                h + "layernorm_after.weight": sd[s + "norm2.weight"], h + "layernorm_after.bias": sd[s + "norm2.bias"],
            })
    return out


@pytest.mark.parametrize("name", sorted(ARCHS))
def test_oracle_matches_hf_swinv2(name):
    a = ARCHS[name]
    ours = randomize_(backbone(name, DEPTHS), seed=1).eval()
    cfg = Swinv2Config(image_size=256, patch_size=4, embed_dim=a["embed_dim"], depths=list(DEPTHS), num_heads=list(a["num_heads"]),
                       window_size=a["window_size"], pretrained_window_sizes=list(a["pretrained_window_sizes"]),
                       layer_norm_eps=1e-5, drop_path_rate=0.0)
    hf = Swinv2Model(cfg, add_pooling_layer=False).eval()
    missing, unexpected = hf.load_state_dict(_hf_state(ours.state_dict(), DEPTHS), strict=False)
    assert not unexpected
    assert all(k.endswith(("relative_coords_table", "relative_position_index")) for k in missing), missing
    # the shifted blocks are where the roll / mask / CPB conventions could disagree
    assert [b.shift for b in ours.layers[0].blocks] == [0, a["window_size"] // 2]
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        o = ours(x)
        r = hf(pixel_values=x).last_hidden_state.reshape(o.shape)
    assert o.shape == (2, 8, 8, 8 * a["embed_dim"])
    torch.testing.assert_close(o, r, rtol=2e-5, atol=2e-5)


def test_oracle_matches_torchvision_swin_v2_base():
    name = "swinv2_base_window8_256"
    a = ARCHS[name]
    ours = randomize_(backbone(name, DEPTHS), seed=2).eval()
    tv = SwinTransformer(patch_size=[4, 4], embed_dim=a["embed_dim"], depths=list(DEPTHS), num_heads=list(a["num_heads"]),
                         window_size=[8, 8], stochastic_depth_prob=0.0, block=SwinTransformerBlockV2,
                         downsample_layer=PatchMergingV2).eval()
    sd = ours.state_dict()
    m = {"features.0.0.weight": sd["patch_embed.proj.weight"], "features.0.0.bias": sd["patch_embed.proj.bias"],
         "features.0.2.weight": sd["patch_embed.norm.weight"], "features.0.2.bias": sd["patch_embed.norm.bias"],
         "norm.weight": sd["norm.weight"], "norm.bias": sd["norm.bias"]}
    for i, d in enumerate(DEPTHS):
        if i > 0:
            for k in ("reduction.weight", "norm.weight", "norm.bias"):
                m[f"features.{2 * i}.{k}"] = sd[f"layers.{i}.downsample.{k}"]
        for j in range(d):
            s, t = f"layers.{i}.blocks.{j}.", f"features.{2 * i + 1}.{j}."
            qb = sd[s + "attn.q_bias"]
            for k in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "attn.qkv.weight", "attn.proj.weight",
                      "attn.proj.bias", "attn.logit_scale", "attn.cpb_mlp.0.weight", "attn.cpb_mlp.0.bias", "attn.cpb_mlp.2.weight"):
                m[t + k] = sd[s + k]
            m[t + "attn.qkv.bias"] = torch.cat([qb, torch.zeros_like(qb), sd[s + "attn.v_bias"]])
            m[t + "mlp.0.weight"], m[t + "mlp.0.bias"] = sd[s + "mlp.fc1.weight"], sd[s + "mlp.fc1.bias"]
            m[t + "mlp.3.weight"], m[t + "mlp.3.bias"] = sd[s + "mlp.fc2.weight"], sd[s + "mlp.fc2.bias"]
    missing, unexpected = tv.load_state_dict(m, strict=False)
    assert not unexpected
    assert all(k.endswith(("relative_coords_table", "relative_position_index")) or k.startswith("head.") for k in missing), missing
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        torch.testing.assert_close(ours(x), tv.norm(tv.features(x)), rtol=2e-5, atol=2e-5)
