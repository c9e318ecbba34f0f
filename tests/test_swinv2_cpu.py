"""CPU checks of the Swin V2 surface: the neck the reference's rank rule builds and its fold, the merge-weight permutation,
the CPB table and per-stage windows against the oracle, timm key sets and checkpoint loading, refusals, the reference
cbir.yaml with each listed Swin V2 backbone, the new ABI struct and the window attention's argument validation."""
import ctypes as C
import math
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from swinv2_ref import ARCHS, PatchMerging, WrapperOracle, attention_mask, backbone, coords_table, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.swin import (SWINV2_ARCHS, SwinV2NetC, SwinV2Wrapper, fold_nhwc_neck, merge_weight_khkw,
                                relative_coords_table, stage_windows)

DEPTHS = (2, 2, 2, 2)


@pytest.mark.parametrize("name", sorted(SWINV2_ARCHS))
def test_neck_is_the_cnn_branch_over_the_h_axis(name):
    c = ARCHS[name]["embed_dim"] * 8
    ref = WrapperOracle(name, 128, depths=(1, 1, 1, 1))
    ours = SwinV2Wrapper(name, 128, 256, pretrained=False, depths=(1, 1, 1, 1))
    for m in (ref, ours):
        bn2, lin = m.output_layer[0], m.output_layer[2]
        assert isinstance(bn2, nn.BatchNorm2d) and bn2.num_features == 8
        assert isinstance(m.output_layer[1], nn.Flatten)
        assert (lin.in_features, lin.out_features) == (64 * c, 128) and isinstance(m.output_layer[3], nn.BatchNorm1d)


@pytest.mark.parametrize("name", sorted(SWINV2_ARCHS))
def test_key_sets_match_the_oracle(name):
    ref = WrapperOracle(name, 64)
    ours = SwinV2Wrapper(name, 64, 256, pretrained=False)
    assert set(ours.state_dict()) == set(ref.state_dict())
    for k, v in ref.state_dict().items():
        assert ours.state_dict()[k].shape == v.shape, k
    ours.load_state_dict(ref.state_dict(), strict=True)


def test_folded_neck_reproduces_the_oracle_neck_in_fp64():
    name = "swinv2_base_window8_256"
    ref = randomize_(WrapperOracle(name, 96, depths=(1, 1, 1, 1)), seed=5).eval().double()
    c = ARCHS[name]["embed_dim"] * 8
    y = torch.randn(3, 8, 8, c, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    w, b = fold_nhwc_neck(ref.output_layer, 8, 8 * c, 96, "cpu")
    with torch.no_grad():
        torch.testing.assert_close(y.reshape(3, -1) @ w.t() + b, ref.output_layer(y), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("c", [128, 192, 768])
def test_merge_weight_as_a_2x2_stride_2_conv(c):
    pm = randomize_(PatchMerging(c), seed=c).double()
    x = torch.randn(2, 16, 8, c, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    w = merge_weight_khkw(pm.reduction.weight.detach())  # [2C, kh, kw, C]
    y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1)
    with torch.no_grad():
        torch.testing.assert_close(pm.norm(y), pm(x), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", sorted(SWINV2_ARCHS))
def test_windows_and_cpb_tables_match_the_oracle(name):
    m = backbone(name)
    wins = stage_windows(ARCHS[name]["window_size"])
    for i, stage in enumerate(m.layers):
        w, s = wins[i]
        assert [(b.window, b.shift) for b in stage.blocks[:2]] == [(w, 0), (w, s)]
        a = stage.blocks[0].attn
        torch.testing.assert_close(relative_coords_table(w, ARCHS[name]["pretrained_window_sizes"][i]),
                                   a.relative_coords_table.reshape(-1, 2), rtol=0, atol=0)
    if name.startswith("swinv2_large"):
        assert wins == [(16, 8), (16, 8), (16, 0), (8, 0)]
    else:
        assert wins == [(8, 4), (8, 4), (8, 4), (8, 0)]


def test_pack_clamps_logit_scales_and_builds_the_bias_tables():
    """The packed per-head scale is exp(min(logit_scale, ln 100)) and the packed bias table the oracle's
    16 sigmoid(cpb_mlp(table)), per block (large tower: stage 4 has its own window 8 and pretrained window 6)."""
    name = "swinv2_large_window12to16_192to256"
    ref = randomize_(backbone(name, DEPTHS), seed=4)
    with torch.no_grad():
        ref.layers[0].blocks[1].attn.logit_scale[0] = 7.0  # far above ln 100
    ours = SwinV2Wrapper(name, 64, 256, pretrained=False, depths=DEPTHS)
    ours.model.load_state_dict(ref.state_dict(), strict=True)
    net = ours._pack("cpu")
    by_ptr = {t.data_ptr(): t for t in ours._packed["keep"]}
    blocks = [b for s in ref.layers for b in s.blocks]
    for i, b in enumerate(blocks):
        a = b.attn
        scale = by_ptr[net.blocks[i].attn_scale]
        assert torch.equal(scale, torch.exp(torch.clamp(a.logit_scale.detach(), max=math.log(100.0))).reshape(-1))
        torch.testing.assert_close(by_ptr[net.blocks[i].attn_bias], a.bias_table().detach(), rtol=0, atol=0)
    assert by_ptr[net.blocks[1].attn_scale][0].item() == pytest.approx(100.0)
    assert list(net.window) == [16, 16, 16, 8] and list(net.shift) == [8, 8, 0, 0]


def test_mask_regions_are_timm_slices():
    m = attention_mask(16, 16, 8, 4)
    assert m.shape == (4, 64, 64) and not m[0].any()  # the top-left window is one region
    assert set(m.unique().tolist()) == {0.0, -100.0}
    # the bottom-right window holds four regions of 16 tokens: every token sees 16 unmasked keys
    assert ((m[3] == 0).sum(-1) == 16).all()


def test_timm_checkpoint_loads_as_pretrained(tmp_path, monkeypatch):
    name = "swinv2_base_window8_256"
    m = randomize_(backbone(name), seed=3)
    sd = dict(m.state_dict())
    sd["head.fc.weight"], sd["head.fc.bias"] = torch.zeros(1000, 1024), torch.zeros(1000)
    sd["layers.0.blocks.1.attn_mask"] = torch.zeros(64, 64, 64)
    sd["layers.0.blocks.0.attn.relative_position_index"] = torch.zeros(64, 64, dtype=torch.long)
    sd["layers.0.blocks.0.attn.relative_coords_table"] = torch.zeros(1, 15, 15, 2)
    torch.save(sd, tmp_path / f"{name}.pth")
    monkeypatch.setenv("VDK_PRETRAINED_DIR", str(tmp_path))
    ours = SwinV2Wrapper(name, 64, 256, pretrained=True)
    assert torch.equal(ours.model.layers[2].blocks[17].attn.cpb_mlp[2].weight, m.layers[2].blocks[17].attn.cpb_mlp[2].weight)


def test_refusals():
    m = SwinV2Wrapper("swinv2_base_window8_256", 64, 256, pretrained=False, depths=(1, 1, 1, 1))
    with pytest.raises(NotImplementedError):
        m.train()(torch.zeros(1, 3, 256, 256))
    with pytest.raises(ValueError, match="image_size must be 256"):
        SwinV2Wrapper("swinv2_base_window8_256", 64, 224, pretrained=False)
    for name in ("timm-swin_base_patch4_window7_224.ms_in22k_ft_in1k", "timm-swin_tiny_patch4_window7_224",
                 "timm-swinv2_tiny_window8_256", "timm-swinv2_cr_small_224"):
        with pytest.raises(ValueError, match="not built for H100"):
            BackboneFactory({name: {"pretrained": False, "image_size": 256, "feat_dim": 64}}).get_backbone()


@pytest.mark.parametrize("backbone_name,model_name", [("timm-swinv2_base_window8_256.ms_in1k", "swinv2_base_window8_256"),
                                                      ("timm-swinv2_large_window12to16_192to256.ms_in22k_ft_in1k",
                                                       "swinv2_large_window12to16_192to256")])
def test_reference_cbir_yaml_with_swinv2(backbone_name, model_name):
    from engine.vision_engine import check, yaml_load
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_configs")
    with open(os.path.join(root, "cbir.yaml")) as f:
        assert f"# {backbone_name}: # imgsz 256" in f.read()  # the file's own list of alternatives
    cfgs = yaml_load(os.path.join(root, "cbir.yaml"))
    head = next(iter(cfgs["model"]["head"].values()))
    cfgs["data"]["root"] = f"synthetic://cbir?ids={head['num_class']}&per_id=2&queries=4"
    old = next(iter(cfgs["model"]["backbone"].values()))
    cfgs["model"]["backbone"] = {backbone_name: dict(old, pretrained=False, image_size=256)}
    cfgs["model"]["image_size"] = 256  # the file's "# imgsz 256" for these entries
    check("cbir", cfgs)
    m = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    assert type(m) is SwinV2Wrapper and m.model_name == model_name and m.feat_dim == head["feat_dim"]


def test_swinv2_struct_size(lib):
    out = (C.c_size_t * 2)()
    assert lib.vdk_swinv2_struct_sizes(out, 2) == 1
    assert out[0] == C.sizeof(SwinV2NetC)


def test_window_attention_argument_validation(lib):
    s, b = (C.c_float * 4)(), (C.c_float * 4)()
    call = lambda H, W, heads, w, shift: lib.vdk_window_attention_fwd(256, 1, H, W, heads, w, shift, s, b, 256, None)  # noqa: E731
    for args, msg in (((56, 56, 4, 7, 0), "window must be 8 or 16"), ((60, 64, 4, 8, 0), "multiples of the window"),
                      ((64, 64, 4, 8, 3), "shift"), ((8, 8, 4, 8, 4), "shift"), ((32, 32, 4, 16, 4), "shift"),
                      ((64, 64, 0, 8, 0), "heads")):
        assert call(*args) == _lib.VDK_ERR_INVALID and msg in _lib.last_error(), (args, _lib.last_error())
    assert lib.vdk_postnorm_residual(256, 256, 4, 1544, s, b, 1e-5, None) == _lib.VDK_ERR_INVALID
