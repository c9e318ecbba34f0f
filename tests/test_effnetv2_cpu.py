"""CPU-side checks of the EfficientNetV2 extract path: the wrapper's parameter tree equals the oracle's (timm's keys), timm
checkpoints load strictly with their classifier dropped, the refusals, the factory dispatch, and the ctypes mirrors of
vdk_conv_ex_desc / vdk_effnetv2_net."""
import ctypes as C

import pytest
import torch

from effnetv2_ref import WrapperOracle
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.efficientnet import EFFNETV2_ARCHS, ConvExDesc, EffNetV2NetC, EfficientNetV2Wrapper, pack_conv_ex


@pytest.mark.parametrize("name", sorted(EFFNETV2_ARCHS))
def test_state_dict_matches_oracle(name):
    ours = EfficientNetV2Wrapper(name, 256, 224, pretrained=False).state_dict()
    ref = WrapperOracle(name, 256, 224).state_dict()
    assert list(ours) == list(ref)
    for k in ref:
        assert ours[k].shape == ref[k].shape, k


def test_block_counts_and_se_widths():
    m = EfficientNetV2Wrapper("tf_efficientnetv2_l", 64, 224, pretrained=False).model
    blocks = [b for s in m.blocks for b in s]
    assert len(blocks) == 79 and sum(b.kind == "ir" for b in blocks) == 61
    assert m.blocks[3][0].se.conv_reduce.out_channels == 24 and m.blocks[6][1].se.conv_reduce.out_channels == 160
    assert m.blocks[6][1].conv_dw.out_channels == 3840


def test_checkpoint_with_classifier_loads_strictly(tmp_path, monkeypatch):
    src = EfficientNetV2Wrapper("tf_efficientnetv2_s", 64, 64, pretrained=False, depths=(1, 1, 1, 1, 1, 1))
    sd = dict(src.model.state_dict())
    sd["classifier.weight"] = torch.zeros(1000, 1280)
    sd["classifier.bias"] = torch.zeros(1000)
    torch.save(sd, tmp_path / "tf_efficientnetv2_s.pth")
    monkeypatch.setenv("VDK_PRETRAINED_DIR", str(tmp_path))
    got = EfficientNetV2Wrapper("tf_efficientnetv2_s", 64, 64, pretrained=True, depths=(1, 1, 1, 1, 1, 1))
    for k, v in src.model.state_dict().items():
        assert torch.equal(got.model.state_dict()[k], v), k


def test_refusals():
    with pytest.raises(ValueError, match="not built for H100"):
        EfficientNetV2Wrapper("tf_efficientnetv2_xl", 64, 224, pretrained=False)
    with pytest.raises(ValueError, match="multiple of 32"):
        EfficientNetV2Wrapper("tf_efficientnetv2_s", 64, 200, pretrained=False)
    m = EfficientNetV2Wrapper("tf_efficientnetv2_s", 64, 64, pretrained=False, depths=(1,) * 6).train()
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 64, 64))
    for name in ("timm-efficientnetv2_rw_s", "timm-tf_efficientnet_b0"):
        with pytest.raises(ValueError, match="not built for H100"):
            BackboneFactory({name: {"pretrained": False, "image_size": 224, "feat_dim": 64}}).get_backbone()


def test_factory_builds_the_wrapper():
    m = BackboneFactory({"timm-tf_efficientnetv2_l.in21k_ft_in1k": {"pretrained": False, "image_size": 224, "feat_dim": 512}}).get_backbone()
    assert isinstance(m, EfficientNetV2Wrapper) and m.model_name == "tf_efficientnetv2_l"
    assert m.output_layer[2].in_features == 1280 * 7 * 7


def test_pack_conv_ex_pads_channels_to_64():
    w = torch.randn(16, 24, 3, 3)
    p = pack_conv_ex(w)
    assert p.shape == (16, 3, 3, 64) and torch.equal(p[..., :24], w.permute(0, 2, 3, 1)) and not p[..., 24:].any()
    assert pack_conv_ex(torch.randn(16, 24, 1, 1)).shape == (16, 24)


def test_effnetv2_struct_mirrors(lib):
    out = (C.c_size_t * 4)()
    assert lib.vdk_effnetv2_struct_sizes(out, 4) == 2
    assert (C.sizeof(ConvExDesc), C.sizeof(EffNetV2NetC)) == (out[0], out[1])


def test_effnetv2_argument_validation_needs_no_gpu(lib):
    net = EffNetV2NetC()
    net.image_size, net.feat_dim, net.num_blocks = 64, 64, 0
    assert lib.vdk_effnetv2_forward(C.byref(net), 16, 1, 0, 16, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert "num_blocks" in _lib.last_error()
    assert lib.vdk_dwconv3_silu(16, 1, 7, 7, 48, 1, 16, 16, 16, 16, 0) == _lib.VDK_ERR_INVALID
    d = ConvExDesc(x=16, w=16, y=16, B=1, H=8, W=8, Cin=20, Cout=16, kernel=3, stride=1, epilogue=_lib.EPI_SILU)
    assert lib.vdk_conv2d_ex(C.byref(d), 0) == _lib.VDK_ERR_INVALID and "multiple of 8" in _lib.last_error()
