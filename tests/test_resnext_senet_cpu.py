"""CPU checks of the ResNeXt and legacy SENet surface: the ResNeXt oracle against torchvision's ResNeXts, the SE module
against torchvision.ops.SqueezeExcitation, the SE bottlenecks and the ceil-mode stem pool against modules assembled here,
the block-diagonal packing of grouped weights, timm key sets and strict loads, timm checkpoints through
$VDK_PRETRAINED_DIR, the train-mode refusal, the new ABI struct, vdk_conv2d_grouped's argument validation, and the
reference's cbir.yaml with both new backbones through the factory."""
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision

from resnext_senet_ref import RESNEXT_ARCHS as ORACLE_RESNEXT, SENET_ARCHS as ORACLE_SENET
from resnext_senet_ref import SEModule, SENet, WrapperOracle, backbone, block_diagonal, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.resnet import RESNET_ARCHS, RESNEXT_ARCHS, BottleneckNetC, ResNetWrapper, pack_grouped
from visiondk_b200.senet import SENET_ARCHS, SENetWrapper


@pytest.mark.parametrize("name", ["resnext50_32x4d", "resnext101_32x8d", "resnext101_64x4d"])
def test_resnext_oracle_matches_torchvision(name):
    ours = randomize_(backbone(name), seed=1).eval()
    ref = getattr(torchvision.models, name)(weights=None).eval()
    missing, unexpected = ref.load_state_dict(ours.state_dict(), strict=False)
    assert set(missing) == {"fc.weight", "fc.bias"} and not unexpected
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        r = ref.layer4(ref.layer3(ref.layer2(ref.layer1(ref.maxpool(ref.relu(ref.bn1(ref.conv1(x))))))))
        o = ours(x)
    assert o.shape == (2, 2048, 2, 2)
    torch.testing.assert_close(o, r, rtol=1e-4, atol=1e-4)


def test_se_module_matches_torchvision_squeeze_excitation():
    se = randomize_(SEModule(256, 16), seed=2)
    tv = torchvision.ops.SqueezeExcitation(256, 16)
    tv.load_state_dict(se.state_dict(), strict=True)  # fc1 / fc2 names match
    x = torch.randn(3, 256, 7, 5, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        torch.testing.assert_close(se(x), tv(x), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", ["legacy_seresnet50", "legacy_seresnext50_32x4d"])
def test_se_stem_and_first_stride_two_block(name):
    """The 7x7 stem + MaxPool2d(3, 2, ceil_mode=True) and the first stride-2 block, against torch.nn pieces: SE-ResNet
    strides its 1x1 conv1, SE-ResNeXt its grouped 3x3 conv2."""
    m = randomize_(backbone(name), seed=4).eval()
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    l0 = m.layer0
    stem = nn.Sequential(l0.conv1, l0.bn1, nn.ReLU(), nn.MaxPool2d(3, 2, ceil_mode=True))
    assert (l0.conv1.kernel_size, l0.conv1.stride, l0.conv1.padding) == ((7, 7), (2, 2), (3, 3))
    with torch.no_grad():
        h = stem(x)
        torch.testing.assert_close(m.pool0(m.layer0(x)), h)
        # on the even 32x32 stem map the unpadded ceil-mode pool has the padded pool's output size, one pixel later
        assert h.shape[-1] == F.max_pool2d(l0.bn1(l0.conv1(x)), 3, 2, 1).shape[-1] == 16
        y = m.layer1(h)
        blk = m.layer2[0]
        seresnet = name.startswith("legacy_seresnet")
        assert blk.conv1.stride == ((2, 2) if seresnet else (1, 1)) and blk.conv2.stride == ((1, 1) if seresnet else (2, 2))
        assert blk.conv2.groups == (1 if seresnet else 32)
        main = blk.bn3(blk.conv3(torch.relu(blk.bn2(blk.conv2(torch.relu(blk.bn1(blk.conv1(y))))))))
        se = blk.se_module
        gate = torch.sigmoid(se.fc2(torch.relu(se.fc1(F.adaptive_avg_pool2d(main, 1)))))
        short = blk.downsample[1](blk.downsample[0](y))
        torch.testing.assert_close(blk(y), torch.relu(main * gate + short))


@pytest.mark.parametrize("cg", [4, 8, 16, 32, 64])
def test_block_diagonal_packing_is_the_grouped_conv(cg):
    cout = 256
    w = torch.randn(cout, cg, 3, 3, generator=torch.Generator().manual_seed(cg), dtype=torch.float64)
    x = torch.randn(2, cout, 6, 6, generator=torch.Generator().manual_seed(cg + 1), dtype=torch.float64)
    ref = F.conv2d(x, w, padding=1, groups=cout // cg)
    torch.testing.assert_close(F.conv2d(x, block_diagonal(w).permute(0, 3, 1, 2), padding=1), ref, rtol=1e-12, atol=1e-12)
    # the kernel's [Cout, 3, 3, 128]: tile t of the output contracts over input channels 128 t .. 128 t + 127
    packed = pack_grouped(w)
    assert packed.shape == (cout, 3, 3, 128)
    dense = block_diagonal(w)
    for t in range(cout // 128):
        torch.testing.assert_close(packed[128 * t:128 * (t + 1)], dense[128 * t:128 * (t + 1), :, :, 128 * t:128 * (t + 1)])


@pytest.mark.parametrize("name", sorted(RESNEXT_ARCHS) + sorted(SENET_ARCHS))
def test_key_set_and_strict_load(name):
    assert (RESNEXT_ARCHS.get(name) or SENET_ARCHS.get(name)) == (ORACLE_RESNEXT.get(name) or ORACLE_SENET.get(name))
    assert name not in RESNET_ARCHS
    oracle = randomize_(WrapperOracle(name, 128, 64), seed=2)
    ours = (ResNetWrapper if name in RESNEXT_ARCHS else SENetWrapper)(name, 128, 64, pretrained=False)
    assert list(ours.state_dict()) == list(oracle.state_dict())
    for k, v in oracle.state_dict().items():
        assert ours.state_dict()[k].shape == v.shape, k
    ours.load_state_dict(oracle.state_dict(), strict=True)
    sd = ours.state_dict()
    groups = (RESNEXT_ARCHS.get(name) or {}).get("cardinality") or SENET_ARCHS.get(name, {}).get("groups")
    w1 = sd["model.layer1.0.conv2.weight"]
    width = w1.shape[0]
    assert w1.shape == (width, width // groups, 3, 3)
    if name in SENET_ARCHS:
        assert {"model.layer0.conv1.weight", "model.layer0.bn1.running_var", "model.layer1.0.se_module.fc1.weight",
                "model.layer1.0.se_module.fc2.bias", "model.layer2.0.downsample.0.weight",
                "model.layer2.0.downsample.1.running_mean"} <= set(sd)
        assert sd["model.layer4.0.se_module.fc1.weight"].shape == (128, 2048, 1, 1)
        assert width == (64 if groups == 1 else 128)
    else:
        assert width == RESNEXT_ARCHS[name]["cardinality"] * RESNEXT_ARCHS[name]["base_width"]


@pytest.mark.parametrize("name,cls,prefix", [("resnext50_32x4d", ResNetWrapper, "fc"),
                                             ("legacy_seresnet50", SENetWrapper, "last_linear")])
def test_timm_checkpoint_loads_as_pretrained(tmp_path, monkeypatch, name, cls, prefix):
    """A timm-layout state dict with its classifier (fc.* / last_linear.*) in $VDK_PRETRAINED_DIR loads strictly, the
    classifier dropped."""
    m = randomize_(backbone(name), seed=3)
    sd = dict(m.state_dict())
    sd[f"{prefix}.weight"], sd[f"{prefix}.bias"] = torch.zeros(1000, 2048), torch.zeros(1000)
    torch.save(sd, tmp_path / f"{name}.pth")
    monkeypatch.setenv("VDK_PRETRAINED_DIR", str(tmp_path))
    ours = cls(name, 64, 64, pretrained=True)
    assert torch.equal(ours.model.layer3[5].conv2.weight, m.layer3[5].conv2.weight)


def test_train_mode_refused_before_any_kernel():
    for m in (ResNetWrapper("resnext50_32x4d", 64, 64, pretrained=False), SENetWrapper("legacy_seresnext26_32x4d", 64, 64, pretrained=False)):
        with pytest.raises(NotImplementedError):
            m.train()(torch.zeros(1, 3, 64, 64))
    with pytest.raises(ValueError):
        SENetWrapper("legacy_seresnet50", 64, 100, pretrained=False)
    with pytest.raises(ValueError, match="not built for H100"):
        SENetWrapper("seresnet50", 64, 64, pretrained=False)


def test_bottleneck_struct_size(lib):
    out = (C.c_size_t * 2)()
    assert lib.vdk_bottleneck_struct_sizes(out, 2) == 1
    assert out[0] == C.sizeof(BottleneckNetC)


def test_grouped_conv_argument_validation(lib):
    d = _lib.ConvDesc(x=256, w=256, bias=0, residual=0, y=256, B=1, H=8, W=8, Cin=128, Cout=256, kernel=3, stride=1, pad=1,
                      epilogue=_lib.EPI_RELU)
    assert lib.vdk_conv2d_grouped(C.byref(d), 32, None) == _lib.VDK_ERR_INVALID and "Cin must equal Cout" in _lib.last_error()
    d.Cout = 128
    assert lib.vdk_conv2d_grouped(C.byref(d), 3, None) == _lib.VDK_ERR_INVALID and "groups" in _lib.last_error()  # 128 % 3
    d.Cin = d.Cout = 384
    assert lib.vdk_conv2d_grouped(C.byref(d), 2, None) == _lib.VDK_ERR_INVALID and "groups" in _lib.last_error()  # cg = 192
    assert lib.vdk_conv2d_grouped(C.byref(d), 1, None) == _lib.VDK_ERR_INVALID and "groups" in _lib.last_error()
    d.Cin = d.Cout = 64
    assert lib.vdk_conv2d_grouped(C.byref(d), 16, None) == _lib.VDK_ERR_INVALID and "multiple of 128" in _lib.last_error()
    d.Cin = d.Cout = 256
    for epi in (_lib.EPI_NONE, _lib.EPI_RESIDUAL_RELU, _lib.EPI_GELU):
        d.epilogue = epi
        assert lib.vdk_conv2d_grouped(C.byref(d), 32, None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()
    d.epilogue, d.pad = _lib.EPI_RELU, 3
    assert lib.vdk_conv2d_grouped(C.byref(d), 32, None) == _lib.VDK_ERR_INVALID and "pad" in _lib.last_error()


@pytest.mark.parametrize("backbone_name,cls,model_name", [("timm-resnext50_32x4d.a3_in1k", ResNetWrapper, "resnext50_32x4d"),
                                                          ("timm-legacy_seresnet50.in1k", SENetWrapper, "legacy_seresnet50")])
def test_reference_cbir_yaml_with_the_new_backbones(backbone_name, cls, model_name):
    from engine.vision_engine import check, yaml_load
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_configs")
    cfgs = yaml_load(os.path.join(root, "cbir.yaml"))
    head = next(iter(cfgs["model"]["head"].values()))
    cfgs["data"]["root"] = f"synthetic://cbir?ids={head['num_class']}&per_id=2&queries=4"
    old = next(iter(cfgs["model"]["backbone"].values()))
    cfgs["model"]["backbone"] = {backbone_name: dict(old, pretrained=False)}
    check("cbir", cfgs)
    m = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    assert type(m) is cls and m.model_name == model_name and m.feat_dim == head["feat_dim"]
