"""CPU checks of the ResNet surface: the fp32 oracle against torchvision's ResNets (which share timm's key names for the
plain and wide variants), the ResNet-D deep stem and avg-down shortcut against modules assembled here, the timm key set
and strict loading, the train-mode refusal, the ABI struct sizes, argument validation of vdk_conv2d, and the reference's
cbir.yaml with a ResNet backbone through the factory."""
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn
import torchvision

from oracle.resnet import RESNET_ARCHS as ORACLE_ARCHS, ResNet, ResNetWrapperOracle, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.resnet import RESNET_ARCHS, ResNetNetC, ResNetWrapper


@pytest.mark.parametrize("name,tv", [("resnet50", "resnet50"), ("resnet101", "resnet101"), ("wide_resnet50_2", "wide_resnet50_2")])
def test_oracle_matches_torchvision(name, tv):
    ours = randomize_(ResNet(**ORACLE_ARCHS[name]), seed=1).eval()
    ref = getattr(torchvision.models, tv)(weights=None).eval()
    sd = ours.state_dict()
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert set(missing) == {"fc.weight", "fc.bias"} and not unexpected
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        r = ref.layer4(ref.layer3(ref.layer2(ref.layer1(ref.maxpool(ref.relu(ref.bn1(ref.conv1(x))))))))
        o = ours(x)
    assert o.shape == (2, 2048, 2, 2)
    torch.testing.assert_close(o, r, rtol=1e-4, atol=1e-4)


def test_resnet_d_stem_and_avg_down_shortcut():
    """resnet50d: the deep stem and the first stride-2 block's shortcut against nn.Sequential built module by module."""
    m = randomize_(ResNet(**ORACLE_ARCHS["resnet50d"]), seed=4).eval()
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    c = m.conv1
    stem = nn.Sequential(c[0], c[1], nn.ReLU(), c[3], c[4], nn.ReLU(), c[6], m.bn1, nn.ReLU(), nn.MaxPool2d(3, 2, 1))
    assert [type(c[i]) for i in range(7)] == [nn.Conv2d, nn.BatchNorm2d, nn.ReLU, nn.Conv2d, nn.BatchNorm2d, nn.ReLU, nn.Conv2d]
    assert (c[0].stride, c[0].out_channels, c[3].out_channels, c[6].out_channels) == ((2, 2), 32, 32, 64)
    with torch.no_grad():
        h = stem(x)
        torch.testing.assert_close(m.maxpool(m.act1(m.bn1(m.conv1(x)))), h)
        y = m.layer1(h)
        blk = m.layer2[0]
        d = blk.downsample
        assert isinstance(d[0], nn.AvgPool2d) and d[1].stride == (1, 1) and m.layer1[0].downsample[0].__class__ is nn.Identity
        short = nn.Sequential(nn.AvgPool2d(2, 2, ceil_mode=True, count_include_pad=False), d[1], d[2])(y)
        main = blk.bn3(blk.conv3(blk.act2(blk.bn2(blk.conv2(blk.act1(blk.bn1(blk.conv1(y))))))))
        torch.testing.assert_close(blk(y), torch.relu(main + short))
        # on even maps the pool + 1x1 conv equals one 2x2/s2 conv with w / 4 at every tap (how the kernel runs it)
        w2 = d[1].weight.expand(-1, -1, 2, 2) / 4
        torch.testing.assert_close(nn.functional.conv2d(y, w2, stride=2), d[1](d[0](y)), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", sorted(RESNET_ARCHS))
def test_key_set_and_strict_load(name):
    assert RESNET_ARCHS[name] == ORACLE_ARCHS[name]
    oracle = randomize_(ResNetWrapperOracle(name, 128, 64), seed=2)
    ours = ResNetWrapper(name, 128, 64, pretrained=False)
    assert list(ours.state_dict()) == list(oracle.state_dict())
    ours.load_state_dict(oracle.state_dict(), strict=True)
    keys = set(ours.state_dict())
    assert "model.bn1.num_batches_tracked" in keys and "model.layer4.2.bn3.running_var" in keys
    if name.endswith("d"):
        assert {"model.conv1.0.weight", "model.conv1.1.weight", "model.conv1.3.weight", "model.conv1.4.weight",
                "model.conv1.6.weight", "model.layer2.0.downsample.1.weight", "model.layer2.0.downsample.2.running_mean"} <= keys
        assert "model.layer2.0.downsample.0.weight" not in keys
    else:
        assert {"model.conv1.weight", "model.layer2.0.downsample.0.weight", "model.layer2.0.downsample.1.running_mean"} <= keys
    width = 128 if name.startswith("wide") else 64
    assert ours.state_dict()["model.layer1.0.conv2.weight"].shape == (width, width, 3, 3)


def test_timm_checkpoint_loads_as_pretrained(tmp_path, monkeypatch):
    """A timm-layout state dict (with the classifier fc.*) in $VDK_PRETRAINED_DIR loads strictly, fc dropped."""
    m = randomize_(ResNet(**ORACLE_ARCHS["resnet50"]), seed=3)
    sd = dict(m.state_dict())
    sd["fc.weight"], sd["fc.bias"] = torch.zeros(1000, 2048), torch.zeros(1000)
    torch.save(sd, tmp_path / "resnet50.pth")
    monkeypatch.setenv("VDK_PRETRAINED_DIR", str(tmp_path))
    ours = ResNetWrapper("resnet50", 64, 64, pretrained=True)
    assert torch.equal(ours.model.layer3[5].conv2.weight, m.layer3[5].conv2.weight)


def test_train_mode_refused_before_any_kernel():
    m = ResNetWrapper("resnet50", 64, 64, pretrained=False).train()
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 64, 64))
    with pytest.raises(ValueError):
        ResNetWrapper("resnet50", 64, 100, pretrained=False)
    with pytest.raises(ValueError, match="not built for H100"):
        ResNetWrapper("resnet18", 64, 64, pretrained=False)


def test_resnet_struct_sizes(lib):
    out = (C.c_size_t * 4)()
    assert lib.vdk_resnet_struct_sizes(out, 4) == 2
    assert (out[0], out[1]) == (C.sizeof(_lib.ConvDesc), C.sizeof(ResNetNetC))


def test_conv_and_gemm_argument_validation(lib):
    d = _lib.ConvDesc(x=256, w=256, bias=0, residual=0, y=256, B=1, H=8, W=8, Cin=32, Cout=64, kernel=3, stride=1, pad=1,
                      epilogue=_lib.EPI_RELU)
    assert lib.vdk_conv2d(C.byref(d), None) == _lib.VDK_ERR_INVALID and "Cin" in _lib.last_error()
    d.Cin, d.epilogue = 64, _lib.EPI_GELU
    assert lib.vdk_conv2d(C.byref(d), None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()
    d.epilogue = _lib.EPI_RESIDUAL_RELU
    assert lib.vdk_conv2d(C.byref(d), None) == _lib.VDK_ERR_INVALID and "residual" in _lib.last_error()
    d.epilogue, d.pad = _lib.EPI_RELU, 3
    assert lib.vdk_conv2d(C.byref(d), None) == _lib.VDK_ERR_INVALID
    for epi in (_lib.EPI_RELU, _lib.EPI_RESIDUAL_RELU):  # the plain GEMM keeps refusing the convolution epilogues
        g = _lib.GemmDesc(A=256, B=256, D=256, M=8, N=8, K=8, lda=8, ldb=8, ldd=8, in_dtype=0, out_dtype=0, epilogue=epi,
                          residual=256, ldr=8, split_k=1)
        assert lib.vdk_gemm(C.byref(g), None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()


def test_reference_cbir_yaml_with_a_resnet_backbone():
    from engine.vision_engine import check, yaml_load
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_configs")
    cfgs = yaml_load(os.path.join(root, "cbir.yaml"))
    head = next(iter(cfgs["model"]["head"].values()))
    cfgs["data"]["root"] = f"synthetic://cbir?ids={head['num_class']}&per_id=2&queries=4"
    old = next(iter(cfgs["model"]["backbone"].values()))
    cfgs["model"]["backbone"] = {"timm-resnet50d.gluon_in1k": dict(old, pretrained=False)}
    check("cbir", cfgs)
    m = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    assert isinstance(m, ResNetWrapper) and m.model_name == "resnet50d" and m.feat_dim == head["feat_dim"]
    assert m.model.deep_stem and m.model.avg_down
