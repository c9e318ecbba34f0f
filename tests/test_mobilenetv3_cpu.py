"""CPU-side checks of the MobileNetV3 extract path: the fp32 oracle (tests/mobilenetv3_ref.py) against torchvision's
mobilenet_v3_large / _small, which have the same blocks, widths, SE widths and activations; the minimal variants and TF
padding against their pieces; the wrapper's parameter tree against the oracle's (timm's keys); strict checkpoint loads with
the classifier dropped; the factory's routing and refusals; the ctypes mirror of vdk_mobilenetv3_net; and the reference's
own configs with their commented MobileNetV3 line."""
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from mobilenetv3_ref import Block, WrapperOracle, backbone, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.mobilenetv3 import MOBILENETV3_ARCHS, MobileNetV3NetC, MobileNetV3Wrapper, make_divisible

tv_models = pytest.importorskip("torchvision.models")

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_configs")
NAMES = sorted(MOBILENETV3_ARCHS)


def params(module):
    return sum(p.numel() for p in module.parameters())


@pytest.mark.parametrize("name,tv_name,size", [("mobilenetv3_large_100", "mobilenet_v3_large", 97),
                                               ("mobilenetv3_small_100", "mobilenet_v3_small", 64)])
def test_oracle_body_matches_torchvision(name, tv_name, size):
    ours = randomize_(backbone(name), seed=5).eval()
    tv_full = getattr(tv_models, tv_name)(weights=None)
    tv = tv_full.features.eval()
    src = [(k, v) for k, v in ours.state_dict().items() if not k.endswith("num_batches_tracked") and not k.startswith("conv_head")]
    dst = [(k, v) for k, v in tv.state_dict().items() if not k.endswith("num_batches_tracked")]
    assert len(src) == len(dst)
    sd = {}
    for (ka, a), (kb, b) in zip(src, dst):
        assert a.shape == b.shape, (ka, kb, a.shape, b.shape)
        sd[kb] = a
    tv.load_state_dict(sd, strict=True)
    for m in tv.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.eps = 1e-5  # torchvision builds eps 1e-3; timm's non-TF MobileNetV3 keeps nn.BatchNorm2d's 1e-5
    x = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        a, b = ours.forward_features(x), tv(x)
    assert a.shape == b.shape
    rel = ((a - b).norm() / b.norm()).item()
    assert rel <= 1e-4, rel
    # conv_head (1x1 with bias) + a 1000-class classifier = torchvision's classifier Linear(last, head) + Linear(head, 1000)
    head = MOBILENETV3_ARCHS[name]["head"]
    assert params(ours) + head * 1000 + 1000 == params(tv_full)


def test_minimal_variants_and_tf_padding_from_their_pieces():
    large, small = backbone("tf_mobilenetv3_large_minimal_100"), backbone("tf_mobilenetv3_small_minimal_100")
    for m, head in ((large, 1280), (small, 1024)):
        blocks = [b for s in m.blocks for b in s]
        assert all(isinstance(b.se, nn.Identity) for b in blocks if b.kind != "cn")
        assert all(b.conv_dw.kernel_size == (3, 3) for b in blocks if b.kind != "cn")
        assert all(b.act is F.relu for b in blocks) and m.act is F.relu and m.conv_head.out_channels == head
        assert all(mm.eps == 1e-3 for mm in m.modules() if isinstance(mm, nn.BatchNorm2d))
    full = backbone("tf_mobilenetv3_large_100")
    assert [b.conv_dw.kernel_size[0] for s in full.blocks for b in s if b.kind != "cn"] == [3, 3, 3, 5, 5, 5, 3, 3, 3, 3, 3, 3, 5, 5, 5]
    # a TF-"same" IR block is the same arithmetic as explicit F.pad pads + unpadded convs: (1, 2) for 5x5/s2 on an even map
    torch.manual_seed(1)
    blk = randomize_(Block("ir", 24, 40, 5, 2, 72, "hard_swish", 24, 1e-3, True), seed=2).eval()
    x = torch.randn(2, 24, 16, 16)
    with torch.no_grad():
        y = F.hardswish(blk.bn1(F.conv2d(x, blk.conv_pw.weight)))
        y = F.hardswish(blk.bn2(F.conv2d(F.pad(y, (1, 2, 1, 2)), blk.conv_dw.weight, stride=2, groups=72)))
        s = F.relu(F.conv2d(y.mean((2, 3), keepdim=True), blk.se.conv_reduce.weight, blk.se.conv_reduce.bias))
        y = y * (F.conv2d(s, blk.se.conv_expand.weight, blk.se.conv_expand.bias) + 3).clamp(0, 6) / 6
        ref = blk.bn3(F.conv2d(y, blk.conv_pwl.weight))
        torch.testing.assert_close(blk(x), ref, rtol=1e-5, atol=1e-5)
        # the stem's 3x3/s2 pads (0, 1)
        st = backbone("tf_mobilenetv3_small_100").conv_stem
        img = torch.randn(1, 3, 32, 32)
        torch.testing.assert_close(st(img), F.conv2d(F.pad(img, (0, 1, 0, 1)), st.weight, stride=2))


def test_make_divisible_widths():
    assert [make_divisible(16 * e) for e in (4, 4.5)] == [64, 72]
    assert [make_divisible(24 * e) for e in (3, 3.67, 4)] == [72, 88, 96]
    assert [make_divisible(80 * e) for e in (2.5, 2.3)] == [200, 184]
    assert [make_divisible(c * 0.25) for c in (16, 72, 120, 480, 672, 960)] == [8, 24, 32, 120, 168, 240]


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_matches_oracle(name):
    ours = MobileNetV3Wrapper(name, 256, 224, pretrained=False).state_dict()
    ref = WrapperOracle(name, 256, 224).state_dict()
    assert list(ours) == list(ref)
    for k in ref:
        assert ours[k].shape == ref[k].shape, k


def test_checkpoint_with_classifier_loads_strictly(tmp_path, monkeypatch):
    name = "tf_mobilenetv3_large_minimal_100"
    src = MobileNetV3Wrapper(name, 64, 64, pretrained=False)
    sd = dict(src.model.state_dict())
    sd["classifier.weight"] = torch.zeros(1000, 1280)
    sd["classifier.bias"] = torch.zeros(1000)
    torch.save(sd, tmp_path / f"{name}.pth")
    monkeypatch.setenv("VDK_PRETRAINED_DIR", str(tmp_path))
    got = MobileNetV3Wrapper(name, 64, 64, pretrained=True)
    for k, v in src.model.state_dict().items():
        assert torch.equal(got.model.state_dict()[k], v), k


@pytest.mark.parametrize("name", NAMES)
def test_factory_builds_every_model(name):
    key = "timm-tf_mobilenetv3_large_minimal_100.in1k" if name == "tf_mobilenetv3_large_minimal_100" else f"timm-{name}"
    m = BackboneFactory({key: {"pretrained": False, "image_size": 224, "feat_dim": 512}}).get_backbone()
    assert type(m) is MobileNetV3Wrapper and m.model_name == name
    assert m.output_layer[2].in_features == MOBILENETV3_ARCHS[name]["head"] * 7 * 7


def test_refusals():
    for name in ("mobilenetv3_large_075", "tf_mobilenetv3_large_075", "mobilenetv3_small_050", "tf_mobilenetv3_small_075",
                 "mobilenetv3_small_075", "mobilenetv3_rw", "lcnet_100", "fbnetv3_b", "mobilenetv2_100"):
        with pytest.raises(ValueError, match="not built for H100"):
            BackboneFactory({f"timm-{name}": {"pretrained": False, "image_size": 224, "feat_dim": 64}}).get_backbone()
    with pytest.raises(ValueError, match="multiple of 32"):
        MobileNetV3Wrapper("mobilenetv3_large_100", 64, 200, pretrained=False)
    m = MobileNetV3Wrapper("mobilenetv3_small_100", 64, 64, pretrained=False).train()
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 64, 64))


def test_mobilenetv3_struct_mirror(lib):
    out = (C.c_size_t * 2)()
    assert lib.vdk_mobilenetv3_struct_sizes(out, 2) == 1
    assert out[0] == C.sizeof(MobileNetV3NetC)


def test_argument_validation_needs_no_gpu(lib):
    net = MobileNetV3NetC()
    net.image_size, net.feat_dim, net.num_blocks = 64, 64, 0
    assert lib.vdk_mobilenetv3_forward(C.byref(net), 16, 1, 0, 16, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert "num_blocks" in _lib.last_error()
    net.num_blocks, net.image_size = 1, 100
    assert lib.vdk_mobilenetv3_forward(C.byref(net), 16, 1, 0, 16, 256, 1 << 30, 0) == _lib.VDK_ERR_INVALID
    assert "multiple of 32" in _lib.last_error()
    dw = lambda C_, k, s, pad=0, act=1, x=256: lib.vdk_dwconv_mnv3(x, 1, 8, 8, C_, k, s, pad, act, 256, 256, 256, 0, None)
    assert dw(20, 3, 1) == _lib.VDK_ERR_INVALID and "bad shape" in _lib.last_error()
    assert dw(16, 7, 1) == _lib.VDK_ERR_INVALID and "bad shape" in _lib.last_error()
    assert dw(16, 3, 3) == _lib.VDK_ERR_INVALID and "bad shape" in _lib.last_error()
    assert dw(16, 3, 1, pad=2) == _lib.VDK_ERR_INVALID and "pad" in _lib.last_error()
    assert dw(16, 3, 1, act=2) == _lib.VDK_ERR_INVALID and "act" in _lib.last_error()
    assert dw(16, 3, 1, x=258) == _lib.VDK_ERR_INVALID and "alignment" in _lib.last_error()
    assert lib.vdk_mnv3_se(256, 256, 1, 4, 20, 8, 256, 256, 256, 256, 256, None) == _lib.VDK_ERR_INVALID


def test_new_epilogues_stay_with_conv2d_ex(lib):
    """vdk_gemm, vdk_conv2d and the grouped convs keep refusing HARDSWISH; vdk_conv2d_ex still refuses the ResNet residual."""
    g = _lib.GemmDesc(A=256, B=256, D=256, M=8, N=8, K=8, lda=8, ldb=8, ldd=8, in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_BF16,
                      epilogue=_lib.EPI_HARDSWISH, split_k=1)
    assert lib.vdk_gemm(C.byref(g), None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()
    d = _lib.ConvDesc(x=256, w=256, bias=0, residual=0, y=256, B=1, H=8, W=8, Cin=64, Cout=64, kernel=1, stride=1, pad=0,
                      epilogue=_lib.EPI_HARDSWISH)
    assert lib.vdk_conv2d(C.byref(d), None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()
    assert lib.vdk_conv2d_grouped_ex(C.byref(d), 2, None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()
    d.Cin, d.Cout, d.kernel, d.pad = 128, 128, 3, 1
    assert lib.vdk_conv2d_grouped(C.byref(d), 2, None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()
    from visiondk_b200.efficientnet import ConvExDesc
    e = ConvExDesc(x=256, w=256, y=256, residual=256, B=1, H=8, W=8, Cin=16, Cout=16, kernel=1, stride=1,
                   epilogue=_lib.EPI_RESIDUAL_RELU)
    assert lib.vdk_conv2d_ex(C.byref(e), None) == _lib.VDK_ERR_INVALID and "epilogue" in _lib.last_error()


@pytest.mark.parametrize("name,task", [("cbir.yaml", "cbir"), ("face.yaml", "face")])
def test_reference_configs_build_their_commented_mobilenetv3(name, task):
    from engine.vision_engine import check, yaml_load
    with open(os.path.join(REF, name)) as f:
        assert "# timm-tf_mobilenetv3_large_minimal_100.in1k:" in f.read()
    cfgs = yaml_load(os.path.join(REF, name))
    head = next(iter(cfgs["model"]["head"].values()))
    cfgs["data"]["root"] = f"synthetic://cbir?ids={head['num_class']}&per_id=2&queries=4"
    old = next(iter(cfgs["model"]["backbone"].values()))
    cfgs["model"]["backbone"] = {"timm-tf_mobilenetv3_large_minimal_100.in1k": dict(old, pretrained=False)}
    check(task, cfgs)
    m = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    assert type(m) is MobileNetV3Wrapper and m.model_name == "tf_mobilenetv3_large_minimal_100"
    assert m.feat_dim == head["feat_dim"] and m.image_size == old["image_size"]
