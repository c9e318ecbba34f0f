"""CPU checks of the ResNeSt extract path: the oracle's SplitAttn against an independent per-(radix, cardinal group)
formulation, its avd_first / avd_last blocks against their pieces, timm's key sets and parameter counts, the split conv's
packed weight, strict checkpoint loads through $VDK_PRETRAINED_DIR, the train-mode refusal, the ctypes mirror of
vdk_resnest_net, the argument validation of vdk_conv2d_grouped_ex / vdk_split_attn_gate / vdk_avgpool3s2, and the
reference's cbir.yaml with the ResNeSt it lists through the factory."""
import ctypes as C
import os

import pytest
import torch
import torch.nn.functional as F

from resnest_ref import RESNEST_ARCHS as ORACLE_ARCHS
from resnest_ref import ResNestBottleneck, SplitAttn, WrapperOracle, backbone, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.resnest import RESNEST_ARCHS, ResNeStNetC, ResNeStWrapper, pack_split, split_conv_blocks, split_tile_start


def split_attn_loops(sa: SplitAttn, x):
    """SplitAttn restated without its reshapes: conv per (radix r, cardinal group g) on channel slices, BN + ReLU, the radix
    sum and mean, grouped fc1 / fc2 per g, then an explicit softmax over r (sigmoid for one radix) per output channel."""
    R, card = sa.radix, sa.fc1.groups
    C = sa.fc1.in_channels
    Cg, cgi = C // card, C // (card * R)
    A = sa.fc1.out_channels
    Ag = A // card
    bn0 = lambda t, sl: (t - sa.bn0.running_mean[sl, None, None]) / torch.sqrt(sa.bn0.running_var[sl, None, None] + sa.bn0.eps) \
        * sa.bn0.weight[sl, None, None] + sa.bn0.bias[sl, None, None]
    u = [[None] * card for _ in range(R)]  # u[r][g]: [B, Cg, H, W], output channels r C + g Cg .. + Cg
    for r in range(R):
        for g in range(card):
            gi = r * card + g  # conv group index: output channels gi * Cg .. == r C + g Cg ..
            out = slice(gi * Cg, (gi + 1) * Cg)
            y = F.conv2d(x[:, gi * cgi:(gi + 1) * cgi], sa.conv.weight[out], padding=1)
            u[r][g] = torch.relu(bn0(y, out))
    gap = [sum(u[r][g] for r in range(R)).mean((2, 3)) for g in range(card)]  # [B, Cg] per g
    outs = []
    for g in range(card):
        h = gap[g] @ sa.fc1.weight[g * Ag:(g + 1) * Ag].flatten(1).T + sa.fc1.bias[g * Ag:(g + 1) * Ag]
        h = (h - sa.bn1.running_mean[g * Ag:(g + 1) * Ag]) / torch.sqrt(sa.bn1.running_var[g * Ag:(g + 1) * Ag] + sa.bn1.eps) \
            * sa.bn1.weight[g * Ag:(g + 1) * Ag] + sa.bn1.bias[g * Ag:(g + 1) * Ag]
        h = torch.relu(h)
        rows = slice(g * R * Cg, (g + 1) * R * Cg)  # fc2's group g: R * Cg rows, radix-major inside the group
        z = (h @ sa.fc2.weight[rows].flatten(1).T + sa.fc2.bias[rows]).view(-1, R, Cg)
        a = torch.sigmoid(z) if R == 1 else torch.exp(z - z.max(1, keepdim=True).values) / torch.exp(z - z.max(1, keepdim=True).values).sum(1, keepdim=True)
        outs.append(sum(a[:, r, :, None, None] * u[r][g] for r in range(R)))
    return torch.cat(outs, dim=1)


@pytest.mark.parametrize("radix,card,width", [(1, 4, 96), (2, 1, 64), (4, 2, 80)])
def test_split_attn_matches_loop_formulation(radix, card, width):
    sa = randomize_(SplitAttn(width, width, groups=card, radix=radix), seed=radix * 10 + card).eval()
    x = torch.randn(2, width, 7, 9, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        torch.testing.assert_close(sa(x), split_attn_loops(sa, x), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("avd_first", [True, False])
def test_avd_first_and_avd_last_blocks(avd_first):
    """A stride-2 block pools the conv1 output before SplitAttn (avd_first) or SplitAttn's output after it, with
    AvgPool2d(3, 2, 1) counting the padding; the split conv itself always has stride 1."""
    planes, inplanes = 128, 256
    radix, card, bw = (4, 2, 40) if avd_first else (2, 1, 64)
    down = torch.nn.Sequential(torch.nn.AvgPool2d(2, 2, ceil_mode=True, count_include_pad=False),
                               torch.nn.Conv2d(inplanes, planes * 4, 1, bias=False), torch.nn.BatchNorm2d(planes * 4))
    blk = randomize_(ResNestBottleneck(inplanes, planes, 2, down, radix, card, bw, avd_first=avd_first), seed=7).eval()
    assert blk.conv2.conv.stride == (1, 1) and (blk.avd_first is not None) == avd_first and (blk.avd_last is None) == avd_first
    x = torch.randn(2, inplanes, 10, 10, generator=torch.Generator().manual_seed(8))
    pool = lambda t: F.avg_pool2d(t, 3, 2, 1, count_include_pad=True)
    with torch.no_grad():
        t = torch.relu(blk.bn1(blk.conv1(x)))
        t = split_attn_loops(blk.conv2, pool(t)) if avd_first else pool(split_attn_loops(blk.conv2, t))
        ref = torch.relu(blk.bn3(blk.conv3(t)) + down(x))
        torch.testing.assert_close(blk(x), ref, rtol=1e-4, atol=1e-4)


def test_no_avd_pool_without_stride():
    m = backbone("resnest50d_4s2x40d")
    for i in range(4):
        for j, blk in enumerate(getattr(m, f"layer{i + 1}")):
            strided = i > 0 and j == 0
            assert (blk.avd_first is not None) == strided and blk.avd_last is None


# timm's published parameter counts include the 1000-class classifier (2048 x 1000 + 1000)
PARAMS_M = {"resnest14d": 10.61, "resnest26d": 17.07, "resnest50d": 27.48, "resnest50d_1s4x24d": 25.68, "resnest50d_4s2x40d": 30.42}


@pytest.mark.parametrize("name", sorted(RESNEST_ARCHS))
def test_key_set_and_parameter_count(name):
    assert RESNEST_ARCHS[name] == ORACLE_ARCHS[name]
    oracle = randomize_(WrapperOracle(name, 128, 64), seed=2)
    ours = ResNeStWrapper(name, 128, 64, pretrained=False)
    assert list(ours.state_dict()) == list(oracle.state_dict())
    for k, v in oracle.state_dict().items():
        assert ours.state_dict()[k].shape == v.shape, k
    ours.load_state_dict(oracle.state_dict(), strict=True)
    n = sum(p.numel() for p in ours.model.parameters())
    assert round((n + 2048 * 1000 + 1000) / 1e6, 2) == PARAMS_M[name]
    sd = ours.state_dict()
    assert {"model.conv1.0.weight", "model.conv1.1.running_var", "model.conv1.3.weight", "model.conv1.4.bias", "model.conv1.6.weight",
            "model.bn1.weight", "model.layer1.0.conv2.conv.weight", "model.layer1.0.conv2.bn0.running_mean",
            "model.layer1.0.conv2.fc1.bias", "model.layer1.0.conv2.bn1.weight", "model.layer1.0.conv2.fc2.weight",
            "model.layer2.0.downsample.1.weight", "model.layer2.0.downsample.2.running_var"} <= set(sd)


@pytest.mark.parametrize("cin,cout,groups", [(64, 128, 2), (512, 1024, 2), (96, 96, 4), (768, 768, 4), (80, 320, 8), (640, 2560, 8),
                                             (24, 40, 8)])
def test_packed_split_weight_is_the_grouped_conv(cin, cout, groups):
    """Tile t of the packed weight, applied to input channels c_lo(t) .. c_lo(t) + cpb * 64 (zero past Cin), is the grouped conv."""
    g = torch.Generator().manual_seed(cin + groups)
    w = torch.randn(cout, cin // groups, 3, 3, generator=g, dtype=torch.float64)
    x = torch.randn(1, cin, 5, 5, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, padding=1, groups=groups)
    cpb = split_conv_blocks(cin, cout, groups)
    packed = pack_split(w, groups)
    assert packed.shape == (cout, 3, 3, cpb * 64)
    xp = F.pad(x, (0, 0, 0, 0, 0, cpb * 64 + cin))  # zero channels past Cin, as the TMA fill
    for n0 in range(0, cout, 128):
        lo = n0 // (cout // groups) * (cin // groups) // 8 * 8  # 16-byte aligned
        assert lo == split_tile_start(n0, cin // groups, cout // groups)
        got = F.conv2d(xp[:, lo:lo + cpb * 64], packed[n0:n0 + 128].permute(0, 3, 1, 2), padding=1)
        torch.testing.assert_close(got, ref[:, n0:n0 + 128], rtol=1e-12, atol=1e-12)


def test_checkpoint_with_classifier_loads_strictly(tmp_path, monkeypatch):
    m = randomize_(backbone("resnest50d_4s2x40d"), seed=3)
    sd = dict(m.state_dict())
    sd["fc.weight"], sd["fc.bias"] = torch.zeros(1000, 2048), torch.zeros(1000)
    torch.save(sd, tmp_path / "resnest50d_4s2x40d.pth")
    monkeypatch.setenv("VDK_PRETRAINED_DIR", str(tmp_path))
    ours = ResNeStWrapper("resnest50d_4s2x40d", 64, 64, pretrained=True)
    for k, v in m.state_dict().items():
        assert torch.equal(ours.model.state_dict()[k], v), k
    sd["layer1.0.conv2.extra"] = torch.zeros(1)  # strict: an unknown key is refused
    torch.save(sd, tmp_path / "resnest50d_4s2x40d.pth")
    with pytest.raises(RuntimeError):
        ResNeStWrapper("resnest50d_4s2x40d", 64, 64, pretrained=True)


def test_train_mode_and_bad_arguments_refused():
    m = ResNeStWrapper("resnest14d", 64, 64, pretrained=False)
    with pytest.raises(NotImplementedError):
        m.train()(torch.zeros(1, 3, 64, 64))
    with pytest.raises(ValueError):
        ResNeStWrapper("resnest14d", 64, 100, pretrained=False)
    with pytest.raises(ValueError, match="not built for H100"):
        ResNeStWrapper("resnest101e", 64, 64, pretrained=False)


def test_resnest_struct_size(lib):
    out = (C.c_size_t * 2)()
    assert lib.vdk_resnest_struct_sizes(out, 2) == 1
    assert out[0] == C.sizeof(ResNeStNetC)


def test_grouped_ex_conv_argument_validation(lib):
    d = _lib.ConvDesc(x=256, w=256, bias=0, residual=0, y=256, B=1, H=8, W=8, Cin=80, Cout=320, kernel=3, stride=1, pad=1,
                      epilogue=_lib.EPI_RELU)
    bad = lambda groups, what: lib.vdk_conv2d_grouped_ex(C.byref(d), groups, None) == _lib.VDK_ERR_INVALID and what in _lib.last_error()
    assert bad(3, "groups")  # 80 % 3
    assert bad(0, "groups")
    d.Cin = 84
    assert bad(2, "multiples of 8")
    d.Cin, d.Cout = 80, 324
    assert bad(2, "multiples of 8")
    d.Cout = 320
    assert bad(1, "groups=1 takes a 1x1")  # a dense 3x3 belongs to vdk_conv2d
    for epi in (_lib.EPI_GELU, _lib.EPI_SILU, _lib.EPI_SCALE_RESIDUAL):
        d.epilogue = epi
        assert bad(8, "epilogue")
    d.epilogue = _lib.EPI_RESIDUAL_RELU
    assert bad(8, "residual")
    d.epilogue, d.pad = _lib.EPI_RELU, 3
    assert bad(8, "pad")
    d.pad, d.x = 1, 258
    assert bad(8, "aligned")
    d.x = 0
    assert bad(8, "null")
    # the existing entry points keep refusing these shapes
    d.x = 256
    assert lib.vdk_conv2d_grouped(C.byref(d), 8, None) == _lib.VDK_ERR_INVALID
    d.kernel, d.pad, d.Cout = 1, 0, 256
    assert lib.vdk_conv2d(C.byref(d), None) == _lib.VDK_ERR_INVALID and "multiple of 64" in _lib.last_error()


def test_split_attn_gate_and_pool_argument_validation(lib):
    f = lambda C_, R, card, A, pool=0, u=256: lib.vdk_split_attn_gate(u, 2, 8, 8, C_, R, card, A, 256, 256, 256, 256, 256, 256, pool,
                                                                        256, None)
    assert f(84, 2, 1, 32) == _lib.VDK_ERR_INVALID and "multiple of 8" in _lib.last_error()
    assert f(80, 5, 2, 80) == _lib.VDK_ERR_INVALID and "radix" in _lib.last_error()
    assert f(80, 4, 3, 81) == _lib.VDK_ERR_INVALID and "cardinality" in _lib.last_error()
    assert f(80, 4, 2, 81) == _lib.VDK_ERR_INVALID and "cardinality" in _lib.last_error()
    assert f(1032, 4, 1, 256) == _lib.VDK_ERR_INVALID and "radix * C" in _lib.last_error()
    assert f(1024, 2, 1, 1024) == _lib.VDK_ERR_INVALID and "C + A" in _lib.last_error()
    assert f(80, 4, 2, 80, pool=2) == _lib.VDK_ERR_INVALID and "pool" in _lib.last_error()
    assert f(80, 4, 2, 80, u=0) == _lib.VDK_ERR_INVALID and "null" in _lib.last_error()
    assert lib.vdk_avgpool3s2(256, 1, 8, 8, 84, 256, None) == _lib.VDK_ERR_INVALID
    assert lib.vdk_avgpool3s2(258, 1, 8, 8, 80, 256, None) == _lib.VDK_ERR_INVALID and "alignment" in _lib.last_error()


def test_reference_cbir_yaml_with_resnest():
    from engine.vision_engine import check, yaml_load
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_configs")
    cfgs = yaml_load(os.path.join(root, "cbir.yaml"))
    head = next(iter(cfgs["model"]["head"].values()))
    cfgs["data"]["root"] = f"synthetic://cbir?ids={head['num_class']}&per_id=2&queries=4"
    old = next(iter(cfgs["model"]["backbone"].values()))
    cfgs["model"]["backbone"] = {"timm-resnest50d_4s2x40d.in1k": dict(old, pretrained=False)}
    check("cbir", cfgs)
    m = BackboneFactory(cfgs["model"]["backbone"]).get_backbone()
    assert type(m) is ResNeStWrapper and m.model_name == "resnest50d_4s2x40d" and m.feat_dim == head["feat_dim"]
    with pytest.raises(ValueError, match="not built for H100"):
        BackboneFactory({"timm-resnest101e.in1k": dict(old, pretrained=False)}).get_backbone()


@pytest.mark.parametrize("name", ["resnest14d", "resnest50d_1s4x24d", "resnest50d_4s2x40d"])
def test_oracle_against_timm(name):
    timm = pytest.importorskip("timm")
    ours = randomize_(backbone(name, depths=(1, 1, 1, 1)), seed=11).eval()
    kw = dict(RESNEST_ARCHS[name])
    ref = timm.create_model(name, pretrained=False, num_classes=0, global_pool="", layers=[1, 1, 1, 1]).eval()
    ref.load_state_dict(ours.state_dict(), strict=True)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        torch.testing.assert_close(ours(x), ref(x), rtol=1e-4, atol=1e-4)
    assert kw["radix"] == ref.layer1[0].conv2.radix
