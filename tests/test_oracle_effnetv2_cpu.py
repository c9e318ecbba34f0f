"""The EfficientNetV2 oracle (tests/effnetv2_ref.py) against torchvision's efficientnet_v2_{s,m,l}, whose module tree has the
same blocks, widths, depths, SE widths and BatchNorm eps: weights mapped across by order with shape asserts, at odd image
sizes where TF-"same" padding equals torchvision's symmetric padding.  And the oracle's TF-"same" conv against an explicit
F.pad + F.conv2d at even sizes, where it is asymmetric."""
import pytest
import torch
import torch.nn.functional as F

from effnetv2_ref import Conv2dSame, backbone, randomize_

tv_models = pytest.importorskip("torchvision.models")


@pytest.mark.parametrize("name,size", [("tf_efficientnetv2_s", 97), ("tf_efficientnetv2_m", 97), ("tf_efficientnetv2_l", 225)])
def test_oracle_matches_torchvision(name, size):
    ours = randomize_(backbone(name), seed=5).eval()
    tv = getattr(tv_models, "efficientnet_v2_" + name[-1])(weights=None).features.eval()
    src = [(k, v) for k, v in ours.state_dict().items() if not k.endswith("num_batches_tracked")]
    dst = [(k, v) for k, v in tv.state_dict().items() if not k.endswith("num_batches_tracked")]
    assert len(src) == len(dst)
    sd = {}
    for (ka, a), (kb, b) in zip(src, dst):
        assert a.shape == b.shape, (ka, kb, a.shape, b.shape)
        sd[kb] = a
    tv.load_state_dict(sd, strict=False)
    for m in tv.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            assert m.eps == 1e-3
    torch.manual_seed(0)
    x = torch.randn(1, 3, size, size)
    with torch.no_grad():
        a, b = ours(x), tv(x)
    assert a.shape == b.shape == (1, 1280, -(-size // 32), -(-size // 32))
    rel = ((a - b).norm() / b.norm()).item()
    assert rel <= 1e-4, rel


@pytest.mark.parametrize("size,stride,pads", [(16, 2, (0, 1)), (17, 2, (1, 1)), (16, 1, (1, 1)), (10, 2, (0, 1))])
def test_tf_same_conv_matches_explicit_padding(size, stride, pads):
    torch.manual_seed(size + stride)
    conv = Conv2dSame(8, 16, 3, stride, bias=False)
    x = torch.randn(2, 8, size, size + 2)  # both axes
    lo, hi = pads
    w_total = max((-(-(size + 2) // stride) - 1) * stride + 3 - (size + 2), 0)
    ref = F.conv2d(F.pad(x, (w_total // 2, w_total - w_total // 2, lo, hi)), conv.weight, stride=stride)
    with torch.no_grad():
        assert torch.equal(conv(x), ref)
    assert ref.shape[2] == -(-size // stride)
