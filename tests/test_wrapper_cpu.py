"""The host scaffolding every backbone wrapper shares (visiondk_b200/wrapper.py): the packed-weight cache and the refusal of
CPU input, for one small configuration of each family."""
import pytest
import torch

from visiondk_b200.backbone import TimmWrapper
from visiondk_b200.efficientnet import EfficientNetV2Wrapper
from visiondk_b200.resnest import ResNeStWrapper
from visiondk_b200.resnet import ResNetWrapper
from visiondk_b200.senet import SENetWrapper
from visiondk_b200.swin import SwinV2Wrapper
from visiondk_b200.vit import ViTWrapper

CONFIGS = {
    "convnext_atto": lambda: TimmWrapper("convnext_atto", 64, 64, pretrained=False),
    "vit_depth1": lambda: ViTWrapper("vit_depth1", 64, 32, pretrained=False, patch=16, dim=128, depth=1, heads=2),
    "resnet50d": lambda: ResNetWrapper("resnet50d", 64, 64, pretrained=False, depths=(1, 1, 1, 1)),
    "resnext50_32x4d": lambda: ResNetWrapper("resnext50_32x4d", 64, 64, pretrained=False, depths=(1, 1, 1, 1)),
    "legacy_seresnext26_32x4d": lambda: SENetWrapper("legacy_seresnext26_32x4d", 64, 64, pretrained=False),
    "resnest50d_4s2x40d": lambda: ResNeStWrapper("resnest50d_4s2x40d", 64, 64, pretrained=False, depths=(1, 1, 1, 1)),
    "tf_efficientnetv2_s": lambda: EfficientNetV2Wrapper("tf_efficientnetv2_s", 64, 64, pretrained=False, depths=(1,) * 6),
    "swinv2_base_window8_256": lambda: SwinV2Wrapper("swinv2_base_window8_256", 64, 256, pretrained=False, depths=(1, 1, 1, 1)),
}


@pytest.fixture(scope="module", params=sorted(CONFIGS))
def wrapper(request):
    torch.manual_seed(0)
    return CONFIGS[request.param]().eval()


def _neck_bias(m, net):
    """The packed neck bias, looked up through the tensors the pack keeps alive."""
    return next(t for t in m._packed["keep"] if t.data_ptr() == net.neck_b)


def test_pack_is_reused_while_nothing_changes(wrapper):
    net = wrapper._pack("cpu")
    assert wrapper._pack("cpu") is net
    assert wrapper._pack(torch.device("cpu")) is net


def test_pack_is_rebuilt_after_an_in_place_parameter_change(wrapper):
    net = wrapper._pack("cpu")
    before = _neck_bias(wrapper, net).clone()
    with torch.no_grad():
        wrapper.output_layer[2].bias.add_(1.0)
    rebuilt = wrapper._pack("cpu")
    assert rebuilt is not net
    assert not torch.equal(_neck_bias(wrapper, rebuilt), before)


def test_pack_is_rebuilt_after_a_batchnorm_running_statistic_changes(wrapper):
    net = wrapper._pack("cpu")
    before = _neck_bias(wrapper, net).clone()
    wrapper.output_layer[3].running_mean.add_(1.0)
    rebuilt = wrapper._pack("cpu")
    assert rebuilt is not net
    assert not torch.equal(_neck_bias(wrapper, rebuilt), before)


def test_pack_is_rebuilt_after_invalidate_pack(wrapper):
    net = wrapper._pack("cpu")
    before = _neck_bias(wrapper, net).clone()
    wrapper.output_layer[2].bias.data.add_(1.0)  # a write that does not bump `_version`, as the fused optimizer's kernels do
    assert wrapper._pack("cpu") is net
    wrapper.invalidate_pack()
    rebuilt = wrapper._pack("cpu")
    assert rebuilt is not net
    assert not torch.equal(_neck_bias(wrapper, rebuilt), before)


def test_cpu_input_is_refused(wrapper):
    x = torch.zeros(1, 3, wrapper.image_size, wrapper.image_size)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        wrapper.embed(x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        wrapper(x)
