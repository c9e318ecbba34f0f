"""GPU parity of the MobileNetV3 embedding forward (csrc/mobilenetv3.cu vdk_mobilenetv3_forward: folded BatchNorms, the 1x1
convolutions on vdk_conv2d_ex's ReLU / hard-swish epilogues, the depthwise + hard-sigmoid SE path, conv_head, the CNN neck)
against the fp32 oracle of tests/mobilenetv3_ref.py: relative L2 error <= 1e-2 and cosine >= 0.9999 per row, tighter than
the project's embedding tolerance (3e-2 / 0.999); the measured worst case is 3.5e-3 / 0.999994 (the minimal models at 160^2).  Every BatchNorm's statistics and affine parameters are randomised, the projections' included."""
import pytest
import torch
import torch.nn.functional as F

from mobilenetv3_ref import WrapperOracle, randomize_
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.mobilenetv3 import MOBILENETV3_ARCHS, MobileNetV3Wrapper

pytestmark = pytest.mark.gpu


def embed_and_compare(name, feat, size, batch, seed=0):
    oracle = randomize_(WrapperOracle(name, feat, size), seed=seed).eval()
    ours = MobileNetV3Wrapper(name, feat, size, pretrained=False)
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().eval()
    torch.manual_seed(seed + 1)
    x = torch.randn(batch, 3, size, size)
    with torch.no_grad():
        ref = oracle(x)
    got = ours(x.cuda()).cpu()
    rel = ((got - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    cos = F.cosine_similarity(got, ref).min().item()
    print(f"{name} {size}: rel L2 err {rel:.4f}, min cosine {cos:.6f}")
    assert rel <= 1e-2 and cos >= 0.9999, f"{name}: rel L2 err {rel:.4f}, min cosine {cos:.5f}"
    got_n = ours.embed(x.cuda(), l2_normalize=True).cpu()
    assert torch.allclose(got_n.norm(dim=1), torch.ones(batch), atol=1e-5)
    assert F.cosine_similarity(got_n, F.normalize(ref)).min().item() >= 0.999
    return ours, x


@pytest.mark.parametrize("name", sorted(MOBILENETV3_ARCHS))
@pytest.mark.parametrize("size", [224, 160])
def test_full_depth_embeddings_match_oracle(lib, name, size):
    ours, x = embed_and_compare(name, 256, size, 3, seed=size + len(name))
    a = ours.embed(x.cuda())
    assert torch.equal(a, ours.embed(x.cuda()))  # bit-identical from run to run


def test_refits_after_weight_update_and_refuses_training(lib):
    ours, x = embed_and_compare("tf_mobilenetv3_small_100", 64, 64, 2, seed=9)
    x = x.cuda()
    a = ours.embed(x)
    with torch.no_grad():
        ours.model.blocks[2][0].bn2.weight.mul_(2.0)  # a new weight version: the folded depthwise taps are rebuilt
    assert not torch.equal(a, ours.embed(x))
    ours.train()
    with pytest.raises(NotImplementedError):
        ours(x)


def test_valuate_with_a_mobilenetv3_backbone(lib):
    from engine.cbir.evaluation import valuate
    model = BackboneFactory({"timm-tf_mobilenetv3_large_minimal_100.in1k": {"pretrained": False, "image_size": 64,
                                                                           "feat_dim": 64}}).get_backbone()
    randomize_(model, seed=2)
    model = model.cuda().eval()
    cfg = {"root": "synthetic://cbir?ids=8&per_id=4&queries=4", "nw": 0,
           "val": {"bs": 8, "augment": [], "metrics": {"metrics": ["mrr", "recall"], "cutoffs": [1, 5]}}}
    got = valuate(model, cfg, "cuda", image_size=64)
    assert got and all(0.0 <= v <= 1.0 for v in got.values())
