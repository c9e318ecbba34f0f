"""GPU parity of the ResNeSt embedding forward (csrc/resnest.cu vdk_resnest_forward: folded BatchNorms, split convs on
vdk_conv2d_grouped_ex, the split-attention gate, avd pools, the CNN neck) against the fp32 oracle of tests/resnest_ref.py,
at the project's embedding tolerance: relative L2 error <= 3e-2 and cosine >= 0.999 per row, with every BatchNorm's
statistics and affine parameters randomised.  Also: run-to-run bit-identical embeddings, the refit after a weight update,
the train-mode refusal, and valuate with a ResNeSt backbone."""
import pytest
import torch
import torch.nn.functional as F

from resnest_ref import WrapperOracle, randomize_
from visiondk_b200.backbone import BackboneFactory
from visiondk_b200.resnest import RESNEST_ARCHS, ResNeStWrapper

pytestmark = pytest.mark.gpu


def embed_and_compare(name, feat, size, batch, depths=None, seed=0):
    oracle = randomize_(WrapperOracle(name, feat, size, depths=depths), seed=seed).eval()
    ours = ResNeStWrapper(name, feat, size, pretrained=False, depths=depths)
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
    assert rel <= 3e-2 and cos >= 0.999, f"{name}: rel L2 err {rel:.4f}, min cosine {cos:.5f}"
    got_n = ours.embed(x.cuda(), l2_normalize=True).cpu()
    assert torch.allclose(got_n.norm(dim=1), torch.ones(batch), atol=1e-5)
    assert F.cosine_similarity(got_n, F.normalize(ref)).min().item() >= 0.999
    return ours, x


@pytest.mark.parametrize("name", sorted(RESNEST_ARCHS))
def test_every_arch_at_depth_one_per_stage(lib, name):
    embed_and_compare(name, 128, 64, 3, depths=(1, 1, 1, 1), seed=len(name))


@pytest.mark.parametrize("name,size", [("resnest50d_4s2x40d", 224), ("resnest50d", 224), ("resnest50d_1s4x24d", 288)])
def test_full_size_embeddings_match_oracle(lib, name, size):
    ours, x = embed_and_compare(name, 512, size, 2, seed=3)
    a = ours.embed(x.cuda())
    b = ours.embed(x.cuda())
    assert torch.equal(a, b), "embeddings differ between two runs on the same batch"


def test_refits_after_weight_update_and_refuses_training(lib):
    ours, _ = embed_and_compare("resnest50d_4s2x40d", 64, 64, 2, depths=(1, 2, 1, 1), seed=9)
    x = torch.randn(2, 3, 64, 64, device="cuda")
    a = ours.embed(x)
    with torch.no_grad():
        ours.model.layer1[0].conv2.bn1.weight.mul_(2.0)  # a new weight version: the folded attention weights are rebuilt
    assert not torch.equal(a, ours.embed(x))
    ours.train()
    with pytest.raises(NotImplementedError):
        ours(x)


def test_valuate_with_a_resnest_backbone(lib):
    from engine.cbir.evaluation import valuate
    model = BackboneFactory({"timm-resnest14d.gluon_in1k": {"pretrained": False, "image_size": 64, "feat_dim": 64}}).get_backbone()
    randomize_(model, seed=2)
    model = model.cuda().eval()
    cfg = {"root": "synthetic://cbir?ids=8&per_id=4&queries=4", "nw": 0,
           "val": {"bs": 8, "augment": [], "metrics": {"metrics": ["mrr", "recall"], "cutoffs": [1, 5]}}}
    got = valuate(model, cfg, "cuda", image_size=64)
    assert got and all(0.0 <= v <= 1.0 for v in got.values())
