"""GPU parity of the ConvNeXt embedding forward (csrc/convnext.cu + wgmma GEMM epilogues) against the fp32
oracle (oracle/convnext.py, timm 0.9.16 restatement).

Tolerance (stated, floating point): the CUDA path keeps activations in bf16 between kernels (fp32 accumulation
inside), the oracle is fp32 end to end.  Building-block kernels are held to 2 bf16 ulps of the output scale;
whole-network embeddings to relative L2 error <= 3e-2 and cosine >= 0.999 per row.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle.convnext import TimmWrapperOracle, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import TimmWrapper, BackboneFactory

pytestmark = pytest.mark.gpu


def bf(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("B,H,W,C", [(2, 14, 14, 512), (3, 7, 7, 1024), (2, 56, 56, 128), (1, 9, 13, 96), (2, 8, 8, 40)])
def test_dwconv7_ln_block(lib, B, H, W, C):
    torch.manual_seed(C + H)
    x = bf(torch.randn(B, H, W, C, device="cuda"))
    w = 0.2 * torch.randn(C, 1, 7, 7, device="cuda")
    b, lw, lb = torch.randn(C, device="cuda") * 0.1, 1 + 0.2 * torch.randn(C, device="cuda"), 0.1 * torch.randn(C, device="cuda")
    y = torch.empty_like(x)
    w49 = w.reshape(C, 49).t().contiguous()
    _lib.check(lib.vdk_dwconv7_ln(x.data_ptr(), B, H, W, C, w49.data_ptr(), b.data_ptr(), lw.data_ptr(), lb.data_ptr(),
                                  1e-6, y.data_ptr(), _lib.stream_ptr()), "vdk_dwconv7_ln")
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=3, groups=C).permute(0, 2, 3, 1)
    ref = F.layer_norm(ref, (C,), lw, lb, 1e-6)
    err = (y.float() - ref).abs().max().item()
    assert err <= 0.04, f"dwconv7+LN max err {err}"


@pytest.mark.parametrize("B,H,W,C,patch", [(2, 14, 14, 512, 2), (2, 7, 7, 1024, 1), (1, 56, 56, 128, 2), (3, 6, 10, 96, 2)])
def test_layernorm_patchify(lib, B, H, W, C, patch):
    torch.manual_seed(C)
    x = bf(torch.randn(B, H, W, C, device="cuda") * 2 + 0.5)
    lw, lb = 1 + 0.2 * torch.randn(C, device="cuda"), 0.1 * torch.randn(C, device="cuda")
    out = torch.empty((B * (H // patch) * (W // patch), patch * patch * C), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.vdk_layernorm_patchify(x.data_ptr(), B, H, W, C, lw.data_ptr(), lb.data_ptr(), 1e-6, patch,
                                          out.data_ptr(), _lib.stream_ptr()), "vdk_layernorm_patchify")
    ref = F.layer_norm(x.float(), (C,), lw, lb, 1e-6)
    if patch == 2:
        ref = ref.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(out.shape)
    else:
        ref = ref.reshape(out.shape)
    assert (out.float() - ref).abs().max().item() <= 0.04


@pytest.mark.parametrize("N", [128, 96, 256, 32])
def test_gemm_layernorm_epilogue(lib, N):
    torch.manual_seed(N)
    M, K = 777, 48
    a = bf(torch.randn(M, K, device="cuda"))
    w = bf(torch.randn(N, K, device="cuda") * 0.3)
    bias, lw, lb = torch.randn(N, device="cuda"), 1 + 0.1 * torch.randn(N, device="cuda"), 0.1 * torch.randn(N, device="cuda")
    d = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=N,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_BF16, epilogue=_lib.EPI_LAYERNORM,
                      bias=bias.data_ptr(), gamma=lw.data_ptr(), beta=lb.data_ptr(), residual=0, ldr=0, ln_eps=1e-6, split_k=1)
    import ctypes as C
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    ref = F.layer_norm(a.float() @ w.float().t() + bias, (N,), lw, lb, 1e-6)
    assert (d.float() - ref).abs().max().item() <= 0.04


@pytest.mark.parametrize("M,N,K,split", [(64, 512, 50176, 40), (200, 64, 1024, 5), (7, 512, 12544, 300)])
def test_gemm_split_k(lib, M, N, K, split):
    import ctypes as C
    torch.manual_seed(M)
    a = bf(torch.randn(M, K, device="cuda"))
    w = bf(torch.randn(N, K, device="cuda") * 0.05)
    d = torch.zeros(M, N, dtype=torch.float32, device="cuda")
    g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=N,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE,
                      bias=0, gamma=0, beta=0, residual=0, ldr=0, ln_eps=0.0, split_k=split)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    ref = a.float() @ w.float().t()
    assert (d - ref).abs().max().item() <= 2e-3 * K ** 0.5 * 0.05 + 1e-3


def embed_and_compare(model_name, feat, size, batch, depths=None, dims=None, seed=0):
    oracle = randomize_(TimmWrapperOracle(model_name, feat, size, depths=depths, dims=dims), seed=seed).eval()
    ours = TimmWrapper(model_name, feat, size, pretrained=False, depths=depths, dims=dims)
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().eval()
    torch.manual_seed(seed + 1)
    x = torch.randn(batch, 3, size, size)
    with torch.no_grad():
        ref = oracle(x)
    got = ours(x.cuda()).cpu()
    rel = ((got - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    cos = F.cosine_similarity(got, ref).min().item()
    assert rel <= 3e-2 and cos >= 0.999, f"{model_name}: rel L2 err {rel:.4f}, min cosine {cos:.5f}"
    # extract_cbir semantics: L2-normalised rows
    got_n = ours.embed(x.cuda(), l2_normalize=True).cpu()
    assert torch.allclose(got_n.norm(dim=1), torch.ones(batch), atol=1e-5)
    assert F.cosine_similarity(got_n, F.normalize(ref)).min().item() >= 0.999
    return rel, cos


def test_small_convnext_embeddings_match_oracle(lib):
    embed_and_compare("toy", 64, 64, 5, depths=(1, 1, 2, 1), dims=(32, 64, 128, 256))


def test_convnext_base_224_embeddings_match_oracle(lib):
    rel, cos = embed_and_compare("convnext_base", 512, 224, 3, seed=3)
    print(f"convnext_base 224: rel L2 err {rel:.4f}, min cosine {cos:.5f}")


def test_backbone_factory_surface(lib):
    m = BackboneFactory({"timm-convnext_atto": {"pretrained": False, "image_size": 64, "feat_dim": 128}}).get_backbone()
    assert isinstance(m, TimmWrapper) and m.output_layer[2].weight.shape == (128, 320 * 4)
    with pytest.raises(ValueError):
        BackboneFactory({"resnet": {}}).get_backbone()
    with pytest.raises(RuntimeError):
        m.eval()
        m(torch.zeros(1, 3, 64, 64))  # CPU tensors: there is no CPU fallback
