"""GPU parity of the ConvNeXt TRAINING path (csrc/convnext_train.cu, train_ops.cu, the MN-major / GELU-grad GEMM forms)
against torch autograd on the fp32 oracle (oracle/convnext.py in train mode).

Tolerances (floating point, stated): activations and activation gradients are bf16 between kernels while the oracle is
fp32, so building blocks are held to a few bf16 ulps of their output scale, and whole-network parameter gradients to
relative L2 error <= 6e-2 with cosine >= 0.995 per tensor (tensors whose reference gradient is numerically zero are
compared in absolute terms)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle.convnext import TimmWrapperOracle, randomize_
from visiondk_b200 import _lib
from visiondk_b200.backbone import TimmWrapper

pytestmark = pytest.mark.gpu
bf = lambda t: t.to(torch.bfloat16)


def rel(got, ref):
    return ((got.float() - ref.float()).norm() / ref.float().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("B,H,W,Cn,patch", [(2, 14, 14, 512, 1), (3, 8, 8, 128, 2), (2, 7, 7, 1024, 1), (2, 56, 56, 128, 2)])
def test_layernorm_bwd(lib, B, H, W, Cn, patch):
    torch.manual_seed(Cn + patch)
    x = (torch.randn(B, H, W, Cn, device="cuda") * 2 + 0.3).requires_grad_(True)
    lw = (1 + 0.3 * torch.randn(Cn, device="cuda")).requires_grad_(True)
    lb = (0.2 * torch.randn(Cn, device="cuda")).requires_grad_(True)
    yref = F.layer_norm(x, (Cn,), lw, lb, 1e-6)
    if patch == 2:
        rows = yref.reshape(B, H // 2, 2, W // 2, 2, Cn).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * Cn)
    else:
        rows = yref.reshape(-1, Cn)
    dy = bf(torch.randn_like(rows))
    add = bf(torch.randn(B, H, W, Cn, device="cuda"))
    rows.backward(dy.float())
    rstd = (x.detach().var(dim=-1, unbiased=False) + 1e-6).rsqrt().reshape(-1).contiguous()
    ysave = bf(rows.detach()).contiguous()
    dx = torch.empty(B, H, W, Cn, dtype=torch.bfloat16, device="cuda")
    dg, db = torch.zeros(Cn, device="cuda"), torch.zeros(Cn, device="cuda")
    _lib.check(lib.vdk_layernorm_bwd(dy.data_ptr(), ysave.data_ptr(), rstd.data_ptr(), B, H, W, Cn, lw.data_ptr(), lb.data_ptr(),
                                     patch, dx.data_ptr(), add.data_ptr(), dg.data_ptr(), db.data_ptr(), _lib.stream_ptr()), "ln_bwd")
    assert rel(dx, x.grad + add.float()) <= 2e-2
    assert rel(dg, lw.grad) <= 2e-2 and rel(db, lb.grad) <= 1e-2


@pytest.mark.parametrize("B,H,W,Cn", [(2, 14, 14, 512), (3, 7, 7, 1024), (2, 56, 56, 128), (2, 4, 4, 64), (1, 28, 28, 256)])
def test_dwconv7_backward(lib, B, H, W, Cn):
    torch.manual_seed(Cn + H)
    x = bf(torch.randn(B, H, W, Cn, device="cuda"))
    w = (0.2 * torch.randn(Cn, 1, 7, 7, device="cuda")).requires_grad_(True)
    bias = torch.zeros(Cn, device="cuda", requires_grad=True)
    xin = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    out = F.conv2d(xin, w, bias, padding=3, groups=Cn)
    dconv = bf(torch.randn(B, H, W, Cn, device="cuda"))
    out.backward(dconv.float().permute(0, 3, 1, 2))
    # data gradient = the same correlation with reversed taps (+ the residual-branch gradient)
    w49 = w.detach().reshape(Cn, 49).t().contiguous()
    wflip = w49.flip(0).contiguous()
    add = bf(torch.randn(B, H, W, Cn, device="cuda"))
    dx = torch.empty_like(x)
    _lib.check(lib.vdk_dwconv7(1, dconv.data_ptr(), B, H, W, Cn, wflip.data_ptr(), 0, 0, 0, 0.0, dx.data_ptr(), 0, add.data_ptr(),
                               _lib.stream_ptr()), "dwconv7 bwd-data")
    assert rel(dx, xin.grad.permute(0, 2, 3, 1) + add.float()) <= 1.5e-2
    # weight gradient
    dw49 = torch.zeros(49, Cn, device="cuda")
    dbias = torch.zeros(Cn, device="cuda")
    _lib.check(lib.vdk_dwconv7_wgrad(x.data_ptr(), dconv.data_ptr(), B, H, W, Cn, dw49.data_ptr(), dbias.data_ptr(),
                                     _lib.stream_ptr()), "dwconv7 wgrad")
    assert rel(dw49.t().reshape(Cn, 1, 7, 7), w.grad) <= 1e-3
    assert rel(dbias, bias.grad) <= 1e-3


@pytest.mark.parametrize("is_bf16", [1, 0])
def test_batchnorm_train(lib, is_bf16):
    torch.manual_seed(is_bf16)
    R, Cn = 300, 200
    dt = torch.bfloat16 if is_bf16 else torch.float32
    x = (torch.randn(R, Cn, device="cuda") * 1.5 + 0.4).to(dt)
    bn = torch.nn.BatchNorm1d(Cn).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.2)
    xr = x.float().requires_grad_(True)
    yref = bn(xr)
    dy = torch.randn(R, Cn, device="cuda").to(dt)
    yref.backward(dy.float())
    y = torch.empty(R, Cn, dtype=dt, device="cuda")
    mean, rstd = torch.empty(Cn, device="cuda"), torch.empty(Cn, device="cuda")
    rm, rv = torch.zeros(Cn, device="cuda"), torch.ones(Cn, device="cuda")
    _lib.check(lib.vdk_batchnorm_train_fwd(x.data_ptr(), R, Cn, is_bf16, bn.weight.data_ptr(), bn.bias.data_ptr(), 1e-5, 0.1,
                                           y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                                           _lib.stream_ptr()), "bn fwd")
    assert rel(y, yref) <= (1e-2 if is_bf16 else 1e-5)
    assert rel(rm, bn.running_mean) <= 1e-4 and rel(rv, bn.running_var) <= 1e-4
    dx = torch.empty(R, Cn, dtype=dt, device="cuda")
    dw, db = torch.zeros(Cn, device="cuda"), torch.zeros(Cn, device="cuda")
    _lib.check(lib.vdk_batchnorm_train_bwd(dy.data_ptr(), x.data_ptr(), R, Cn, is_bf16, bn.weight.data_ptr(), mean.data_ptr(),
                                           rstd.data_ptr(), dx.data_ptr(), dw.data_ptr(), db.data_ptr(), _lib.stream_ptr()), "bn bwd")
    assert rel(dx, xr.grad) <= (1e-2 if is_bf16 else 1e-4)
    assert rel(dw, bn.weight.grad) <= 1e-3 and rel(db, bn.bias.grad) <= 1e-3


def test_gemm_gelu_aux_out_and_gelu_grad(lib):
    """Training epilogues: GELU that also saves the pre-activation, and dgrad scaled by gelu'(saved pre-activation)."""
    torch.manual_seed(0)
    M, N, K = 1000, 512, 128
    a = bf(0.5 * torch.randn(M, K, device="cuda"))
    w = bf(0.2 * torch.randn(N, K, device="cuda"))
    bias = torch.randn(N, device="cuda")
    hpost = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    hpre = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=hpost.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=N,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_BF16, epilogue=_lib.EPI_GELU, bias=bias.data_ptr(), gamma=0,
                      beta=0, residual=0, ldr=0, ln_eps=0.0, split_k=1, split_stride=0, aux_out=hpre.data_ptr(), trans_a=0, trans_b=0)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "gemm gelu+aux")
    pre_ref = (a.float() @ w.float().t() + bias).requires_grad_(True)
    post_ref = F.gelu(pre_ref)
    assert (hpre.float() - pre_ref).abs().max().item() <= 3e-2
    assert (hpost.float() - post_ref).abs().max().item() <= 3e-2
    # dgrad through the GELU: dpre = (dpost . W2') * gelu'(pre)
    K2 = 256
    dout = bf(torch.randn(M, K2, device="cuda"))
    w2 = bf(0.1 * torch.randn(K2, N, device="cuda"))  # stored [K2 (contraction), N]: trans_b form
    dpre = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    g = _lib.GemmDesc(A=dout.data_ptr(), B=w2.data_ptr(), D=dpre.data_ptr(), M=M, N=N, K=K2, lda=K2, ldb=N, ldd=N,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_BF16, epilogue=_lib.EPI_MUL_GELU_GRAD, bias=0, gamma=0, beta=0,
                      residual=hpre.data_ptr(), ldr=N, ln_eps=0.0, split_k=1, split_stride=0, aux_out=0, trans_a=0, trans_b=1)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "gemm gelu-grad")
    post = F.gelu(hpre.float().requires_grad_(True))
    hp = hpre.float().requires_grad_(True)
    F.gelu(hp).backward(dout.float() @ w2.float())
    assert rel(dpre, hp.grad) <= 2e-2


def build_pair(seed=0, depths=(1, 1, 2, 1), dims=(64, 128, 128, 256), size=64, feat=64):
    oracle = randomize_(TimmWrapperOracle("toy", feat, size, depths=depths, dims=dims), seed=seed).train()
    ours = TimmWrapper("toy", feat, size, pretrained=False, depths=depths, dims=dims)
    ours.load_state_dict(oracle.state_dict(), strict=True)
    return oracle, ours.cuda().train()


def test_train_forward_backward_matches_oracle_autograd(lib):
    oracle, ours = build_pair(seed=7)
    torch.manual_seed(1)
    x = torch.randn(6, 3, 64, 64)
    wout = torch.randn(6, 64)
    out_ref = oracle(x)
    (out_ref * wout).sum().backward()
    out = ours(x.cuda())
    (out * wout.cuda()).sum().backward()
    assert rel(out.detach().cpu(), out_ref.detach()) <= 3e-2
    ref_grads = dict(oracle.named_parameters())
    # LayerNorm right before a batch-statistics BatchNorm: a per-channel scale / shift of the BN input is removed by the
    # normalisation, so the exact gradient of head.norm.{weight,bias} is 0 and only rounding noise remains on both sides
    invariant = {"model.head.norm.weight", "model.head.norm.bias"}
    bn_scale = ref_grads["output_layer.0.weight"].grad.abs().max().item()
    stats, bad = [], []
    for n, p in ours.named_parameters():
        gr = ref_grads[n].grad
        g = p.grad.detach().cpu()
        assert torch.isfinite(g).all(), n
        if n in invariant or gr.norm() < 1e-6 * (1 + gr.numel() ** 0.5):
            err = (g - gr).abs().max().item()
            stats.append((n, "abs", err, 0.0))
            if err > 5e-2 * bn_scale + 1e-3:
                bad.append(f"{n}: |err| {err:.3e} (exact gradient ~0)")
            continue
        r = rel(g, gr)
        c = F.cosine_similarity(g.flatten(), gr.flatten(), dim=0).item()
        stats.append((n, "rel", r, c))
        if not (r <= 6e-2 and c >= 0.995):
            bad.append(f"{n}: rel {r:.4f} cos {c:.5f} |ref| {gr.norm():.3e}")
    for n, kind, a, c in sorted(stats, key=lambda t: -t[2])[:12]:
        print(f"  {kind} {a:.4f} cos {c:.5f} {n}")
    assert not bad, "\n".join(bad)
    # BatchNorm running statistics follow nn.BatchNorm's update
    for i in (0, 3):
        assert rel(ours.output_layer[i].running_mean.cpu(), oracle.output_layer[i].running_mean) <= 2e-2
        assert rel(ours.output_layer[i].running_var.cpu(), oracle.output_layer[i].running_var) <= 2e-2
        assert int(ours.output_layer[i].num_batches_tracked) == 1


def test_convnext_base_224_training_gradients_match_oracle(lib):
    """Full-size ConvNeXt-B 224^2 (BASELINE configs[1] backbone), batch 3: the shapes that select the clustered depthwise
    kernel with 1/2/4/8 chunks, the wide and narrow GEMM tiles with every epilogue, the 14x14 / 7x7 weight-gradient tiles.  Every
    parameter gradient is compared with fp32 autograd of the oracle.  Tolerance: bf16 activations through 36 blocks of
    forward and backward against fp32 -> rel <= 0.15, cos >= 0.99."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oracle = randomize_(TimmWrapperOracle("convnext_base", 512, 224), seed=3).train()
    ours = TimmWrapper("convnext_base", 512, 224, pretrained=False)
    ours.load_state_dict(oracle.state_dict(), strict=True)
    ours = ours.cuda().train()
    torch.manual_seed(5)
    x = torch.randn(3, 3, 224, 224)
    wout = torch.randn(3, 512)
    out_ref = oracle(x)
    (out_ref * wout).sum().backward()
    out = ours(x.cuda())
    (out * wout.cuda()).sum().backward()
    assert rel(out.detach().cpu(), out_ref.detach()) <= 4e-2
    ref = dict(oracle.named_parameters())
    # exact gradient 0: an affine shift / per-channel scale in front of a batch-statistics BatchNorm is normalised away
    # (head LayerNorm -> BN2d; BN2d bias and Linear bias -> BN1d); only rounding noise remains on both sides
    invariant = {"model.head.norm.weight", "model.head.norm.bias", "output_layer.0.bias", "output_layer.2.bias"}
    bn_scale = ref["output_layer.0.weight"].grad.abs().max().item()
    bad, worst = [], []
    for n, p in ours.named_parameters():
        gr, g = ref[n].grad, p.grad.detach().cpu()
        assert torch.isfinite(g).all(), n
        if n in invariant or gr.norm() < 1e-6 * (1 + gr.numel() ** 0.5):
            if (g - gr).abs().max().item() > 5e-2 * bn_scale + 1e-3:
                bad.append(f"{n}: exact gradient ~0 but |err| {(g - gr).abs().max().item():.3e}")
            continue
        r = rel(g, gr)
        c = F.cosine_similarity(g.flatten(), gr.flatten(), dim=0).item()
        worst.append((r, c, n))
        if not (r <= 0.15 and c >= 0.99):
            bad.append(f"{n}: rel {r:.4f} cos {c:.5f}")
    for r, c, n in sorted(worst, reverse=True)[:8]:
        print(f"  rel {r:.4f} cos {c:.5f} {n}")
    assert not bad, "\n".join(bad[:20])


def test_backward_in_unit_ranges_equals_single_call(lib):
    """vdk_convnext_train_backward_range over the sections the DDP overlap uses == the one-call backward (same kernels in the
    same order; only atomics' summation order may differ), and the sections hand over every parameter exactly once."""
    _, ours = build_pair(seed=11)
    torch.manual_seed(3)
    x = torch.randn(6, 3, 64, 64, device="cuda")
    wout = torch.randn(6, 64, device="cuda")
    for p in ours.parameters():
        p.grad = torch.zeros_like(p)  # pre-allocated fp32 buffers: the kernels accumulate straight into them
    (ours(x) * wout).sum().backward()
    one_call = {n: p.grad.clone() for n, p in ours.named_parameters()}
    for p in ours.parameters():
        p.grad.zero_()
    seen = []
    ours.grad_section_hook = lambda names: seen.extend(names)
    (ours(x) * wout).sum().backward()
    ours.grad_section_hook = None
    assert sorted(seen) == sorted(n for n, _ in ours.named_parameters())
    for n, p in ours.named_parameters():
        a, b = p.grad, one_call[n]
        assert (a - b).abs().max().item() <= 1e-4 * (b.abs().max().item() + 1e-6) + 1e-6, n


def test_train_step_with_head_and_fused_optimizer(lib):
    """One full faceX train step on the H100 kernels: backbone fwd -> ArcFace+CE -> backward -> clip+SGD+EMA."""
    import copy
    from visiondk_b200.heads import ArcFace, margin_ce_loss
    from visiondk_b200.optim import FusedSGDClipEMA
    oracle, ours = build_pair(seed=9)
    head = ArcFace(64, 40, 0.35, 0.0, 32).cuda()
    model = torch.nn.ModuleDict({"backbone": ours, "head": head})
    ema_model = copy.deepcopy(model).eval()
    opt = FusedSGDClipEMA([{"params": ours.parameters(), "lr": 0.01}, {"params": head.parameters(), "lr": 0.1}], lr=0.01,
                          momentum=0.8, weight_decay=5e-4, model=model, ema_model=ema_model)
    torch.manual_seed(2)
    x = torch.randn(8, 3, 64, 64, device="cuda")
    y = torch.randint(0, 40, (8,), device="cuda")
    losses = []
    for _ in range(5):
        feats = ours(x)
        loss = margin_ce_loss(head, feats, y, 0.1)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(torch.isfinite(torch.tensor(losses))), losses
    assert losses[-1] < losses[0], f"loss did not decrease on a repeated batch: {losses}"
