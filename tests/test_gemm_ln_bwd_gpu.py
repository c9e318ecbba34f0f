"""The LayerNorm-backward epilogue of the wgmma dgrad GEMM (vdk_gemm with VDK_EPI_LN_BWD, csrc/gemm.cu) against fp64 and
against vdk_layernorm_bwd on the same bf16 dy, under layernorm_bwd_bound (kernel_ref.py) with the fused kernel's summation
depths.  Cases: every ConvNeXt-B width (blocks at C = 128 / 256 / 512 / 1024, downsample patch rows at Cin = 128 / 256 /
512; 512 and 1024 span 2 / 4 tiles and run as clusters), ragged M, more than three tiles per persistent CTA, gamma = 0
channels and |beta / gamma| up to 30.  Group widths the kernel has no form for are rejected."""
import ctypes as C

import pytest
import torch

from kernel_ref import (bf16_store_bound, check_within, fused_launch, layernorm_bwd_bound, layernorm_bwd_dgamma,
                        layernorm_bwd_reference, ln_bwd_launch)
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu
STATS = {}


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gemm_desc(A, Bw, D, M, N, K, epi, **kw):
    return _lib.GemmDesc(A=A.data_ptr(), B=Bw.data_ptr(), D=D.data_ptr(), M=M, N=N, K=K, lda=K, ldb=N, ldd=N,
                         in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_BF16, epilogue=epi, split_k=1, trans_b=1, **kw)


def ln_problem(P, G, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(P, G, device="cuda", dtype=torch.float64, generator=gen) * 2 + 0.3
    mean = x.mean(-1, keepdim=True)
    rstd64 = ((x - mean).pow(2).mean(-1) + 1e-6).rsqrt()
    xhat = (x - mean) * rstd64[:, None]
    sign = torch.where(torch.rand(G, device="cuda", generator=gen) < 0.5, -1.0, 1.0)
    gamma = (sign * (0.2 + 1.3 * torch.rand(G, device="cuda", generator=gen))).float()
    beta = 0.2 * torch.randn(G, device="cuda", generator=gen)
    far = torch.arange(G, device="cuda") % 8 == 3
    beta[far] = (gamma[far] * 30 * (2 * torch.rand(int(far.sum()), device="cuda", generator=gen) - 1)).float()
    gamma[5] = 0.0
    beta[5] = 0.1
    gamma[77] = 0.0
    y = (gamma.double() * xhat + beta.double()).to(torch.float32).to(torch.bfloat16)
    return gen, xhat, rstd64, gamma, beta, y


# (B, H, W, G, patch): H x W is the LayerNorm's image; patch 2: the GEMM rows are its 2x2 patches (N = 4 G)
CASES = [
    (21, 56, 56, 128, 1),   # ConvNeXt-B stage 0 blocks: M = 65856 (ragged), 4 tiles per CTA
    (85, 28, 28, 256, 1),   # stage 1 blocks: M = 66640
    (41, 56, 56, 128, 2),   # downsample into stage 1: Cin = 128, two groups per 256-column tile
    (83, 28, 40, 256, 2),   # downsample into stage 2: Cin = 256, one group per tile, non-square image
    (130, 14, 14, 512, 1),  # stage 2 blocks: clusters of 2, M = 25480
    (260, 7, 7, 1024, 1),   # stage 3 blocks: clusters of 4, M = 12740
    (131, 14, 14, 512, 2),  # downsample into stage 3: Cin = 512, clusters of 2 over 8 column tiles, M = 6419
]


def to_patch(t, B, H, W, G):
    return t.view(B, H // 2, 2, W // 2, 2, G).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * G).contiguous()


@pytest.mark.parametrize("B,H,W,G,patch", CASES)
def test_gemm_ln_bwd(lib, B, H, W, G, patch):
    sm = sm_count()
    P = B * H * W
    M = P // (patch * patch)
    N = G * patch * patch
    K = 4 * G
    L = fused_launch(M, N, G, sm)
    assert L["per_cta"] > 3 and M % 128 != 0, (L, M)
    gen, xhat, rstd64, gamma, beta, y = ln_problem(P, G, seed=G * 7 + patch)
    rstd = rstd64.float()
    A = (torch.randn(M, K, device="cuda", generator=gen)).to(torch.bfloat16)
    Bw = (torch.randn(K, N, device="cuda", generator=gen) * K ** -0.5).to(torch.bfloat16)
    y_k = to_patch(y, B, H, W, G) if patch == 2 else y
    dg_init = torch.randn(G, device="cuda", generator=gen)
    db_init = torch.randn(G, device="cuda", generator=gen)

    # dy = bf16(A . B^T) from the plain GEMM, and vdk_layernorm_bwd on it
    dy_k = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    _lib.check(lib.vdk_gemm(C.byref(gemm_desc(A, Bw, dy_k, M, N, K, _lib.EPI_NONE)), _lib.stream_ptr()), "gemm")
    dx_sep = torch.empty(P, G, device="cuda", dtype=torch.bfloat16)
    dg_sep, db_sep = dg_init.clone(), db_init.clone()
    _lib.check(lib.vdk_layernorm_bwd(dy_k.data_ptr(), y_k.data_ptr(), rstd.data_ptr(), B, H, W, G, gamma.data_ptr(), beta.data_ptr(),
                                     patch, dx_sep.data_ptr(), 0, dg_sep.data_ptr(), db_sep.data_ptr(), _lib.stream_ptr()), "ln_bwd")

    slab = torch.empty(2 * N * sm, device="cuda")
    outs = []
    for _ in range(2):
        dx = torch.full((P + 64, G), float("nan"), device="cuda", dtype=torch.bfloat16)  # 64 guard rows
        dg, db = dg_init.clone(), db_init.clone()
        g = gemm_desc(A, Bw, dx, M, N, K, _lib.EPI_LN_BWD, gamma=gamma.data_ptr(), beta=beta.data_ptr(), residual=y_k.data_ptr(),
                      ldr=N, ln_rstd=rstd.data_ptr(), ln_dgamma=dg.data_ptr(), ln_dbeta=db.data_ptr(), ln_slab=slab.data_ptr(),
                      ln_group=G, ln_wo=W // 2 if patch == 2 else 0)
        _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "gemm ln_bwd")
        outs.append((dx, dg, db))
    torch.cuda.synchronize()
    dx, dg, db = outs[0]
    assert torch.isnan(dx[P:].float()).all(), "write past the last pixel"
    dx = dx[:P]
    assert torch.equal(dg, outs[1][1]) and torch.equal(db, outs[1][2]), "dgamma / dbeta differ between two runs"
    assert torch.equal(dx, outs[1][0][:P])

    dy = dy_k.view(B, H // 2, W // 2, 2, 2, G).permute(0, 1, 3, 2, 4, 5).reshape(P, G) if patch == 2 else dy_k
    dx_ref, _, db_ref, m1, m2 = layernorm_bwd_reference(xhat, rstd64, gamma, dy, None, patch)
    keep = gamma != 0
    for name, launch, (o_dx, o_dg, o_db) in (("fused", L, (dx, dg, db)), ("ln_bwd", ln_bwd_launch(P, G, sm), (dx_sep, dg_sep, db_sep))):
        e32, _, db_b = layernorm_bwd_bound(xhat, rstd64, gamma, beta, y, dy, None, m1, m2, launch, dg_init, db_init)
        tag = f"{name} G={G} patch={patch} M={M}"
        check_within(o_dx, dx_ref, bf16_store_bound(dx_ref, e32), tag + " dx",
                     lambda bad: f"pixels {bad.any(-1).nonzero().flatten()[:8].tolist()}", STATS)
        dg_ref, dg_b = layernorm_bwd_dgamma(y, beta, gamma, dy, launch, dg_init)
        check_within(o_dg[keep], dg_ref[keep], dg_b[keep], tag + " dgamma",
                     lambda bad: f"channels {keep.nonzero().flatten()[bad.nonzero().flatten()][:8].tolist()}", STATS)
        assert float(o_dg[5]) == float(dg_init[5]) and float(o_dg[77]) == float(dg_init[77])
        check_within(o_db, db_init.double() + db_ref, db_b, tag + " dbeta",
                     lambda bad: f"channels {bad.nonzero().flatten()[:8].tolist()}", STATS)
        if name == "fused":
            fused_b = bf16_store_bound(dx_ref, e32)
        else:  # the two kernels agree within the sum of their bounds
            both = fused_b + bf16_store_bound(dx_ref, e32)
            check_within(dx, dx_sep.double(), both, tag + " fused vs ln_bwd dx", lambda bad: "", STATS)


@pytest.mark.parametrize("G,patch", [(64, 1), (384, 1), (2048, 1), (64, 2)])
def test_gemm_ln_bwd_rejects_unsupported_groups(lib, G, patch):
    M, N = 256, G * patch * patch
    A = torch.zeros(M, 64, device="cuda", dtype=torch.bfloat16)
    Bw = torch.zeros(64, N, device="cuda", dtype=torch.bfloat16)
    D = torch.zeros(M * patch * patch, G, device="cuda", dtype=torch.bfloat16)
    v = torch.zeros(max(G, 256), device="cuda")
    slab = torch.zeros(2 * N * sm_count(), device="cuda")
    g = gemm_desc(A, Bw, D, M, N, 64, _lib.EPI_LN_BWD, gamma=v.data_ptr(), beta=v.data_ptr(), residual=D.data_ptr(), ldr=N,
                  ln_rstd=v.data_ptr(), ln_dgamma=v.data_ptr(), ln_dbeta=v.data_ptr(), ln_slab=slab.data_ptr(), ln_group=G,
                  ln_wo=16 if patch == 2 else 0)
    assert lib.vdk_gemm(C.byref(g), _lib.stream_ptr()) == _lib.VDK_ERR_INVALID
