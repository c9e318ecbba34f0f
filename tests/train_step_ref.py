"""fp64 references and bounds of the pieces that join the train step's kernels (csrc/convnext_train.cu, the training half of
csrc/vit.cu, and the small kernels only they call), for tests/test_train_step_units_gpu.py.

Every reference takes the kernel's own saved inputs from the train workspace.  The GEMM, depthwise, LayerNorm-backward,
BatchNorm and attention bounds are kernel_ref.py's; the ones derived here are the weight-gradient GEMM in its split-K slab
form with the fixed-order reduction, the LayerNorm forward of launch_ln_patchify, and layerscale_finalize.  The fixed-order
fp32 kernels (patchify, assemble, slab and column sums, casts, un-permutations) are reproduced bit for bit instead.
"""
import math

import torch

from kernel_ref import A32, U32, ulp

SLAB_GROUPS = 8   # slab_reduce_kernel: 8 strided slab groups per column, then the 8 group sums in order


def wgrad_splits(M, N, K, sm, lib):
    """train_gemm.h wgrad_splits: the split count of a weight-gradient GEMM D[M, N] over a contraction of K rows."""
    tiles = -(-M // 128) * -(-N // 256)
    return lib.vdk_gemm_effective_splits(K, max(2, (2 * sm) // max(1, tiles)))


def split_ranges(K, n_split):
    """The contraction rows [k0, k1) of each split (gemm.cu: 64-row K blocks, ceil-divided over the splits)."""
    per = -(-(-(-K // 64)) // n_split)
    return [(s * per * 64, min((s + 1) * per * 64, K)) for s in range(n_split)], per


def gemm_wgrad_reference(a, b, init, n_split, bias_init=None):
    """Weight gradient D = init + A^T B of G.wgrad (a [K, M], b [K, N] as stored; init None without accumulation), and the
    bias gradient init_b + sum_k A[k, :] it computes from the same tiles.  Returns (ref, bound, bias_ref, bias_bound).

      dW: every split runs one wgmma chain over at most `per` 64-row K blocks: (4 per + 17) 2^-23 (|A|^T |B|) restricted to
          its rows (the model of DESIGN.md §3), and slab_reduce adds the n_split partials in 8 strided groups
          (ceil(n_split / 8) adds each), the 8 group sums in order (7) and the initial value (1): each of these
          ceil(n_split / 8) + 8 roundings is 2^-24 of a partial sum bounded by |A|^T |B| + |init|.
          The bound is kept per split: a dropped or doubled slab is one partial, ~sqrt(K / n_split) times the operand
          scales, while the bound grows with |A|^T |B| over only `per` blocks.
      bias: a thread adds its rows of one split in order (at most 32 per + 1 terms, test_wgrad_bias_gpu.py), and the
          column-sum slabs go through the same slab_reduce with accumulation: gamma_n (sum |A| + |init|) with
          n = 32 per + 1 + ceil(n_split / 8) + 8."""
    A, Bm = a.double(), b.double()
    K = A.shape[0]
    _, per = split_ranges(K, n_split)
    absprod = A.abs().t() @ Bm.abs()
    ref = A.t() @ Bm
    n_red = -(-n_split // SLAB_GROUPS) + SLAB_GROUPS
    i0 = init.double() if init is not None else torch.zeros_like(ref)
    bound = ((4 * per + 17) * U32 * absprod + n_red * A32 * (absprod + i0.abs())) * 1.001
    n_b = 32 * per + 1 + n_red
    gam = n_b * A32 / (1 - n_b * A32)
    b0 = bias_init.double() if bias_init is not None else torch.zeros_like(A[0])
    return i0 + ref, bound, b0 + A.sum(0), gam * (A.abs().sum(0) + b0.abs()) * 1.001


def colsum_f32_sequential(x, init):
    """col_sum_f32_small and vit_assemble_bwd's batch sum: out = init + (((0 + x[0]) + x[1]) + ...) in fp32, bit for bit."""
    s = torch.zeros_like(x[0], dtype=torch.float32)
    for r in range(x.shape[0]):
        s = s + x[r].float()
    return init + s


def slab_reduce_bias(slabs, bias):
    """slab_reduce_bias_kernel bit for bit: bias, then the slabs in order."""
    v = bias.expand_as(slabs[0]).clone()
    for s in range(slabs.shape[0]):
        v = v + slabs[s]
    return v


def ln_fwd_reference(x, gamma, beta, eps):
    """fp64 LayerNorm over the last dimension of the bf16 rows x [P, C]: y, rstd, and what ln_fwd_bound needs."""
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    d = xd - mu
    r = (d.pow(2).mean(-1) + eps).rsqrt()
    return dict(x=xd, mu=mu, d=d, rstd=r, y=d * r[:, None] * gamma.double() + beta.double())


def ln_fwd_bound(ref, gamma, beta, eps, lpp):
    """Bounds of launch_ln_patchify's output and saved 1/sigma (patch 1 and 2 alike: the 2x2 gather only moves rows); a = 2^-24.

    Kernel order (convnext.cu ln_patchify_kernel, LPP lanes per pixel, it = ceil(C / 8 LPP) 8-vectors per lane): bf16 inputs
    are exact in fp32.
      s: a lane adds its 8 it values in order, then log2(LPP) shuffle adds; mean = s / C: n_s = 8 it + log2(LPP) + 1
         roundings of partial sums bounded by sum |x|:   |mu~ - mu| <= e_mu = n_s a mean|x|
      q = sum (x - mu~)^2: each d = fl(x - mu~) (a |d|), an fma chain of 8 it steps, log2(LPP) shuffles.  With
         Q' = sum (x - mu~)^2 = Q + C (mu~ - mu)^2:   |q~ - Q| <= e_Q = (n_s + 2) a (Q + C e_mu^2) + C e_mu^2
      rstd = rsqrtf(q / C + eps): the divide and the add (2a) and rsqrtf (2^-22):
         relative e_r = e_Q / (2 (Q + C eps)) + 2^-22 + 2a                           -> the saved rstd's bound r e_r
      y = fl(fl(fl(x - mu~) rstd) g + b): |dxhat| <= rstd e_mu + |xhat| e_r, then 4 roundings on |g xhat| + |b| and half a
         bf16 ulp."""
    a = A32
    x, d, r = ref["x"], ref["d"], ref["rstd"]
    C = x.shape[-1]
    it = -(-C // (8 * lpp))
    n_s = 8 * it + int(math.log2(lpp)) + 1
    e_mu = n_s * a * x.abs().mean(-1, keepdim=True)
    Q = d.pow(2).sum(-1)
    eQ = (n_s + 2) * a * (Q + C * e_mu[:, 0] ** 2) + C * e_mu[:, 0] ** 2
    e_r = (eQ / (2 * (Q + C * eps)) + 2.0 ** -22 + 2 * a) * 1.01
    xhat = d * r[:, None]
    g = gamma.double().abs()
    e32 = (g * (r[:, None] * e_mu + xhat.abs() * e_r[:, None]) + 4 * a * (g * xhat.abs() + beta.double().abs())) * 1.01
    return e32 + 0.5 * ulp(ref["y"].abs() + e32, torch.bfloat16), r * e_r


def ln_lpp(C):
    """launch_ln_patchify's lanes per pixel."""
    return 8 if C // 8 <= 8 else (16 if C // 8 <= 16 else 32)


def layerscale_finalize_reference(G, W2, b2, gamma, sdo, dW2_init, dg_init, db2_init):
    """layerscale_finalize_kernel on the kernel's own G [C, K4] and sdo [C]; returns [(ref, bound)] for dW2, dgamma, db2.

      dW2 += gamma G: the product and the add are one or two fp32 roundings (two unless the compiler contracts them into an
          fma): 2 a (|gamma G| + |ref|).
      dgamma += sum_k G W2 + b2 sdo: a thread runs an fmaf chain of K4 / 256 steps, a 5-level warp tree, thread 0 adds the 8
          warp sums in order, then b2 sdo (product and add) and the += : n = K4 / 256 + 5 + 8 + 3 roundings, each of a
          partial sum bounded by sum_k |G W2| + |b2 sdo| + |init|: gamma_n times that.
      db2 += gamma sdo: 2 a (|gamma sdo| + |ref|)."""
    a = A32
    Gd, W2d, gm = G.double(), W2.double(), gamma.double()
    K4 = Gd.shape[1]
    dW2 = dW2_init.double() + gm[:, None] * Gd
    dW2_b = 2 * a * ((gm[:, None] * Gd).abs() + dW2.abs()) * 1.001
    n = K4 // 256 + 5 + 8 + 3
    gam = n * a / (1 - n * a)
    bs = b2.double() * sdo.double()
    dg = dg_init.double() + (Gd * W2d).sum(1) + bs
    dg_b = gam * ((Gd * W2d).abs().sum(1) + bs.abs() + dg_init.double().abs()) * 1.001
    db = db2_init.double() + gm * sdo.double()
    db_b = 2 * a * ((gm * sdo.double()).abs() + db.abs()) * 1.001
    return (dW2, dW2_b), (dg, dg_b), (db, db_b)
