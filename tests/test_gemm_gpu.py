"""GPU parity of vdk_gemm (wgmma/TMA GEMM) and its epilogues against an fp64 reference of the same 16-bit inputs.

Bounds are elementwise.  The fp32 accumulation follows the model of DESIGN.md §3: a K-long dot product on wgmma is off by at
most (ceil(K/16) + 17) 2^-23 (|A| |B|^T)_mn.  Each fp32 operation of the epilogue adds one rounding (2^-24 relative to its
result), the 16-bit output one ulp of the output type at |ref|, and the activations their documented approximation error.

The kernel is persistent (min(tiles, SM count) CTAs, each looping over tiles 128 x BN), so the regime cases size M from the
device's SM count to give every CTA at least three tiles, and one case exactly SM + 1 tiles.  Outputs sit in NaN-guarded
buffers (padding columns for ldd > N, trailing rows, a tail); a failure names the wrong tiles and the CTA that ran them.
"""
import ctypes as C

import pytest
import torch

from kernel_ref import (GELU_GRAD_ERR, GELU_REL_ERR, Guarded, check_within, epilogue_reference, gelu64, gelu_grad64,
                        split_k_bound, ulp)
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu

DT = {"bf16": (torch.bfloat16, _lib.DTYPE_BF16), "fp16": (torch.float16, _lib.DTYPE_FP16),
      "fp32": (torch.float32, _lib.DTYPE_FP32)}
CODE = {torch.bfloat16: _lib.DTYPE_BF16, torch.float16: _lib.DTYPE_FP16, torch.float32: _lib.DTYPE_FP32}

def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tile_n(N, epilogue):
    wide = N % 256 == 0 or N > 512
    if epilogue == _lib.EPI_LAYERNORM:
        wide = N > 128
    return 256 if wide else 128


def describe_tiles(M, N, BN):
    """bad [M, N] -> the (tile row, tile column) tiles holding failures, the CTAs that ran them (tile % grid) and how many
    wrong tiles each round of the persistent loop (tile // grid) had."""
    num_n = -(-N // BN)
    tiles = -(-M // 128) * num_n
    grid = min(tiles, sm_count())

    def describe(bad):
        idx = bad.nonzero()
        t = torch.unique((idx[:, 0] // 128) * num_n + idx[:, 1] // BN)
        return (f"{t.numel()}/{tiles} tiles wrong (BN {BN}, grid {grid}); wrong tiles per CTA round "
                f"{torch.bincount(t // grid).tolist()}; first (tile row, tile col, CTA) "
                f"{[(int(x) // num_n, int(x) % num_n, int(x) % grid) for x in t[:6]]}; first element {idx[0].tolist()}")
    return describe


def run(a, b, out_dtype, epilogue=_lib.EPI_NONE, bias=None, gamma=None, beta=None, residual=None, ldr_pad=0, ldd_pad=0,
        aux=False, ta=0, tb=0, ln_eps=1e-6, in_place=False):
    """vdk_gemm of logical a [M, K] and b [N, K] (stored transposed when ta / tb) into a guarded D [M, N] with pitch
    N + ldd_pad.  `residual` holds the values of the residual (SCALE_RESIDUAL) or saved pre-activation (MUL_GELU_GRAD): copied
    into D itself when in_place, else into a guarded [M, N] buffer of pitch N + ldr_pad.  Returns (D, aux or None)."""
    lib = _lib.load()
    M, K = a.shape
    N = b.shape[0]
    a_st = a.t().contiguous() if ta else a
    b_st = b.t().contiguous() if tb else b
    d = Guarded(M, N, N + ldd_pad, out_dtype)
    res, ldr = None, 0
    if residual is not None:
        if in_place:
            d.fill_(residual)
            res, ldr = d, N + ldd_pad
        else:
            res, ldr = Guarded(M, N, N + ldr_pad, residual.dtype).fill_(residual), N + ldr_pad
    ax = Guarded(M, N, N + ldd_pad, out_dtype) if aux else None
    g = _lib.GemmDesc(A=a_st.data_ptr(), B=b_st.data_ptr(), D=d.ptr(), M=M, N=N, K=K, lda=a_st.stride(0), ldb=b_st.stride(0),
                      ldd=N + ldd_pad, in_dtype=CODE[a.dtype], out_dtype=CODE[out_dtype], epilogue=epilogue,
                      bias=_lib.ptr(bias), gamma=_lib.ptr(gamma), beta=_lib.ptr(beta), residual=res.ptr() if res else 0,
                      ldr=ldr, ln_eps=ln_eps, split_k=1, split_stride=0, aux_out=ax.ptr() if ax else 0, trans_a=ta, trans_b=tb)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    for name, buf in (("D", d), ("aux", ax), ("residual", res if res is not d else None)):
        if buf is not None:
            assert not buf.guard_errors(), f"{name}: {buf.guard_errors()}"
    return d, ax


def check_epilogue(a, b, out_dtype, epilogue, d, ax, bias=None, gamma=None, beta=None, residual=None, ln_eps=1e-6, name=""):
    """Compares D (and the saved pre-activation) with the fp64 epilogue of the exact accumulator, within
    kernel_ref.epilogue_reference's bounds."""
    M, N = d.view.shape
    describe = describe_tiles(M, N, tile_n(N, epilogue))
    r = epilogue_reference(a, b, epilogue, out_dtype, bias=bias, gamma=gamma, beta=beta, residual=residual,
                           aux=ax.view if ax is not None else None, ln_eps=ln_eps)
    if ax is not None:
        check_within(ax.view, r["aux_ref"], r["aux_bound"], f"{name} aux", describe)
    got = d.view.double()
    check_within(got, r["ref"], r["bound"], f"{name} D", describe)
    return got, r["ref"]


def operands(M, N, K, in_dtype, seed, a_scale=1.0, b_scale=1.0):
    torch.manual_seed(seed)
    dt = DT[in_dtype][0]
    a = (a_scale * torch.randn(M, K, device="cuda")).to(dt)
    b = (b_scale * torch.randn(N, K, device="cuda")).to(dt)
    return a, b


# ------------------------------------------------------------------------------------------------------------------------------
# plain products (shapes of the original suite) on the fp64 reference


@pytest.mark.parametrize("in_dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 256, 64), (128, 128, 256), (256, 512, 128),
                                   (1000, 384, 200), (300, 1000, 512), (4096, 512, 128), (77, 8, 8),
                                   (20000, 1024, 256)])
def test_gemm_plain_fp32_out(lib, in_dtype, M, N, K):
    a, b = operands(M, N, K, in_dtype, M * 7 + N * 3 + K)
    d, _ = run(a, b, torch.float32)
    check_epilogue(a, b, torch.float32, _lib.EPI_NONE, d, None, name="plain")


def test_gemm_exact_small_integers(lib):
    # integer-valued operands: every product and partial sum is exact, so the result must be bit-exact
    torch.manual_seed(0)
    a = torch.randint(-4, 5, (256, 192), device="cuda").to(torch.bfloat16)
    b = torch.randint(-4, 5, (384, 192), device="cuda").to(torch.bfloat16)
    d, _ = run(a, b, torch.float32)
    assert torch.equal(d.view.double(), a.double() @ b.double().t())


def test_gemm_strided_operands(lib):
    torch.manual_seed(1)
    abuf = torch.randn(500, 320, device="cuda").to(torch.bfloat16)
    bbuf = torch.randn(264, 448, device="cuda").to(torch.bfloat16)
    a, b = abuf[:, :256], bbuf[:, 64:320]  # pitches 320 / 448, 16-byte aligned starts
    d, _ = run(a, b, torch.float32)
    check_epilogue(a, b, torch.float32, _lib.EPI_NONE, d, None, name="strided")


@pytest.mark.parametrize("out_dtype", ["bf16", "fp32"])
def test_gemm_bias_gelu(lib, out_dtype):
    a, b = operands(1568, 512, 128, "bf16", 2, 0.5, 0.2)
    bias = torch.randn(512, device="cuda")
    d, _ = run(a, b, DT[out_dtype][0], _lib.EPI_GELU, bias=bias)
    check_epilogue(a, b, DT[out_dtype][0], _lib.EPI_GELU, d, None, bias=bias, name="bias_gelu")


@pytest.mark.parametrize("out_dtype", ["bf16", "fp32"])
def test_gemm_layerscale_residual(lib, out_dtype):
    a, b = operands(784, 256, 1024, "bf16", 3, 0.3, 0.1)
    bias = torch.randn(256, device="cuda")
    gamma = torch.rand(256, device="cuda")
    res = torch.randn(784, 256, device="cuda").to(DT[out_dtype][0])
    d, _ = run(a, b, DT[out_dtype][0], _lib.EPI_SCALE_RESIDUAL, bias=bias, gamma=gamma, residual=res)
    check_epilogue(a, b, DT[out_dtype][0], _lib.EPI_SCALE_RESIDUAL, d, None, bias=bias, gamma=gamma, residual=res,
                   name="layerscale")


def test_gemm_rejects_bad_arguments(lib):
    a = torch.zeros(8, 8, device="cuda", dtype=torch.bfloat16)
    d = torch.zeros(8, 8, device="cuda")
    rc = lib.vdk_gemm_tn(a.data_ptr(), a.data_ptr(), d.data_ptr(), 8, 7, 8, 8, 8, 8, 0, 2, 0, 0, 0, 0, 0, 0)
    assert rc == _lib.VDK_ERR_INVALID and "multiple of 8" in _lib.last_error()


@pytest.mark.parametrize("ta,tb", [(1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 192), (512, 2048, 50176 // 49), (1000, 384, 200), (2048, 512, 3000)])
def test_gemm_transposed_storage(lib, ta, tb, M, N, K):
    """MN-major operands (contraction index slow): the forms the backward GEMMs use (dgrad: trans_b, wgrad: both)."""
    a, b = operands(M, N, K, "bf16", M + N + K + ta * 2 + tb)
    d, _ = run(a, b, torch.float32, ta=ta, tb=tb)
    check_epilogue(a, b, torch.float32, _lib.EPI_NONE, d, None, name="transposed")


def test_gemm_wgrad_form_split_k(lib):
    """dW[N_out, K_in] = dY^T . X with the token index (M = 50k) as the contraction: both operands MN-major, split-K."""
    torch.manual_seed(9)
    tokens, n_out, k_in = 50176, 512, 256
    dy = (0.1 * torch.randn(tokens, n_out, device="cuda")).to(torch.bfloat16)
    x = torch.randn(tokens, k_in, device="cuda").to(torch.bfloat16)
    d = torch.zeros(n_out, k_in, device="cuda")
    g = _lib.GemmDesc(A=dy.data_ptr(), B=x.data_ptr(), D=d.data_ptr(), M=n_out, N=k_in, K=tokens, lda=n_out, ldb=k_in,
                      ldd=k_in, in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0,
                      beta=0, residual=0, ldr=0, ln_eps=0.0, split_k=37, trans_a=1, trans_b=1)
    _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
    torch.cuda.synchronize()
    ref, bound = split_k_bound(dy.t(), x.t(), lib.vdk_gemm_effective_splits(tokens, 37))
    check_within(d, ref, bound, "split-K atomics", describe_tiles(n_out, k_in, tile_n(k_in, _lib.EPI_NONE)))


def test_gemm_split_k_slabs_are_deterministic(lib):
    """split_stride > 0: every split writes its own slab (no atomics); the slab sum is bitwise reproducible."""
    torch.manual_seed(4)
    M, N, K = 200, 512, 12544
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (0.05 * torch.randn(N, K, device="cuda")).to(torch.bfloat16)
    n_split = lib.vdk_gemm_effective_splits(K, 40)
    outs = []
    for _ in range(2):
        d = torch.full((n_split, M, N), float("nan"), device="cuda")
        g = _lib.GemmDesc(A=a.data_ptr(), B=w.data_ptr(), D=d.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldd=N,
                          in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_FP32, epilogue=_lib.EPI_NONE, bias=0, gamma=0, beta=0,
                          residual=0, ldr=0, ln_eps=0.0, split_k=40, split_stride=M * N, trans_a=0, trans_b=0)
        _lib.check(lib.vdk_gemm(C.byref(g), _lib.stream_ptr()), "vdk_gemm")
        torch.cuda.synchronize()
        assert torch.isfinite(d).all()
        outs.append(d.sum(0))
    assert torch.equal(outs[0], outs[1])
    ref, bound = split_k_bound(a, w, n_split)
    check_within(outs[0], ref, bound, "split-K slabs", describe_tiles(M, N, tile_n(N, _lib.EPI_NONE)))


# ------------------------------------------------------------------------------------------------------------------------------
# every epilogue in the persistent regime: >= 3 tiles per CTA, both tile widths, ragged M and ragged last 64-column chunk,
# fp16 inputs, every output type an epilogue accepts, ldd / ldr > N, the transposed operand forms

E = _lib
# (id, in, out, epilogue, N, K, options); M is derived from the SM count (ragged: 37 rows short of a full tile row)
REGIME = [
    ("none_bias_bf16_fp32_N512", "bf16", "fp32", E.EPI_NONE, 512, 96, dict(bias=True, ldd_pad=8)),
    ("none_bias_fp16_fp16_N200", "fp16", "fp16", E.EPI_NONE, 200, 80, dict(bias=True, ldd_pad=24)),
    ("none_bf16_bf16_N520_ta", "bf16", "bf16", E.EPI_NONE, 520, 136, dict(ta=1)),
    ("none_bf16_fp32_N512_tb", "bf16", "fp32", E.EPI_NONE, 512, 200, dict(tb=1)),
    ("none_bf16_fp32_N136_ta_tb", "bf16", "fp32", E.EPI_NONE, 136, 72, dict(ta=1, tb=1, ldd_pad=4)),
    ("gelu_bf16_bf16_N520", "bf16", "bf16", E.EPI_GELU, 520, 64, dict(bias=True)),
    ("gelu_fp16_fp32_N136", "fp16", "fp32", E.EPI_GELU, 136, 96, dict(bias=True, ldd_pad=4)),
    ("gelu_fp16_fp16_N200", "fp16", "fp16", E.EPI_GELU, 200, 64, dict(bias=True)),
    ("gelu_aux_bf16_bf16_N512", "bf16", "bf16", E.EPI_GELU, 512, 64, dict(bias=True, aux=True, ldd_pad=16)),
    ("gelu_aux_fp16_fp16_N200", "fp16", "fp16", E.EPI_GELU, 200, 128, dict(bias=True, aux=True)),
    ("scale_res_inplace_bf16_bf16_N512", "bf16", "bf16", E.EPI_SCALE_RESIDUAL, 512, 64, dict(bias=True, in_place=True, ldd_pad=8)),
    ("scale_res_inplace_fp16_fp16_N136", "fp16", "fp16", E.EPI_SCALE_RESIDUAL, 136, 64, dict(bias=True, in_place=True)),
    ("scale_res_bf16_fp32_N200", "bf16", "fp32", E.EPI_SCALE_RESIDUAL, 200, 96, dict(bias=True, ldr_pad=12, ldd_pad=4)),
    ("scale_res_fp16_fp16_N520", "fp16", "fp16", E.EPI_SCALE_RESIDUAL, 520, 64, dict(bias=True, ldr_pad=8)),
    ("layernorm_bf16_bf16_N200", "bf16", "bf16", E.EPI_LAYERNORM, 200, 64, dict(bias=True, ldd_pad=8)),
    ("layernorm_fp16_fp32_N136", "fp16", "fp32", E.EPI_LAYERNORM, 136, 96, dict(bias=True)),
    ("layernorm_bf16_fp16_N8", "bf16", "fp16", E.EPI_LAYERNORM, 8, 64, dict(bias=True)),
    ("layernorm_bf16_bf16_N256", "bf16", "bf16", E.EPI_LAYERNORM, 256, 64, dict()),
    ("gelu_grad_bf16_bf16_N512_tb", "bf16", "bf16", E.EPI_MUL_GELU_GRAD, 512, 64, dict(tb=1, ldr_pad=8)),
    ("gelu_grad_fp16_fp16_N200", "fp16", "fp16", E.EPI_MUL_GELU_GRAD, 200, 96, dict(ldr_pad=8, ldd_pad=8)),
    ("gelu_grad_bf16_fp16_N136_tb", "bf16", "fp16", E.EPI_MUL_GELU_GRAD, 136, 64, dict(tb=1)),
]


def regime_case(case_id, in_dtype, out_dtype, epilogue, N, K, opts, tiles_per_cta=3, exact_tiles=None):
    sm = sm_count()
    BN = tile_n(N, epilogue)
    num_n = -(-N // BN)
    if exact_tiles is not None:
        row_tiles = -(-exact_tiles // num_n)
        assert row_tiles * num_n == exact_tiles
    else:
        row_tiles = -(-tiles_per_cta * sm // num_n) + 1
    M = row_tiles * 128 - 40 if opts.get("ta") else row_tiles * 128 - 37  # trans_a needs M % 8 == 0
    tiles = row_tiles * num_n
    if exact_tiles is None:
        assert tiles >= tiles_per_cta * sm, (tiles, sm)
    seed = sum(map(ord, case_id))
    a, b = operands(M, N, K, in_dtype, seed, 0.5, 0.25)
    odt = DT[out_dtype][0]
    dev = "cuda"
    bias = torch.randn(N, device=dev) if opts.get("bias") else None
    gamma = beta = residual = None
    if epilogue == E.EPI_SCALE_RESIDUAL:
        gamma = torch.rand(N, device=dev) * 2 - 0.5
        residual = torch.randn(M, N, device=dev).to(odt)
    elif epilogue == E.EPI_LAYERNORM:
        gamma = torch.rand(N, device=dev) + 0.5
        beta = torch.randn(N, device=dev)
    elif epilogue == E.EPI_MUL_GELU_GRAD:
        residual = (3 * torch.randn(M, N, device=dev)).to(odt)
    d, ax = run(a, b, odt, epilogue, bias=bias, gamma=gamma, beta=beta, residual=residual, ldr_pad=opts.get("ldr_pad", 0),
                ldd_pad=opts.get("ldd_pad", 0), aux=opts.get("aux", False), ta=opts.get("ta", 0), tb=opts.get("tb", 0),
                in_place=opts.get("in_place", False))
    check_epilogue(a, b, odt, epilogue, d, ax, bias=bias, gamma=gamma, beta=beta, residual=residual, name=case_id)


@pytest.mark.parametrize("case_id,in_dtype,out_dtype,epilogue,N,K,opts", REGIME, ids=[c[0] for c in REGIME])
def test_gemm_epilogue_persistent_regime(lib, case_id, in_dtype, out_dtype, epilogue, N, K, opts):
    regime_case(case_id, in_dtype, out_dtype, epilogue, N, K, opts)


def test_gemm_exactly_one_tile_more_than_sms(lib):
    """SM + 1 tiles of 128 x 128: one CTA runs a second tile, with the saved pre-activation and a bias."""
    regime_case("gelu_aux_sm_plus_1", "bf16", "bf16", E.EPI_GELU, 128, 64, dict(bias=True, aux=True),
                exact_tiles=sm_count() + 1)


# ------------------------------------------------------------------------------------------------------------------------------
# LayerNorm edges


@pytest.mark.parametrize("offset", [0.0, 1e4])
@pytest.mark.parametrize("N,out_dtype", [(8, "bf16"), (136, "fp32"), (200, "bf16"), (256, "fp16")])
def test_gemm_layernorm_constant_rows_and_offset(lib, N, out_dtype, offset):
    """Every third row of A is zero, so its row of acc + bias is the constant bias `offset + 3`: variance 0 and the output is
    beta exactly.  With offset 1e4 the other rows have mean ~1e4 and spread ~1 (the fp32 rounding of x = acc + bias at 1e4 is
    what the bound's 2^-24 |x| term carries).  Multi-tile M (>= 3 tiles per CTA)."""
    sm = sm_count()
    M = (3 * sm + 1) * 128 - 5
    a, b = operands(M, N, 64, "bf16", N, 0.5, 0.25)
    a[::3] = 0
    bias = torch.full((N,), offset + 3.0, device="cuda")
    gamma = torch.rand(N, device="cuda") + 0.5
    beta = torch.randn(N, device="cuda")
    odt = DT[out_dtype][0]
    d, _ = run(a, b, odt, E.EPI_LAYERNORM, bias=bias, gamma=gamma, beta=beta, ldd_pad=8)
    check_epilogue(a, b, odt, E.EPI_LAYERNORM, d, None, bias=bias, gamma=gamma, beta=beta, name=f"layernorm N{N} +{offset}")
    const = d.view[::3]
    assert torch.equal(const, beta.to(odt).expand_as(const)), "rows of zero variance must equal beta"


# ------------------------------------------------------------------------------------------------------------------------------
# activation sweeps: one-hot A rows make the accumulator equal chosen 16-bit values exactly


def finite_values(dtype):
    v = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)
    return v[torch.isfinite(v)]


def one_hot(M, K, dtype):
    a = torch.zeros(M, K, device="cuda", dtype=dtype)
    a[torch.arange(M), torch.arange(M) % K] = 1
    return a


@pytest.mark.parametrize("in_dtype,out_dtype,aux", [("bf16", "fp32", False), ("bf16", "bf16", True),
                                                    ("fp16", "fp16", False), ("fp16", "fp16", True)])
def test_gemm_gelu_sweeps_every_16bit_value(lib, in_dtype, out_dtype, aux):
    """acc[m, n] = B[n, m % 64] runs through every finite value x of the input type.  The epilogue's GELU is within
    GELU_REL_ERR |x| of fp64 erf-GELU plus the output rounding (fp32: 2^-24 |ref|, 16-bit: one ulp); y == x exactly for
    x >= 8 and y == 0 for x <= -8 (tanh saturates to +-1 in fp16, gemm.cu); the saved pre-activation equals x."""
    dt, odt = DT[in_dtype][0], DT[out_dtype][0]
    vals = finite_values(dt)
    K, N = 64, 1024
    b = torch.zeros(N * K, dtype=dt, device="cuda")
    b[:vals.numel()] = vals
    b = b.view(N, K)
    a = one_hot(128, K, dt)
    d, ax = run(a, b, odt, E.EPI_GELU, aux=aux)
    x = (a.double() @ b.double().t())
    if aux:
        assert torch.equal(ax.view.double(), x), "the saved pre-activation must equal the accumulator"
    y = d.view.double()
    ref = gelu64(x)
    rnd = 2.0 ** -24 * ref.abs() if odt == torch.float32 else ulp(ref, odt)
    err = (y - ref).abs()
    measured = float(((err - rnd).clamp_min(0) / x.abs().clamp_min(1e-300)).max())
    print(f"GELU {in_dtype}->{out_dtype}{' aux' if aux else ''}: max (|err| - rounding) / |x| = {measured:.3e}")
    check_within(y, ref, GELU_REL_ERR * x.abs() + rnd, f"gelu sweep {in_dtype}", describe_tiles(128, N, 256))
    assert torch.equal(y[x >= 8], x[x >= 8])
    assert bool((y[x <= -8] == 0).all())


@pytest.mark.parametrize("in_dtype,out_dtype", [("bf16", "bf16"), ("fp16", "fp16"), ("bf16", "fp16")])
def test_gemm_gelu_grad_sweeps_every_16bit_value(lib, in_dtype, out_dtype):
    """acc = 1 everywhere, the saved pre-activation runs through every finite value of the output type (|x| up to 3.4e38 for
    bf16, where fp16 conversion gives inf before the clamp to [-8, 8]): D = gelu~'(x) within GELU_GRAD_ERR of fp64
    d/dx erf-GELU, plus one ulp of the output."""
    dt, odt = DT[in_dtype][0], DT[out_dtype][0]
    vals = finite_values(odt)
    M, N, K = 128, 512, 64
    pre = torch.zeros(M * N, dtype=odt, device="cuda")
    pre[:vals.numel()] = vals
    pre = pre.view(M, N)
    a = one_hot(M, K, dt)
    b = torch.ones(N, K, dtype=dt, device="cuda")
    d, _ = run(a, b, odt, E.EPI_MUL_GELU_GRAD, residual=pre)
    ref = gelu_grad64(pre.double())
    y = d.view.double()
    rnd = ulp(ref, odt)
    measured = float(((y - ref).abs() - rnd).clamp_min(0).max())
    print(f"GELU' {out_dtype}: max |err| - rounding = {measured:.3e}")
    check_within(y, ref, GELU_GRAD_ERR + rnd, f"gelu' sweep {out_dtype}", describe_tiles(M, N, 256))
