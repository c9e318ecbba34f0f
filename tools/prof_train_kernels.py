"""Stand-alone timing of the training step's individual kernels at ConvNeXt-B shapes (not the bench contract).

    python tools/prof_train_kernels.py [stage] [batch] [iters]        # CUDA-event timings, one JSON line per kernel
    ncu --set full ... python tools/prof_train_kernels.py 2 128 1     # the same launches for an ncu capture

Stage s of ConvNeXt-B: (H, C) = (56,128) (28,256) (14,512) (7,1024).  Every GEMM line names its kernel instantiation:
the tile width BN and the trans_a / trans_b operand forms.  Without a stage argument, all four stages run in turn.
"""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from visiondk_b200 import _lib

if len(sys.argv) == 1 or sys.argv[1] == "all":
    import subprocess
    for s in range(4):
        subprocess.run([sys.executable, os.path.abspath(__file__), str(s), *sys.argv[2:]], check=True)
    sys.exit(0)
stage = int(sys.argv[1])
B = int(sys.argv[2]) if len(sys.argv) > 2 else 128
iters = int(sys.argv[3]) if len(sys.argv) > 3 else 10
only = sys.argv[4].split(",") if len(sys.argv) > 4 else None
H = (56, 28, 14, 7)[stage]
Cn = (128, 256, 512, 1024)[stage]
M = B * H * H
lib = _lib.load()
dev = "cuda"
sp = _lib.stream_ptr()


def bf(*shape, scale=1.0):
    return (scale * torch.randn(*shape, device=dev)).to(torch.bfloat16)


x = bf(B, H, H, Cn)
y = torch.empty_like(x)
dy = bf(B, H, H, Cn)
rstd = torch.rand(M, device=dev) + 0.5
w49 = 0.2 * torch.randn(49, Cn, device=dev)
vec = lambda: torch.randn(Cn, device=dev)
bias, ln_w, ln_b = vec(), vec() + 2.0, vec()
dw49 = torch.zeros(49, Cn, device=dev)
dbias, dgamma, dbeta = torch.zeros(Cn, device=dev), torch.zeros(Cn, device=dev), torch.zeros(Cn, device=dev)
hpre = torch.empty(M, 4 * Cn, dtype=torch.bfloat16, device=dev)
hpost = torch.empty(M, 4 * Cn, dtype=torch.bfloat16, device=dev)
w1 = bf(4 * Cn, Cn, scale=0.05)
w2 = bf(Cn, 4 * Cn, scale=0.05)
b1 = torch.randn(4 * Cn, device=dev)
gam = torch.randn(Cn, device=dev)
out = torch.empty_like(x)
slabs = torch.empty(64 * 1024 * 1024 // 4, device=dev)
colsl = torch.empty(1024 * 1024, device=dev)  # per-split column sums of A (the bias gradient) of the "wgrad + bias" lines
# downsample into the next stage: 2x2 / stride-2 patches of the LayerNorm output as a GEMM (tokens M/4, K = 4C, N = 2C)
Md = M // 4
dsw = bf(2 * Cn, 4 * Cn, scale=0.05)
dsb = torch.randn(2 * Cn, device=dev)
dso = torch.empty(Md, 2 * Cn, dtype=torch.bfloat16, device=dev)


def inst(N_, epi=_lib.EPI_NONE, ta=0, tb=0):
    """the kernel instantiation vdk_gemm picks (gemm.cu, gemm_run): tile width and operand forms"""
    wide = N_ > 128 if epi == _lib.EPI_LAYERNORM else (N_ % 256 == 0 or N_ > 512)
    return f"BN{256 if wide else 128} ta{ta} tb{tb}"


def gemm(A, Bm, D, M_, N_, K_, lda, ldb, ldd, epi=_lib.EPI_NONE, bias=0, gamma=0, residual=0, ldr=0, out_dtype=_lib.DTYPE_BF16,
         split=1, stride=0, aux=0, ta=0, tb=0, colsums=0):
    g = _lib.GemmDesc(A=A.data_ptr(), B=Bm.data_ptr(), D=D.data_ptr(), M=M_, N=N_, K=K_, lda=lda, ldb=ldb, ldd=ldd,
                      in_dtype=_lib.DTYPE_BF16, out_dtype=out_dtype, epilogue=epi, bias=bias, gamma=gamma, beta=0, residual=residual,
                      ldr=ldr, ln_eps=1e-6, split_k=split, split_stride=stride, aux_out=aux, trans_a=ta, trans_b=tb,
                      a_col_sums=colsums)
    _lib.check(lib.vdk_gemm(C.byref(g), sp), "gemm")


xf = x.reshape(M, Cn)
dxf = dy.reshape(M, Cn)
tiles = ((Cn + 127) // 128) * ((4 * Cn + 255) // 256)
split = lib.vdk_gemm_effective_splits(M, max(2, 296 // tiles))
tiles1 = ((4 * Cn + 127) // 128) * ((Cn + 255) // 256)
split1 = lib.vdk_gemm_effective_splits(M, max(2, 296 // tiles1))

kernels = {
    "dwconv7_ln fwd": (lambda: _lib.check(lib.vdk_dwconv7(0, x.data_ptr(), B, H, H, Cn, w49.data_ptr(), bias.data_ptr(), ln_w.data_ptr(),
                                                          ln_b.data_ptr(), 1e-6, y.data_ptr(), rstd.data_ptr(), 0, sp), "dw0"),
                       2.0 * M * Cn * 49, 4.0 * M * Cn, None),
    "dwconv7 bwd-data": (lambda: _lib.check(lib.vdk_dwconv7(1, dy.data_ptr(), B, H, H, Cn, w49.data_ptr(), 0, 0, 0, 0.0, y.data_ptr(), 0,
                                                            x.data_ptr(), sp), "dw1"), 2.0 * M * Cn * 49, 6.0 * M * Cn, None),
    "dwconv7 wgrad": (lambda: _lib.check(lib.vdk_dwconv7_wgrad(x.data_ptr(), dy.data_ptr(), B, H, H, Cn, dw49.data_ptr(), dbias.data_ptr(), sp),
                                         "dww"), 2.0 * M * Cn * 49, 4.0 * M * Cn, None),
    # the train step's depthwise backward: both of the above from one pass over the gradient
    "dwconv7 bwd (data + wgrad)": (lambda: _lib.check(lib.vdk_dwconv7_bwd(x.data_ptr(), dy.data_ptr(), B, H, H, Cn, w49.data_ptr(),
                                                                          x.data_ptr(), y.data_ptr(), dw49.data_ptr(), dbias.data_ptr(),
                                                                          sp), "dwb"), 4.0 * M * Cn * 49, 8.0 * M * Cn, None),
    "ln_bwd": (lambda: _lib.check(lib.vdk_layernorm_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr(), B, H, H, Cn, ln_w.data_ptr(),
                                                        ln_b.data_ptr(), 1, y.data_ptr(), 0, dgamma.data_ptr(), dbeta.data_ptr(), sp), "lnb"),
               0.0, 6.0 * M * Cn, None),
    "fc1 fwd (GELU + saved pre-activation)": (lambda: gemm(xf, w1, hpost, M, 4 * Cn, Cn, Cn, Cn, 4 * Cn, _lib.EPI_GELU, b1.data_ptr(),
                                                           aux=hpre.data_ptr()), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 9, inst(4 * Cn, _lib.EPI_GELU)),
    "fc1 fwd (GELU only)": (lambda: gemm(xf, w1, hpost, M, 4 * Cn, Cn, Cn, Cn, 4 * Cn, _lib.EPI_GELU, b1.data_ptr()),
                            8.0 * M * Cn * Cn, 2.0 * M * Cn * 5, inst(4 * Cn, _lib.EPI_GELU)),
    "fc1 fwd (bias only)": (lambda: gemm(xf, w1, hpost, M, 4 * Cn, Cn, Cn, Cn, 4 * Cn, _lib.EPI_NONE, b1.data_ptr()),
                            8.0 * M * Cn * Cn, 2.0 * M * Cn * 5, inst(4 * Cn)),
    "fc1 fwd (no epilogue math)": (lambda: gemm(xf, w1, hpost, M, 4 * Cn, Cn, Cn, Cn, 4 * Cn, _lib.EPI_NONE),
                                   8.0 * M * Cn * Cn, 2.0 * M * Cn * 5, inst(4 * Cn)),
    "fc2 fwd (layer scale + residual)": (lambda: gemm(hpost, w2, out, M, Cn, 4 * Cn, 4 * Cn, 4 * Cn, Cn, _lib.EPI_SCALE_RESIDUAL,
                                                      bias.data_ptr(), gam.data_ptr(), xf.data_ptr(), Cn), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 6, inst(Cn, _lib.EPI_SCALE_RESIDUAL)),
    "fc2 dgrad (x gelu')": (lambda: gemm(dxf, w2, hpost, M, 4 * Cn, Cn, Cn, 4 * Cn, 4 * Cn, _lib.EPI_MUL_GELU_GRAD, residual=hpre.data_ptr(),
                                         ldr=4 * Cn, tb=1), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 9,
                             inst(4 * Cn, _lib.EPI_MUL_GELU_GRAD, tb=1)),
    "fc1 dgrad": (lambda: gemm(hpost, w1, y.reshape(M, Cn), M, Cn, 4 * Cn, 4 * Cn, Cn, Cn, tb=1), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 5, inst(Cn, tb=1)),
    "fc2 wgrad (slabs)": (lambda: gemm(dxf, hpost, slabs, Cn, 4 * Cn, M, Cn, 4 * Cn, 4 * Cn, out_dtype=_lib.DTYPE_FP32, split=split,
                                       stride=Cn * 4 * Cn, ta=1, tb=1), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 5, inst(4 * Cn, ta=1, tb=1)),
    "fc1 wgrad (slabs)": (lambda: gemm(hpost, xf, slabs, 4 * Cn, Cn, M, 4 * Cn, Cn, Cn, out_dtype=_lib.DTYPE_FP32, split=split1,
                                       stride=4 * Cn * Cn, ta=1, tb=1), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 5, inst(Cn, ta=1, tb=1)),
    "fc2 wgrad + bias (slabs)": (lambda: gemm(dxf, hpost, slabs, Cn, 4 * Cn, M, Cn, 4 * Cn, 4 * Cn, out_dtype=_lib.DTYPE_FP32, split=split,
                                              stride=Cn * 4 * Cn, ta=1, tb=1, colsums=colsl.data_ptr()), 8.0 * M * Cn * Cn,
                                 2.0 * M * Cn * 5, inst(4 * Cn, ta=1, tb=1)),
    "fc1 wgrad + bias (slabs)": (lambda: gemm(hpost, xf, slabs, 4 * Cn, Cn, M, 4 * Cn, Cn, Cn, out_dtype=_lib.DTYPE_FP32, split=split1,
                                              stride=4 * Cn * Cn, ta=1, tb=1, colsums=colsl.data_ptr()), 8.0 * M * Cn * Cn,
                                 2.0 * M * Cn * 5, inst(Cn, ta=1, tb=1)),
}
if stage < 3:
    kernels["downsample (bias)"] = (lambda: gemm(x.reshape(Md, 4 * Cn), dsw, dso, Md, 2 * Cn, 4 * Cn, 4 * Cn, 4 * Cn, 2 * Cn,
                                                 bias=dsb.data_ptr()), 2.0 * Md * 2 * Cn * 4 * Cn,
                                    2.0 * (Md * 4 * Cn + 8 * Cn * Cn + Md * 2 * Cn), inst(2 * Cn))
    # its backward: dgrad into the 2x2 patch rows, then the LayerNorm backward over them (ln_bwd patch mode 2)
    dsdy = bf(Md, 2 * Cn)
    kernels["downsample dgrad"] = (lambda: gemm(dsdy, dsw, x.reshape(Md, 4 * Cn), Md, 4 * Cn, 2 * Cn, 2 * Cn, 4 * Cn, 4 * Cn, tb=1),
                                   2.0 * Md * 2 * Cn * 4 * Cn, 2.0 * (Md * 2 * Cn + 8 * Cn * Cn + Md * 4 * Cn), inst(4 * Cn, tb=1))
    kernels["ln_bwd (2x2 patch rows)"] = (lambda: _lib.check(lib.vdk_layernorm_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr(), B, H, H, Cn,
                                                                                  ln_w.data_ptr(), ln_b.data_ptr(), 2, y.data_ptr(), 0,
                                                                                  dgamma.data_ptr(), dbeta.data_ptr(), sp), "lnb2"),
                                          0.0, 6.0 * M * Cn, None)

# the LayerNorm backward in the epilogue of the dgrad GEMM that produces its input gradient (VDK_EPI_LN_BWD): against the
# sum of "fc1 dgrad" + "ln_bwd" and of "downsample dgrad" + "ln_bwd (2x2 patch rows)" (C = 512 / 1024: clusters of 2 / 4)
if Cn in (128, 256, 512, 1024):
    def ln_fused(A, Bw, N_, K_, wo):
        g = _lib.GemmDesc(A=A.data_ptr(), B=Bw.data_ptr(), D=out.data_ptr(), M=A.shape[0], N=N_, K=K_, lda=K_, ldb=N_, ldd=N_,
                          in_dtype=_lib.DTYPE_BF16, out_dtype=_lib.DTYPE_BF16, epilogue=_lib.EPI_LN_BWD, gamma=ln_w.data_ptr(),
                          beta=ln_b.data_ptr(), residual=x.data_ptr(), ldr=N_, split_k=1, trans_b=1, ln_rstd=rstd.data_ptr(),
                          ln_dgamma=dgamma.data_ptr(), ln_dbeta=dbeta.data_ptr(), ln_slab=slabs.data_ptr(), ln_group=Cn, ln_wo=wo)
        _lib.check(lib.vdk_gemm(C.byref(g), sp), "gemm ln_bwd")

    kernels["fc1 dgrad + LN bwd (fused)"] = (lambda: ln_fused(hpost, w1, Cn, 4 * Cn, 0), 8.0 * M * Cn * Cn, 2.0 * M * Cn * 7,
                                             f"BN{256 if Cn % 256 == 0 else 128} ta0 tb1 ln_bwd cluster{max(1, Cn // 256)}")
    if stage < 3:
        kernels["downsample dgrad + LN bwd (fused)"] = (lambda: ln_fused(dsdy, dsw, 4 * Cn, 2 * Cn, H // 2), 2.0 * Md * 2 * Cn * 4 * Cn,
                                                        2.0 * (Md * 2 * Cn + 8 * Cn * Cn) + 6.0 * M * Cn,
                                                        f"BN256 ta0 tb1 ln_bwd cluster{max(1, Cn // 256)}")


for name, (fn, flops, bytes_, instantiation) in kernels.items():
    if only and not any(o in name for o in only):
        continue
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / iters * 1e3
    print(json.dumps({"kernel": name, "stage": stage, "batch": B, "us": round(us, 1), "tflops": round(flops / us / 1e6, 1),
                      "algo_GBps": round(bytes_ / us / 1e3, 1), "gemm": instantiation}))
