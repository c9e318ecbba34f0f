"""Device timing of the MobileNetV3 embedding forward (not the bench contract).  argv: model batch iters [--dw].

Times device-resident `embed` at 224x224 with CUDA events and prints one JSON line: the card's name and power limit (read
in the same run), embeddings/s and ms per batch; from one torch.profiler forward of its own, the launches per forward and
the shares of kernel time taken by the depthwise kernels and the SE path (excitation + gate application; the SE mean is
fused into the depthwise kernel).  These models are bound by memory traffic and launches, not by the tensor cores.

With --dw it also times every distinct depthwise shape of the model at the same batch against F.conv2d(groups=C) in bf16
channels_last (cuDNN; bias and activation left out of its side), each with CUDA events, and reports the achieved GB/s of
both (input read once + output written once) against the H100 SXM's 3.35 TB/s."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.time_resnet import card, time_fn  # noqa: E402
from visiondk_b200 import _lib  # noqa: E402
from visiondk_b200.backbone import BackboneFactory  # noqa: E402
from visiondk_b200.mobilenetv3 import ACTS, MOBILENETV3_ARCHS, decode_blocks  # noqa: E402


def dw_shapes(name, size):
    """Distinct (C, H, kernel, stride, act, with SE mean) of the model's depthwise convs."""
    spec, out, h = MOBILENETV3_ARCHS[name], [], size // 2
    for stage in decode_blocks(spec["arch"], spec["act"]):
        for kind, cin, cout, k, stride, mid, act, se_rd in stage:
            if kind != "cn" and (mid, h, k, stride, ACTS[act], se_rd > 0) not in out:
                out.append((mid, h, k, stride, ACTS[act], se_rd > 0))
            h = -(-h // stride)
    return out


def time_dw(name, B, size, iters):
    lib, rule = _lib.load(), 0 if MOBILENETV3_ARCHS[name]["tf"] else 1
    rows = []
    for Cc, H, k, stride, act, se in dw_shapes(name, size):
        Ho = -(-H // stride)
        x = torch.randn(B, H, H, Cc, device="cuda").to(torch.bfloat16)
        w = torch.randn(k * k, Cc, device="cuda") / k
        b = torch.zeros(Cc, device="cuda")
        y = torch.empty(B, Ho, Ho, Cc, device="cuda", dtype=torch.bfloat16)
        mean = torch.empty(B, Cc, device="cuda") if se else None
        ours = lambda: _lib.check(lib.vdk_dwconv_mnv3(x.data_ptr(), B, H, H, Cc, k, stride, rule, act, w.data_ptr(), b.data_ptr(),
                                                      y.data_ptr(), _lib.ptr(mean), _lib.stream_ptr()), "vdk_dwconv_mnv3")
        xc = x.permute(0, 3, 1, 2)  # NCHW view of the NHWC tensor: channels_last
        wc = w.t().reshape(Cc, 1, k, k).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        cudnn = lambda: F.conv2d(xc, wc, None, stride, k // 2, 1, Cc)
        ours()
        cudnn()
        t_ours, t_cudnn = time_fn(ours, iters), time_fn(cudnn, iters)
        gb = 2.0 * B * Cc * (H * H + Ho * Ho) / 1e9
        rows.append({"C": Cc, "H": H, "k": k, "stride": stride, "act": act, "se_mean": se, "ours_ms": round(t_ours, 4),
                     "cudnn_ms": round(t_cudnn, 4), "ours_gbs": round(gb / t_ours * 1e3, 1),
                     "cudnn_gbs": round(gb / t_cudnn * 1e3, 1), "ours_of_3350": round(gb / t_ours * 1e3 / 3350, 3)})
    return rows


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    name = args[0] if args else "tf_mobilenetv3_large_minimal_100"
    B = int(args[1]) if len(args) > 1 else 256
    iters = int(args[2]) if len(args) > 2 else 20
    size = 224
    m = BackboneFactory({f"timm-{name}": {"pretrained": False, "image_size": size, "feat_dim": 512}}).get_backbone().cuda().eval()
    x = torch.randn(B, 3, size, size, device="cuda")
    m.embed(x, True)
    ms = time_fn(lambda: m.embed(x, True), iters)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.embed(x, True)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
          and "Memset" not in e.name]
    total_k = sum(e.time_range.elapsed_us() for e in ev)
    dw_us = sum(e.time_range.elapsed_us() for e in ev if "dwconv_mnv3_kernel" in e.name)
    se_us = sum(e.time_range.elapsed_us() for e in ev if "se_excite_kernel" in e.name or "se_apply_kernel" in e.name)
    out = {"model": name, "image_size": size, "batch": B, "ms": round(ms, 3), "emb_per_s": round(B / ms * 1e3, 1),
           "launches": len(ev), "kernel_ms": round(total_k / 1e3, 3), "depthwise_share": round(dw_us / max(total_k, 1e-9), 4),
           "se_share": round(se_us / max(total_k, 1e-9), 4), "card": card()}
    if "--dw" in sys.argv:
        out["dw"] = time_dw(name, B, size, iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
