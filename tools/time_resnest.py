"""Device timing of the ResNeSt embedding forward (not the bench contract).  argv: model batch iters [--convs].

Times device-resident `embed` at 224x224 with CUDA events and prints one JSON line: the card's name and power limit (read
in the same run), embeddings/s, ms per batch, and TFLOP/s on the useful FLOPs (a grouped conv counts k*k*Cin/groups MACs per
output) with the executed FLOPs beside them (the split conv executes k*k*cpb*64, vdk_conv2d_grouped_ex).  The gate kernels'
share of forward kernel time (radix mean, excitation, combine, avd pool) comes from one torch.profiler forward of its own.
With --convs it also prints, per distinct split conv shape, vdk_conv2d_grouped_ex against
torch.nn.functional.conv2d(groups=...) (bf16, channels_last: cuDNN) on the same card — a yardstick only; torch is not on the
product path."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tools.time_resnet import card, time_fn  # noqa: E402
from visiondk_b200 import _lib  # noqa: E402
from visiondk_b200.backbone import BackboneFactory  # noqa: E402
from visiondk_b200.resnest import RESNEST_ARCHS, attn_width, group_width, pack_split, split_conv_blocks  # noqa: E402

GATE_KERNELS = ("radix_mean", "attn_excite", "radix_combine", "avgpool3s2")


def conv_shapes(name, size):
    """[(H_in, Cin, Cout, k, stride, pad, groups)] of every conv of the network (stem included; the split convs at their
    stride-1 resolution), the attention FC widths [(C, R C, A, cardinality)], and the neck's K."""
    a = RESNEST_ARCHS[name]
    R, card_, bw = a["radix"], a["cardinality"], a["base_width"]
    out = [(size, 3, 32, 3, 2, 1, 1), (size // 2, 32, 32, 3, 1, 1, 1), (size // 2, 32, 64, 3, 1, 1, 1)]
    fcs = []
    h, cin = size // 4, 64
    for i, d in enumerate(a["depths"]):
        gw, cout, stride = group_width(64 << i, bw, card_), 256 << i, (1 if i == 0 else 2)
        for j in range(d):
            s = stride if j == 0 else 1
            hs = h // s if a["avd_first"] else h
            out += [(h, cin, gw, 1, 1, 0, 1), (hs, gw, R * gw, 3, 1, 1, card_ * R), (h // s, gw, cout, 1, 1, 0, 1)]
            if j == 0:
                out.append((h, cin, cout, 2, 2, 0, 1) if s == 2 else (h, cin, cout, 1, 1, 0, 1))
            fcs.append((gw, R * gw, attn_width(gw, R), card_))
            h, cin = h // s, cout
    return out, fcs, h * h * 2048


def flops_per_image(name, size, feat=512):
    """(useful, executed) FLOPs of one image's forward."""
    shapes, fcs, kn = conv_shapes(name, size)
    useful = executed = 2.0 * kn * feat + sum(2.0 * (c * a_ + a_ * rc) / g for c, rc, a_, g in fcs)
    for h, cin, cout, k, s, p, g in shapes:
        ho = (h + 2 * p - k) // s + 1
        useful += 2.0 * ho * ho * cout * k * k * cin / g
        executed += 2.0 * ho * ho * cout * k * k * (split_conv_blocks(cin, cout, g) * 64 if g > 1 else cin)
    return useful, executed


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "resnest50d_4s2x40d"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 10
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
    share = {k: round(sum(e.time_range.elapsed_us() for e in ev if k + "_kernel" in e.name) / max(total_k, 1e-9), 4)
             for k in GATE_KERNELS}
    gemm_us = sum(e.time_range.elapsed_us() for e in ev if "gemm_tn_kernel" in e.name)
    useful, executed = flops_per_image(name, size)
    print(json.dumps({"model": name, "image_size": size, "batch": B, "ms": round(ms, 3), "emb_per_s": round(B / ms * 1e3, 1),
                      "useful_tflops": round(B * useful / ms / 1e9, 1), "executed_tflops": round(B * executed / ms / 1e9, 1),
                      "useful_gflop_per_img": round(useful / 1e9, 3), "executed_gflop_per_img": round(executed / 1e9, 3),
                      "gate_share_of_kernel_time": round(sum(share.values()), 4), "gate_shares": share,
                      "gemm_share_of_kernel_time": round(gemm_us / max(total_k, 1e-9), 4), "card": card()}))
    if "--convs" not in sys.argv:
        return
    lib = _lib.load()
    seen = set()
    torch.backends.cudnn.benchmark = True
    for h, cin, cout, k, s, p, g in conv_shapes(name, size)[0]:
        if g == 1 or (h, cin, g) in seen:
            continue
        seen.add((h, cin, g))
        xa = torch.randn(B, h, h, cin, device="cuda").to(torch.bfloat16)
        w = (torch.randn(cout, cin // g, k, k, device="cuda") * 0.05).to(torch.bfloat16)
        wp = pack_split(w.float(), g).to(torch.bfloat16).contiguous()
        bias = torch.zeros(cout, device="cuda")
        y = torch.empty(B, h, h, cout, device="cuda", dtype=torch.bfloat16)
        d = _lib.ConvDesc(x=xa.data_ptr(), w=wp.data_ptr(), bias=bias.data_ptr(), residual=0, y=y.data_ptr(), B=B, H=h, W=h, Cin=cin,
                          Cout=cout, kernel=k, stride=s, pad=p, epilogue=_lib.EPI_RELU)
        ours = time_fn(lambda: _lib.check(lib.vdk_conv2d_grouped_ex(C.byref(d), g, _lib.stream_ptr()), "vdk_conv2d_grouped_ex"), 20)
        xt = xa.permute(0, 3, 1, 2)  # NCHW view of NHWC memory: channels_last
        wt = w.contiguous(memory_format=torch.channels_last)
        ref = time_fn(lambda: torch.relu(torch.nn.functional.conv2d(xt, wt, bias.to(torch.bfloat16), stride=s, padding=p, groups=g)), 20)
        fu = 2.0 * B * h * h * cout * k * k * cin / g
        fe = 2.0 * B * h * h * cout * k * k * split_conv_blocks(cin, cout, g) * 64
        print(json.dumps({"H": h, "Cin": cin, "Cout": cout, "groups": g, "vdk_ms": round(ours, 4),
                          "vdk_useful_tflops": round(fu / ours / 1e9, 1), "vdk_executed_tflops": round(fe / ours / 1e9, 1),
                          "cudnn_ms": round(ref, 4), "cudnn_useful_tflops": round(fu / ref / 1e9, 1)}))


if __name__ == "__main__":
    main()
