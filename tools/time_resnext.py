"""Device timing of the ResNeXt / legacy SENet embedding forward (not the bench contract).  argv: model batch iters [--convs].

Times device-resident `embed` at 224x224 with CUDA events and prints one JSON line: the card's name and power limit (read
in the same run), embeddings/s, ms per batch, and TFLOP/s on the useful FLOPs (a grouped conv counts k*k*Cin/groups MACs per
output) with the executed FLOPs beside them (the block-diagonal grouped conv executes k*k*128).  The SE kernels' share of
forward kernel time comes from one torch.profiler forward of its own.  With --convs it also prints, per distinct grouped conv
shape, vdk_conv2d_grouped against torch.nn.functional.conv2d(groups=...) (bf16, channels_last: cuDNN) on the same card — a
yardstick only; torch is not on the product path."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tools.time_resnet import card, time_fn  # noqa: E402
from visiondk_b200 import _lib  # noqa: E402
from visiondk_b200.backbone import BackboneFactory  # noqa: E402
from visiondk_b200.resnet import RESNEXT_ARCHS, pack_grouped  # noqa: E402
from visiondk_b200.senet import SE_REDUCTION, SENET_ARCHS  # noqa: E402


def conv_shapes(name, size):
    """[(H_in, Cin, Cout, k, stride, pad, groups)] of every conv of the network (stem included), the SE FC widths
    [(C, rd)], and the neck's K."""
    if name in RESNEXT_ARCHS:
        a = RESNEXT_ARCHS[name]
        groups, width0, s_on_1 = a["cardinality"], a["cardinality"] * a["base_width"], False
        deep, avg, se = a.get("stem_type") == "deep", a.get("avg_down", False), False
    else:
        a = SENET_ARCHS[name]
        groups, s_on_1 = a["groups"], a["block"] == "seresnet"
        width0, deep, avg, se = (64 if s_on_1 else 4 * groups), False, False, True
    out, fcs = [], []
    if deep:
        out += [(size, 3, 32, 3, 2, 1, 1), (size // 2, 32, 32, 3, 1, 1, 1), (size // 2, 32, 64, 3, 1, 1, 1)]
    else:
        out.append((size, 3, 64, 7, 2, 3, 1))
    h, cin = size // 4, 64
    for i, d in enumerate(a["depths"]):
        width, cout, stride = width0 << i, 256 << i, (1 if i == 0 else 2)
        for j in range(d):
            s = stride if j == 0 else 1
            s1, s2 = (s, 1) if s_on_1 else (1, s)
            out += [(h, cin, width, 1, s1, 0, 1), (h // s1, width, width, 3, s2, 1, groups), (h // s, width, cout, 1, 1, 0, 1)]
            if j == 0:
                out.append((h, cin, cout, 2, 2, 0, 1) if (avg and s == 2) else (h, cin, cout, 1, s, 0, 1))
            if se:
                fcs.append((cout, cout // SE_REDUCTION))
            h, cin = h // s, cout
    return out, fcs, h * h * 2048


def flops_per_image(name, size, feat=512):
    """(useful, executed) FLOPs of one image's forward."""
    shapes, fcs, kn = conv_shapes(name, size)
    useful = executed = 2.0 * kn * feat + sum(4.0 * c * rd for c, rd in fcs)
    for h, cin, cout, k, s, p, g in shapes:
        ho = (h + 2 * p - k) // s + 1
        useful += 2.0 * ho * ho * cout * k * k * cin / g
        executed += 2.0 * ho * ho * cout * k * k * (128 if g > 1 else cin)
    return useful, executed


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "resnext50_32x4d"
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
    se_us = sum(e.time_range.elapsed_us() for e in ev if "se_" in e.name and "_kernel" in e.name)
    useful, executed = flops_per_image(name, size)
    print(json.dumps({"model": name, "image_size": size, "batch": B, "ms": round(ms, 3), "emb_per_s": round(B / ms * 1e3, 1),
                      "useful_tflops": round(B * useful / ms / 1e9, 1), "executed_tflops": round(B * executed / ms / 1e9, 1),
                      "useful_gflop_per_img": round(useful / 1e9, 3), "executed_gflop_per_img": round(executed / 1e9, 3),
                      "se_share_of_kernel_time": round(se_us / max(total_k, 1e-9), 4), "card": card()}))
    if "--convs" not in sys.argv:
        return
    lib = _lib.load()
    seen = set()
    torch.backends.cudnn.benchmark = True
    for h, cin, cout, k, s, p, g in conv_shapes(name, size)[0]:
        if g == 1 or (h, cin, s, g) in seen:
            continue
        seen.add((h, cin, s, g))
        ho = (h + 2 * p - k) // s + 1
        xa = torch.randn(B, h, h, cin, device="cuda").to(torch.bfloat16)
        w = (torch.randn(cout, cin // g, k, k, device="cuda") * 0.05).to(torch.bfloat16)
        wp = pack_grouped(w.float()).to(torch.bfloat16).contiguous()
        bias = torch.zeros(cout, device="cuda")
        y = torch.empty(B, ho, ho, cout, device="cuda", dtype=torch.bfloat16)
        d = _lib.ConvDesc(x=xa.data_ptr(), w=wp.data_ptr(), bias=bias.data_ptr(), residual=0, y=y.data_ptr(), B=B, H=h, W=h, Cin=cin,
                          Cout=cout, kernel=k, stride=s, pad=p, epilogue=_lib.EPI_RELU)
        ours = time_fn(lambda: _lib.check(lib.vdk_conv2d_grouped(C.byref(d), g, _lib.stream_ptr()), "vdk_conv2d_grouped"), 20)
        xt = xa.permute(0, 3, 1, 2)  # NCHW view of NHWC memory: channels_last
        wt = w.contiguous(memory_format=torch.channels_last)
        ref = time_fn(lambda: torch.relu(torch.nn.functional.conv2d(xt, wt, bias.to(torch.bfloat16), stride=s, padding=p, groups=g)), 20)
        fu = 2.0 * B * ho * ho * cout * k * k * cin / g
        fe = 2.0 * B * ho * ho * cout * k * k * 128
        print(json.dumps({"H": h, "C": cin, "stride": s, "groups": g, "vdk_ms": round(ours, 4),
                          "vdk_useful_tflops": round(fu / ours / 1e9, 1), "vdk_executed_tflops": round(fe / ours / 1e9, 1),
                          "cudnn_ms": round(ref, 4), "cudnn_useful_tflops": round(fu / ref / 1e9, 1)}))


if __name__ == "__main__":
    main()
