"""Device timing of the ResNet embedding forward (not the bench contract).  argv: model batch iters [--convs].

Times device-resident `embed` with CUDA events and prints one JSON line: the card's name and power limit (read in the
same run), embeddings/s, ms per batch and TFLOP/s from the conv shapes below.  The stem's share of the forward comes from a
torch.profiler run of its own (the kernels launched before the max pool).  With --convs it also prints, per distinct conv
shape of the network at that batch, vdk_conv2d against torch.nn.functional.conv2d (bf16, channels_last: cuDNN) on the same
card — a yardstick only; torch is not on the product path."""
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from visiondk_b200 import _lib  # noqa: E402
from visiondk_b200.resnet import RESNET_ARCHS, ResNetWrapper  # noqa: E402


def conv_shapes(name, size):
    """[(H_in, Cin, Cout, k, stride, pad, count)] of every conv of the network (stem included), and the neck's K."""
    a = RESNET_ARCHS[name]
    base, deep, avg = a.get("base_width", 64), a.get("stem_type") == "deep", a.get("avg_down", False)
    out = []
    if deep:
        out += [(size, 3, 32, 3, 2, 1, 1), (size // 2, 32, 32, 3, 1, 1, 1), (size // 2, 32, 64, 3, 1, 1, 1)]
    else:
        out.append((size, 3, 64, 7, 2, 3, 1))
    h, cin = size // 4, 64
    for i, d in enumerate(a["depths"]):
        planes, stride = 64 << i, (1 if i == 0 else 2)
        width = planes * base // 64
        for j in range(d):
            s = stride if j == 0 else 1
            out += [(h, cin, width, 1, 1, 0, 1), (h, width, width, 3, s, 1, 1), (h // s, width, planes * 4, 1, 1, 0, 1)]
            if j == 0:
                out.append((h, cin, planes * 4, 2, 2, 0, 1) if (avg and s == 2) else (h, cin, planes * 4, 1, s, 0, 1))
            h, cin = h // s, planes * 4
    return out, h * h * 2048


def flops_per_image(name, size, feat=512):
    shapes, kn = conv_shapes(name, size)
    f = 0.0
    for h, cin, cout, k, s, p, n in shapes:
        ho = (h + 2 * p - k) // s + 1
        f += n * 2.0 * ho * ho * cout * k * k * cin
    return f + 2.0 * kn * feat


def time_fn(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "resnet50"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    size = 224
    m = ResNetWrapper(name, 512, size, pretrained=False).cuda().eval()
    x = torch.randn(B, 3, size, size, device="cuda")
    m.embed(x, True)
    ms = time_fn(lambda: m.embed(x, True), iters)
    # stem share: kernels from the first patch-rows kernel up to the max pool, in one profiled forward
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.embed(x, True)
        torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                 and "Memset" not in e.name], key=lambda e: e.time_range.start)
    total_k = sum(e.time_range.elapsed_us() for e in ev)
    stem_us = 0.0
    for e in ev:
        if "maxpool" in e.name:
            break
        stem_us += e.time_range.elapsed_us()
    fl = flops_per_image(name, size)
    print(json.dumps({"model": name, "image_size": size, "batch": B, "ms": round(ms, 3), "emb_per_s": round(B / ms * 1e3, 1),
                      "tflops": round(B * fl / ms / 1e9, 1), "gflop_per_img": round(fl / 1e9, 3),
                      "stem_share_of_kernel_time": round(stem_us / max(total_k, 1e-9), 4), "card": card()}))
    if "--convs" not in sys.argv:
        return
    lib = _lib.load()
    seen = set()
    for h, cin, cout, k, s, p, _ in conv_shapes(name, size)[0]:
        if cin % 64 or (h, cin, cout, k, s, p) in seen:
            continue
        seen.add((h, cin, cout, k, s, p))
        ho = (h + 2 * p - k) // s + 1
        xa = torch.randn(B, h, h, cin, device="cuda").to(torch.bfloat16)
        w = (torch.randn(cout, k, k, cin, device="cuda") * 0.05).to(torch.bfloat16)
        bias = torch.zeros(cout, device="cuda")
        y = torch.empty(B, ho, ho, cout, device="cuda", dtype=torch.bfloat16)
        d = _lib.ConvDesc(x=xa.data_ptr(), w=w.data_ptr(), bias=bias.data_ptr(), residual=0, y=y.data_ptr(), B=B, H=h, W=h, Cin=cin,
                          Cout=cout, kernel=k, stride=s, pad=p, epilogue=_lib.EPI_RELU)
        ours = time_fn(lambda: _lib.check(lib.vdk_conv2d(C.byref(d), _lib.stream_ptr()), "vdk_conv2d"), 20)
        xt = xa.permute(0, 3, 1, 2)  # NCHW view of NHWC memory: channels_last
        wt = w.permute(0, 3, 1, 2)
        torch.backends.cudnn.benchmark = True
        ref = time_fn(lambda: torch.relu(torch.nn.functional.conv2d(xt, wt, bias.to(torch.bfloat16), stride=s, padding=p)), 20)
        f = 2.0 * B * ho * ho * cout * k * k * cin
        print(json.dumps({"H": h, "Cin": cin, "Cout": cout, "k": k, "stride": s, "vdk_ms": round(ours, 4), "vdk_tflops": round(f / ours / 1e9, 1),
                          "cudnn_ms": round(ref, 4), "cudnn_tflops": round(f / ref / 1e9, 1)}))


if __name__ == "__main__":
    main()
