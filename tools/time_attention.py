"""Device timing of the wgmma attention forward (vdk_attention_fwd) at head dims 64, 72 and 80 on one shape with the same
B * H * N, and its achieved TFLOP/s from the algorithmic 4 * B * H * N^2 * D (QK^T and PV).  argv: batch heads tokens iters."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from visiondk_b200 import _lib

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
H = int(sys.argv[2]) if len(sys.argv) > 2 else 16
N = int(sys.argv[3]) if len(sys.argv) > 3 else 1024
iters = int(sys.argv[4]) if len(sys.argv) > 4 else 50
lib = _lib.load()
dev = torch.cuda.get_device_properties(0)
for D in (64, 72, 80):
    qkv = torch.randn(B, N, 3, H, D, device="cuda").to(torch.bfloat16)
    out = torch.empty(B, N, H * D, dtype=torch.bfloat16, device="cuda")

    def run():
        _lib.check(lib.vdk_attention_fwd(qkv.data_ptr(), B, N, H, D, out.data_ptr(), _lib.stream_ptr()), "vdk_attention_fwd")

    for _ in range(5):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(json.dumps({"head_dim": D, "batch": B, "heads": H, "tokens": N, "ms": ms,
                      "tflops": 4.0 * B * H * N * N * D / ms / 1e9, "device": dev.name}))
