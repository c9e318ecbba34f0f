"""Device timing of the Swin V2 embedding forward (not the bench contract).  argv: model batch iters [--attention].

Times device-resident `embed` at 256x256 with CUDA events and prints one JSON line: the card's name and power limit (read in
the same run), embeddings/s, ms per batch, and TFLOP/s counting the GEMM FLOPs (patch embedding, qkv, proj, fc1, fc2, patch
merging, neck) plus 4 * w^2 * C per token per block for the window attention.  The window attention's and the post-norm
residual's shares of forward kernel time come from one torch.profiler forward of its own.  With --attention it also times
vdk_window_attention_fwd alone at every distinct (map, C, window, shift) of the tower and reports its bytes/s (8 C bytes per
token: the qkv read and the output write) against the H100 SXM data sheet's 3.35 TB/s."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tools.time_resnet import card, time_fn  # noqa: E402
from visiondk_b200 import _lib  # noqa: E402
from visiondk_b200.backbone import BackboneFactory  # noqa: E402
from visiondk_b200.swin import IMAGE_SIZE, SWINV2_ARCHS, stage_windows  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet


def blocks(name):
    """[(map side, C, heads, window, shift)] of every block of the tower."""
    a = SWINV2_ARCHS[name]
    out = []
    for i, (w, s) in enumerate(stage_windows(a["window_size"])):
        for j in range(a["depths"][i]):
            out.append(((IMAGE_SIZE // 4) >> i, a["embed_dim"] << i, a["num_heads"][i], w, s if j % 2 else 0))
    return out


def flops_per_image(name, feat=512):
    a = SWINV2_ARCHS[name]
    c0, t0 = a["embed_dim"], (IMAGE_SIZE // 4) ** 2
    f = 2.0 * t0 * 48 * c0 + 2.0 * 64 * (8 * c0) * feat  # patch embedding, neck
    for i in range(1, 4):
        f += 2.0 * (t0 >> (2 * i)) * (4 * (c0 << (i - 1))) * (2 * (c0 << (i - 1)))  # patch merging
    for h, c, heads, w, s in blocks(name):
        t = h * h
        f += 2.0 * t * c * (3 * c + c + 4 * c + 4 * c) + 4.0 * t * w * w * c
    return f


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "swinv2_base_window8_256"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 128
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    m = BackboneFactory({f"timm-{name}": {"pretrained": False, "image_size": IMAGE_SIZE, "feat_dim": 512}}).get_backbone().cuda().eval()
    x = torch.randn(B, 3, IMAGE_SIZE, IMAGE_SIZE, device="cuda")
    m.embed(x, True)
    ms = time_fn(lambda: m.embed(x, True), iters)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.embed(x, True)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
          and "Memset" not in e.name]
    total_k = sum(e.time_range.elapsed_us() for e in ev)
    att_us = sum(e.time_range.elapsed_us() for e in ev if "window_attention_kernel" in e.name)
    pn_us = sum(e.time_range.elapsed_us() for e in ev if "postnorm_residual_kernel" in e.name)
    fl = flops_per_image(name)
    print(json.dumps({"model": name, "image_size": IMAGE_SIZE, "batch": B, "ms": round(ms, 3), "emb_per_s": round(B / ms * 1e3, 1),
                      "tflops": round(B * fl / ms / 1e9, 1), "gflop_per_img": round(fl / 1e9, 3),
                      "attention_share_of_kernel_time": round(att_us / max(total_k, 1e-9), 4),
                      "postnorm_share_of_kernel_time": round(pn_us / max(total_k, 1e-9), 4), "card": card()}))
    if "--attention" not in sys.argv:
        return
    lib = _lib.load()
    for h, c, heads, w, s in sorted(set(blocks(name)), reverse=True):
        qkv = (torch.randn(B, h, h, 3 * c, device="cuda")).to(torch.bfloat16)
        out = torch.empty(B, h, h, c, device="cuda", dtype=torch.bfloat16)
        scale = torch.full((heads,), 10.0, device="cuda")
        bias = torch.rand(heads, (2 * w - 1) ** 2, device="cuda")
        t = time_fn(lambda: _lib.check(lib.vdk_window_attention_fwd(qkv.data_ptr(), B, h, h, heads, w, s, scale.data_ptr(), bias.data_ptr(),
                                                                    out.data_ptr(), _lib.stream_ptr()), "vdk_window_attention_fwd"), 20)
        nbytes, flops = 8.0 * B * h * h * c, 4.0 * B * h * h * w * w * c
        print(json.dumps({"map": h, "C": c, "heads": heads, "window": w, "shift": s, "ms": round(t, 4),
                          "tb_per_s": round(nbytes / t / 1e9, 3), "share_of_hbm_peak": round(nbytes / t / 1e9 / HBM_TBS, 3),
                          "tflops": round(flops / t / 1e9, 1)}))


if __name__ == "__main__":
    main()
