"""Device timing of the EfficientNetV2 embedding forward (not the bench contract).  argv: model batch iters.

Times device-resident `embed` at 224x224 with CUDA events and prints one JSON line: the card's name and power limit (read
in the same run), embeddings/s, ms per batch, and TFLOP/s on the useful FLOPs counted from the shapes (the 3x3 convs with
Cin not a multiple of 64 execute Cinp / Cin times more, reported beside them).  From one torch.profiler forward of its own:
the shares of the forward's kernel time taken by the depthwise kernels, the SE path (excitation + gate application; the
SE mean is fused into the depthwise kernel) and stage 0 (its convolutions, in launch order after the stem)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tools.time_resnet import card, time_fn  # noqa: E402
from visiondk_b200.backbone import BackboneFactory  # noqa: E402
from visiondk_b200.efficientnet import EFFNETV2_ARCHS, HEAD_CH  # noqa: E402


def flops_per_image(name, size, feat=512):
    """(useful, executed) FLOPs of one image's forward, SE included."""
    a = EFFNETV2_ARCHS[name]
    h = size // 2
    useful = executed = 2.0 * h * h * a["stem"] * 27
    cin = a["stem"]
    for kind, reps, stride, exp, cout in a["stages"]:
        for j in range(reps):
            s = stride if j == 0 else 1
            ho = -(-h // s)
            cinp = -(-cin // 64) * 64
            if kind == "cn":
                useful += 2.0 * ho * ho * cout * 9 * cin
                executed += 2.0 * ho * ho * cout * 9 * cinp
            elif kind == "er":
                mid = cin * exp
                useful += 2.0 * ho * ho * (mid * 9 * cin + cout * mid)
                executed += 2.0 * ho * ho * (mid * 9 * cinp + cout * mid)
            else:
                mid, rd = cin * exp, round(cin / 4)
                f = 2.0 * h * h * mid * cin + 2.0 * ho * ho * mid * 9 + 4.0 * mid * rd + 2.0 * ho * ho * cout * mid
                useful += f
                executed += f
            h, cin = ho, cout
    f = 2.0 * h * h * HEAD_CH * cin + 2.0 * h * h * HEAD_CH * feat
    return useful + f, executed + f


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "tf_efficientnetv2_l"
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
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                 and "Memset" not in e.name), key=lambda e: e.time_range.start)
    total_k = sum(e.time_range.elapsed_us() for e in ev)
    dw_us = sum(e.time_range.elapsed_us() for e in ev if "dwconv3_silu_kernel" in e.name)
    se_us = sum(e.time_range.elapsed_us() for e in ev if "se_excite_kernel" in e.name or "se_apply_kernel" in e.name)
    # launch order: fill (gamma = 1), stem patch rows, stem GEMM, then stage 0's convolutions
    first = next(i for i, e in enumerate(ev) if "patch_rows" in e.name) + 2
    stage0_us = sum(e.time_range.elapsed_us() for e in ev[first:first + EFFNETV2_ARCHS[name]["stages"][0][1]])
    useful, executed = flops_per_image(name, size)
    print(json.dumps({"model": name, "image_size": size, "batch": B, "ms": round(ms, 3), "emb_per_s": round(B / ms * 1e3, 1),
                      "useful_tflops": round(B * useful / ms / 1e9, 1), "executed_tflops": round(B * executed / ms / 1e9, 1),
                      "useful_gflop_per_img": round(useful / 1e9, 3), "executed_gflop_per_img": round(executed / 1e9, 3),
                      "depthwise_share": round(dw_us / max(total_k, 1e-9), 4), "se_share": round(se_us / max(total_k, 1e-9), 4),
                      "stage0_share": round(stage0_us / max(total_k, 1e-9), 4), "kernel_ms": round(total_k / 1e3, 3),
                      "card": card()}))


if __name__ == "__main__":
    main()
