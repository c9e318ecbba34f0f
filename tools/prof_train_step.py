"""torch.profiler trace of the ConvNeXt-B faceX train step (bench.py's train leg, profiler on): kernel time per class.

    python tools/prof_train_step.py [batch] [steps] [out_dir]       # defaults: 128, 3, prof_train_step

Builds the step exactly as bench.py does, runs 3 warm-up steps, then traces `steps` steps with CUDA activities.  Prints
one JSON line: the summed device time per kernel class (depthwise forward + LayerNorm, depthwise backward, GEMMs, rest),
each class's share of the step's kernel time, and the ten longest kernels.  The Chrome trace goes to out_dir.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from visiondk_b200.train import FaceTrainer, FaceTrainingModel

B = int(sys.argv[1]) if len(sys.argv) > 1 else 128
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
out_dir = sys.argv[3] if len(sys.argv) > 3 else "prof_train_step"
os.makedirs(out_dir, exist_ok=True)

torch.manual_seed(0)
cfg = {"backbone": {"timm-convnext_base": {"pretrained": False, "image_size": 224, "feat_dim": 512}},
       "head": {"arcface": {"feat_dim": 512, "num_class": 1000, "margin_arc": 0.35, "margin_am": 0.0, "scale": 32}}}
model = FaceTrainingModel(cfg).to("cuda")
with torch.no_grad():
    for n, p in model.named_parameters():
        if n.endswith("gamma"):
            p.fill_(0.1)
trainer = FaceTrainer(model, lr0=0.01, momentum=0.937, weight_decay=5e-4, label_smooth=0.1, layer_wise=True, warm_steps=0,
                      total_steps=100000, use_ema=True)
gen = torch.Generator(device="cuda").manual_seed(100)
x = torch.randn(B, 3, 224, 224, device="cuda", generator=gen)
y = torch.randint(0, 1000, (B,), device="cuda", generator=gen)
for _ in range(3):
    trainer.step(x, y)
torch.cuda.synchronize()

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
        trainer.step(x, y)
    torch.cuda.synchronize()
prof.export_chrome_trace(os.path.join(out_dir, "train_step.pt.trace.json"))


def kind(name):
    if "dwconv7_bwd" in name:
        return "depthwise backward"
    if "dwconv7" in name:
        return "depthwise forward + LayerNorm"
    if "gemm" in name.lower() or "wgmma" in name.lower():
        return "gemm"
    return "other"


per_kernel = {}
for e in prof.key_averages():
    t = getattr(e, "device_time_total", None)
    if t is None:
        t = e.cuda_time_total
    if t > 0 and e.key not in ("cudaDeviceSynchronize",):
        per_kernel[e.key] = per_kernel.get(e.key, 0.0) + t / steps / 1e3  # ms per step
classes = {}
for k, ms in per_kernel.items():
    classes[kind(k)] = classes.get(kind(k), 0.0) + ms
total = sum(classes.values())
top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:10]
print(json.dumps({"device": torch.cuda.get_device_name(0), "batch": B, "steps": steps, "kernel_ms_per_step": round(total, 3),
                  "classes_ms": {k: round(v, 3) for k, v in sorted(classes.items())},
                  "classes_share": {k: round(v / total, 4) for k, v in sorted(classes.items())},
                  "top": [[k[:100], round(v, 3)] for k, v in top]}))
