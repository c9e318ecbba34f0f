"""Quick device timing of the ViT embedding forward (not the bench contract).  argv: model batch iters.

Image size, token count (with or without a class token) and MLP width come from visiondk_b200.vit's arch tables."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from visiondk_b200.vit import ViTWrapper, VIT_ARCHS, VIT_IMAGE_SIZE

name = sys.argv[1] if len(sys.argv) > 1 else "vit_base_patch16_224"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
iters = int(sys.argv[3]) if len(sys.argv) > 3 else 10
size = VIT_IMAGE_SIZE.get(name, 224)
m = ViTWrapper(name, 512, size, pretrained=False).cuda().eval()
x = torch.randn(B, 3, size, size, device="cuda")
for _ in range(2):
    y = m.embed(x, True)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(iters):
    y = m.embed(x, True)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
patch, dim, depth, heads = VIT_ARCHS[name]
T, N, mlp = m.model.tokens, (size // patch) ** 2, m.model.mlp_dim
# per block: qkv (3C) + proj (C) + fc1 / fc2 (mlp each) GEMMs, and QK^T + PV; patch embedding; the neck Linear
flops = depth * (2.0 * T * dim * (4 * dim + 2 * mlp) + 4.0 * T * T * dim) + 2.0 * N * 3 * patch * patch * dim + 2.0 * T * dim * 512
dev = torch.cuda.get_device_properties(0)
print(json.dumps({"model": name, "image_size": size, "tokens": T, "batch": B, "ms": ms, "img_per_s": B / ms * 1e3,
                  "tflops": B * flops / ms / 1e9, "gflop_per_img": flops / 1e9, "device": dev.name}))
