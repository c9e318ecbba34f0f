// augment.cu — the training-time image transform of the CBIR / face path on the device, for a batch of decoded RGB images of
// different sizes at source resolution: the reference's `data.train.augment` Compose (dataset/transforms.py:403-555), whose
// random draws the host has already made (visiondk_b200/augment.py) and passes as one vdk_aug_plan per image.
//
// Every source-resolution stage keeps the image size, so each image owns two uint8 buffers of its size and each stage reads
// the image's current buffer and writes the other one.  Stage k of the batch launches once over the images whose plan has a
// k-th op (mixed kinds in one launch), so an image that skips a stage costs nothing.  The last stage is the shared Pillow
// resampler (resample.h) reading the current buffer through the plan's crop box, padded and normalised into the output.
//
// Byte work, restated from what the reference executes on PIL images (Pillow 12, torchvision 0.26):
//   blend (ImageEnhance -> Image.blend, Blend.c): fp32 in1 + alpha * (in2 - in1), truncated, clipped when alpha is outside [0, 1]
//   RGB -> L (Convert.c rgb2l): (19595 r + 38470 g + 7471 b + 0x8000) >> 16
//   contrast degenerate (ImageEnhance.Contrast): int(mean(L) + 0.5), the mean of the image at that point of the order
//   HSV (Convert.c rgb2hsv_row / hsv2rgb): fp32 / fp64 arithmetic as written there
//   SMOOTH (Filter.c ImagingFilter3x3): fp32 kernel 1/13, 5/13, rows y+1, y, y-1, rounded, border pixels copied
//   rotate (Geometry.c affine_transform + bilinear_filter32RGB): fp64 position and interpolation, truncated
//   gaussian blur (torchvision _functional_tensor.gaussian_blur): fp32 n x n sum in row order, reflect padding, round-half-even
#include "resample.h"
#include "vdk_host.h"

#include <cmath>
#include <cstring>
#include <vector>

namespace vdk {

struct AugStep {            // one image's op in one stage
  const uint8_t* in;        // [h][w][3]
  uint8_t* out;             // [h][w][3]
  const vdk_aug_op* op;     // device copy of the plan's op
  unsigned long long* sum;  // CONTRAST: sum of L over the input
  int w, h;
};

__device__ __forceinline__ uint8_t blend8(int in1, int in2, float alpha) {
  const float t = __fadd_rn(static_cast<float>(in1), __fmul_rn(alpha, static_cast<float>(in2 - in1)));
  if (alpha >= 0.0f && alpha <= 1.0f) return static_cast<uint8_t>(t);
  return t <= 0.0f ? 0 : (t >= 255.0f ? 255 : static_cast<uint8_t>(t));
}

__device__ __forceinline__ int luma(const uint8_t* p) { return (p[0] * 19595 + p[1] * 38470 + p[2] * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ int clip255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// torchvision adjust_hue on a PIL image: Pillow RGB -> HSV, H += shift (uint8 wrap), Pillow HSV -> RGB
__device__ void hue_pixel(const uint8_t* p, int shift, uint8_t* o) {
  const int r = p[0], g = p[1], b = p[2];
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  int uh = 0, us = 0;
  if (minc != maxc) {
    const float cr = static_cast<float>(maxc - minc);
    const float s = __fdiv_rn(cr, static_cast<float>(maxc));
    const float rc = __fdiv_rn(static_cast<float>(maxc - r), cr);
    const float gc = __fdiv_rn(static_cast<float>(maxc - g), cr);
    const float bc = __fdiv_rn(static_cast<float>(maxc - b), cr);
    float h;
    if (r == maxc) h = __fsub_rn(bc, gc);
    else if (g == maxc) h = static_cast<float>(__dsub_rn(__dadd_rn(2.0, static_cast<double>(rc)), static_cast<double>(bc)));
    else h = static_cast<float>(__dsub_rn(__dadd_rn(4.0, static_cast<double>(gc)), static_cast<double>(rc)));
    h = static_cast<float>(fmod(__dadd_rn(__ddiv_rn(static_cast<double>(h), 6.0), 1.0), 1.0));
    uh = clip255(static_cast<int>(__dmul_rn(static_cast<double>(h), 255.0)));
    us = clip255(static_cast<int>(__dmul_rn(static_cast<double>(s), 255.0)));
  }
  const int hh = (uh + shift) & 255, ss = us, v = maxc;
  if (ss == 0) {
    o[0] = o[1] = o[2] = static_cast<uint8_t>(v);
    return;
  }
  const double h6 = __ddiv_rn(__dmul_rn(static_cast<double>(static_cast<float>(hh)), 6.0), 255.0);
  const int i = static_cast<int>(floor(h6));
  const float f = static_cast<float>(__dsub_rn(h6, static_cast<double>(static_cast<float>(i))));
  const float fs = static_cast<float>(__ddiv_rn(static_cast<double>(static_cast<float>(ss)), 255.0));
  const double vf = static_cast<double>(static_cast<float>(v));
  const uint8_t up = clip255(static_cast<int>(round(__dmul_rn(vf, __dsub_rn(1.0, fs)))));
  const uint8_t uq = clip255(static_cast<int>(round(__dmul_rn(vf, __dsub_rn(1.0, __dmul_rn(fs, f))))));
  const uint8_t ut = clip255(static_cast<int>(round(__dmul_rn(vf, __dsub_rn(1.0, __dmul_rn(fs, __dsub_rn(1.0, f)))))));
  const uint8_t uv = static_cast<uint8_t>(v);
  switch (i % 6) {
    case 0: o[0] = uv; o[1] = ut; o[2] = up; break;
    case 1: o[0] = uq; o[1] = uv; o[2] = up; break;
    case 2: o[0] = up; o[1] = uv; o[2] = ut; break;
    case 3: o[0] = up; o[1] = uq; o[2] = uv; break;
    case 4: o[0] = ut; o[1] = up; o[2] = uv; break;
    default: o[0] = uv; o[1] = up; o[2] = uq; break;
  }
}

// Image.rotate(BILINEAR): Pillow's affine position of the output pixel centre, its 2x2 bilinear filter (edge-clamped columns,
// the lower row replaced by the upper one past the last row), truncated; outside the source the fill (0) stays
__device__ void rotate_pixel(const uint8_t* in, int w, int h, const double* m, int x, int y, uint8_t* o) {
  const double xo = x + 0.5, yo = y + 0.5;
  double xin = __dadd_rn(__dadd_rn(__dmul_rn(m[0], xo), __dmul_rn(m[1], yo)), m[2]);
  double yin = __dadd_rn(__dadd_rn(__dmul_rn(m[3], xo), __dmul_rn(m[4], yo)), m[5]);
  o[0] = o[1] = o[2] = 0;
  if (xin < 0.0 || xin >= w || yin < 0.0 || yin >= h) return;
  xin = __dsub_rn(xin, 0.5);
  yin = __dsub_rn(yin, 0.5);
  const int xi = xin < 0.0 ? static_cast<int>(floor(xin)) : static_cast<int>(xin);
  const int yi = yin < 0.0 ? static_cast<int>(floor(yin)) : static_cast<int>(yin);
  const double dx = __dsub_rn(xin, xi), dy = __dsub_rn(yin, yi);
  const int yc = min(max(yi, 0), h - 1), x0 = min(max(xi, 0), w - 1), x1 = min(max(xi + 1, 0), w - 1);
  const uint8_t* r0 = in + static_cast<size_t>(yc) * w * 3;
  const bool second = yi + 1 >= 0 && yi + 1 < h;
  const uint8_t* r1 = in + static_cast<size_t>(second ? yi + 1 : yc) * w * 3;
  for (int c = 0; c < 3; ++c) {
    const int a0 = r0[3 * x0 + c], a1 = r0[3 * x1 + c];
    const double v1 = __dadd_rn(static_cast<double>(a0), __dmul_rn(static_cast<double>(a1 - a0), dx));
    double v2 = v1;
    if (second) {
      const int b0 = r1[3 * x0 + c], b1 = r1[3 * x1 + c];
      v2 = __dadd_rn(static_cast<double>(b0), __dmul_rn(static_cast<double>(b1 - b0), dx));
    }
    o[c] = static_cast<uint8_t>(static_cast<int>(__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy))));
  }
}

__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// sum of L over each CONTRAST input of the stage (other entries return at once)
__global__ void __launch_bounds__(256) aug_luma_sum_kernel(const AugStep* __restrict__ steps) {
  const AugStep st = steps[blockIdx.y];
  if (st.op->kind != VDK_AUG_CONTRAST) return;
  const int64_t total = static_cast<int64_t>(st.w) * st.h;
  unsigned long long acc = 0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    acc += luma(st.in + i * 3);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  __shared__ unsigned long long part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int k = 0; k < 8; ++k) t += part[k];
    atomicAdd(st.sum, t);
  }
}

// one stage: one thread per output pixel, each entry (blockIdx.y) with its own op kind
__global__ void __launch_bounds__(256) aug_stage_kernel(const AugStep* __restrict__ steps) {
  const AugStep st = steps[blockIdx.y];
  const vdk_aug_op* op = st.op;
  const int kind = op->kind, w = st.w, h = st.h;
  const int64_t total = static_cast<int64_t>(w) * h;
  int contrast_mean = 0;
  if (kind == VDK_AUG_CONTRAST)  // ImageStat mean (a double quotient), int(mean + 0.5)
    contrast_mean = static_cast<int>(__dadd_rn(__ddiv_rn(static_cast<double>(*st.sum), static_cast<double>(total)), 0.5));
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / w), x = static_cast<int>(i - static_cast<int64_t>(y) * w);
    const uint8_t* p = st.in + i * 3;
    uint8_t* o = st.out + i * 3;
    switch (kind) {
      case VDK_AUG_BRIGHTNESS:
        for (int c = 0; c < 3; ++c) o[c] = blend8(0, p[c], op->alpha);
        break;
      case VDK_AUG_SATURATION: {
        const int l = luma(p);
        for (int c = 0; c < 3; ++c) o[c] = blend8(l, p[c], op->alpha);
        break;
      }
      case VDK_AUG_CONTRAST:
        for (int c = 0; c < 3; ++c) o[c] = blend8(contrast_mean, p[c], op->alpha);
        break;
      case VDK_AUG_HUE:
        hue_pixel(p, op->hue_shift, o);
        break;
      case VDK_AUG_CUTOUT: {
        int hole = -1;
        for (int k = 0; k < op->n; ++k) {
          const int* b = op->box[k];
          if (x >= b[0] && x < b[0] + b[2] && y >= b[1] && y < b[1] + b[3]) hole = k;
        }
        for (int c = 0; c < 3; ++c) o[c] = hole < 0 ? p[c] : static_cast<uint8_t>(op->color[hole][c]);
        break;
      }
      case VDK_AUG_BLUR: {
        const int n = op->n, r = n / 2;
        float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
        for (int ky = 0; ky < n; ++ky) {
          const uint8_t* row = st.in + static_cast<size_t>(reflect(y + ky - r, h)) * w * 3;
          for (int kx = 0; kx < n; ++kx) {
            const float k = __fmul_rn(op->kernel[ky], op->kernel[kx]);
            const uint8_t* q = row + reflect(x + kx - r, w) * 3;
            a0 = __fadd_rn(a0, __fmul_rn(k, static_cast<float>(q[0])));
            a1 = __fadd_rn(a1, __fmul_rn(k, static_cast<float>(q[1])));
            a2 = __fadd_rn(a2, __fmul_rn(k, static_cast<float>(q[2])));
          }
        }
        o[0] = static_cast<uint8_t>(clip255(static_cast<int>(rintf(a0))));
        o[1] = static_cast<uint8_t>(clip255(static_cast<int>(rintf(a1))));
        o[2] = static_cast<uint8_t>(clip255(static_cast<int>(rintf(a2))));
        break;
      }
      case VDK_AUG_ROTATE:
        rotate_pixel(st.in, w, h, op->matrix, x, y, o);
        break;
      case VDK_AUG_SHARPNESS: {
        uint8_t d[3] = {p[0], p[1], p[2]};
        if (x > 0 && x < w - 1 && y > 0 && y < h - 1) {
          const float k1 = __fdiv_rn(1.0f, 13.0f), k5 = __fdiv_rn(5.0f, 13.0f);
          for (int c = 0; c < 3; ++c) {
            float ss = 0.0f;
            for (int dy = 1; dy >= -1; --dy) {
              const uint8_t* q = st.in + (static_cast<size_t>(y + dy) * w + x) * 3 + c;
              const float mid = dy == 0 ? k5 : k1;
              ss = __fadd_rn(ss, __fadd_rn(__fadd_rn(__fmul_rn(static_cast<float>(q[-3]), k1), __fmul_rn(static_cast<float>(q[0]), mid)),
                                           __fmul_rn(static_cast<float>(q[3]), k1)));
            }
            d[c] = ss <= 0.0f ? 0 : (ss >= 255.0f ? 255 : static_cast<uint8_t>(__fadd_rn(ss, 0.5f)));
          }
        }
        for (int c = 0; c < 3; ++c) o[c] = blend8(d[c], p[c], op->alpha);
        break;
      }
      default: {  // VDK_AUG_HFLIP
        const uint8_t* q = st.in + (static_cast<size_t>(y) * w + (w - 1 - x)) * 3;
        o[0] = q[0]; o[1] = q[1]; o[2] = q[2];
      }
    }
  }
}

struct AugLayout {
  PreLayout pre;
  int crop[4];     // x, y, w, h of the resized box
  size_t buf[2];   // the two source-resolution buffers
};

// workspace = [resampler descriptors | stage entries | plans | contrast sums | coefficient tables] (built on the host, one
// upload of `*upload_end` bytes) then [two source-size buffers + one resampler intermediate per image] (device only)
static int aug_plan(const vdk_image_desc* images, const vdk_aug_plan* plans, int n, int size, std::vector<AugLayout>* layouts,
                    int* n_steps, size_t* steps_off, size_t* plans_off, size_t* sums_off, size_t* upload_end, size_t* total) {
  VDK_REQUIRE(images && plans && n > 0 && size > 0, "vdk_augment: bad arguments");
  layouts->resize(n);
  int entries = 0;
  for (int i = 0; i < n; ++i) {
    const int w = images[i].width, h = images[i].height;
    const vdk_aug_plan& P = plans[i];
    VDK_REQUIRE(w > 0 && h > 0 && images[i].offset >= 0, "vdk_augment: bad image %d (%d x %d)", i, w, h);
    VDK_REQUIRE(P.n_ops >= 0 && P.n_ops <= VDK_AUG_MAX_OPS, "vdk_augment: image %d has %d ops (at most %d)", i, P.n_ops, VDK_AUG_MAX_OPS);
    for (int k = 0; k < P.n_ops; ++k) {
      const vdk_aug_op& op = P.ops[k];
      VDK_REQUIRE(op.kind >= VDK_AUG_BRIGHTNESS && op.kind <= VDK_AUG_HFLIP, "vdk_augment: image %d op %d: unknown kind %d", i, k, op.kind);
      VDK_REQUIRE(op.kind != VDK_AUG_CUTOUT || (op.n >= 0 && op.n <= VDK_AUG_MAX_HOLES), "vdk_augment: image %d: %d cutout holes", i, op.n);
      VDK_REQUIRE(op.kind != VDK_AUG_BLUR || (op.n >= 1 && op.n % 2 == 1 && op.n <= VDK_AUG_MAX_KERNEL && op.n / 2 < w && op.n / 2 < h),
                  "vdk_augment: image %d (%d x %d): blur kernel size %d needs an odd size <= %d whose half is below both sides", i,
                  w, h, op.n, VDK_AUG_MAX_KERNEL);
    }
    entries += P.n_ops;
    AugLayout& L = (*layouts)[i];
    if (P.resize == VDK_AUG_CROP_RESIZE) {
      memcpy(L.crop, P.crop, sizeof(L.crop));
      VDK_REQUIRE(L.crop[0] >= 0 && L.crop[1] >= 0 && L.crop[2] > 0 && L.crop[3] > 0 && L.crop[0] + L.crop[2] <= w &&
                  L.crop[1] + L.crop[3] <= h, "vdk_augment: image %d (%d x %d): crop box outside the image", i, w, h);
      L.pre.new_w = L.pre.new_h = size;
      L.pre.left = L.pre.top = 0;
      L.pre.filter = kResampleBilinear;
    } else {
      VDK_REQUIRE(P.resize == VDK_AUG_RESIZE_PAD_BILINEAR || P.resize == VDK_AUG_RESIZE_PAD_NEAREST, "vdk_augment: image %d: "
                  "unknown resize %d", i, P.resize);
      L.crop[0] = L.crop[1] = 0; L.crop[2] = w; L.crop[3] = h;
      resized_shape(w, h, size, &L.pre);
      VDK_REQUIRE(L.pre.new_w > 0 && L.pre.new_h > 0, "vdk_augment: image %d (%d x %d) collapses to an empty side at size %d", i, w,
                  h, size);
      L.pre.filter = P.resize == VDK_AUG_RESIZE_PAD_NEAREST ? kResampleNearest : kResampleBilinear;
    }
  }
  int steps = 0;
  for (int i = 0; i < n; ++i) steps = std::max(steps, plans[i].n_ops);
  *n_steps = steps;
  size_t off = up256p(static_cast<size_t>(n) * sizeof(PreImage));
  *steps_off = off;  off += up256p(static_cast<size_t>(entries) * sizeof(AugStep));
  *plans_off = off;  off += up256p(static_cast<size_t>(n) * sizeof(vdk_aug_plan));
  *sums_off = off;   off += up256p(static_cast<size_t>(entries) * sizeof(unsigned long long));
  for (int i = 0; i < n; ++i) {
    AugLayout& L = (*layouts)[i];
    off = layout_tables(L.crop[2], L.crop[3], off, &L.pre);
  }
  *upload_end = off;
  for (int i = 0; i < n; ++i) {
    AugLayout& L = (*layouts)[i];
    const size_t img = up256p(static_cast<size_t>(images[i].width) * images[i].height * 3);
    L.buf[0] = off;  off += plans[i].n_ops > 0 ? img : 0;
    L.buf[1] = off;  off += plans[i].n_ops > 1 ? img : 0;
    L.pre.tmp = off; off += up256p(static_cast<size_t>(L.crop[3]) * L.pre.new_w * 3);
  }
  *total = off;
  return VDK_OK;
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_augment_workspace_bytes(const vdk_image_desc* images, const vdk_aug_plan* plans, int n, int size) {
  std::vector<AugLayout> layouts;
  int n_steps = 0;
  size_t steps_off, plans_off, sums_off, upload_end, total = 0;
  if (aug_plan(images, plans, n, size, &layouts, &n_steps, &steps_off, &plans_off, &sums_off, &upload_end, &total) != VDK_OK) return 0;
  return total;
}

extern "C" int vdk_augment_batch(const uint8_t* packed, const vdk_image_desc* images, const vdk_aug_plan* plans, int n, int size,
                                 const float* mean, const float* std_, float* out, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  VDK_REQUIRE(packed && mean && std_ && out, "vdk_augment: bad arguments");
  VDK_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_augment: workspace must be 256-byte aligned");
  std::vector<AugLayout> layouts;
  int n_steps = 0;
  size_t steps_off, plans_off, sums_off, upload_end, total = 0;
  int rc = aug_plan(images, plans, n, size, &layouts, &n_steps, &steps_off, &plans_off, &sums_off, &upload_end, &total);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(workspace_bytes >= total, "vdk_augment: workspace too small");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  std::vector<uint8_t> host(upload_end, 0);  // zero contrast sums included
  memcpy(host.data() + plans_off, plans, static_cast<size_t>(n) * sizeof(vdk_aug_plan));
  const vdk_aug_plan* dplans = reinterpret_cast<const vdk_aug_plan*>(ws + plans_off);
  AugStep* steps = reinterpret_cast<AugStep*>(host.data() + steps_off);
  unsigned long long* dsums = reinterpret_cast<unsigned long long*>(ws + sums_off);
  // stage k = the k-th op of every image that has one; the image's current buffer starts at its packed source
  std::vector<const uint8_t*> cur(n);
  for (int i = 0; i < n; ++i) cur[i] = packed + images[i].offset;
  std::vector<int> stage_begin(n_steps + 1, 0);
  std::vector<int64_t> stage_max(n_steps, 0);
  int e = 0;
  for (int k = 0; k < n_steps; ++k) {
    stage_begin[k] = e;
    for (int i = 0; i < n; ++i) {
      if (plans[i].n_ops <= k) continue;
      AugStep& st = steps[e];
      st.in = cur[i];
      st.out = ws + layouts[i].buf[k & 1];
      st.op = &dplans[i].ops[k];
      st.sum = dsums + e;
      st.w = images[i].width;
      st.h = images[i].height;
      cur[i] = st.out;
      stage_max[k] = std::max<int64_t>(stage_max[k], static_cast<int64_t>(st.w) * st.h);
      ++e;
    }
  }
  stage_begin[n_steps] = e;
  PreImage* desc = reinterpret_cast<PreImage*>(host.data());
  int64_t max_tmp = 0;
  for (int i = 0; i < n; ++i) {
    const AugLayout& L = layouts[i];
    const int w = images[i].width;
    desc[i] = describe(L.pre, cur[i] + (static_cast<size_t>(L.crop[1]) * w + L.crop[0]) * 3, w, L.crop[2], L.crop[3], ws);
    fill_tables(L.crop[2], L.crop[3], L.pre, host.data());
    max_tmp = std::max<int64_t>(max_tmp, static_cast<int64_t>(L.crop[3]) * L.pre.new_w);
  }
  VDK_CUDA_OK(cudaMemcpyAsync(ws, host.data(), upload_end, cudaMemcpyHostToDevice, s));
  VDK_CUDA_OK(cudaStreamSynchronize(s));  // `host` is pageable and goes out of scope: the copy must have left it
  const AugStep* dsteps = reinterpret_cast<const AugStep*>(ws + steps_off);
  for (int k = 0; k < n_steps; ++k) {
    const int count = stage_begin[k + 1] - stage_begin[k];
    const int bx = static_cast<int>(std::min<int64_t>((stage_max[k] + 255) / 256, 1024));
    bool contrast = false;
    for (int i = 0; i < n; ++i) contrast |= plans[i].n_ops > k && plans[i].ops[k].kind == VDK_AUG_CONTRAST;
    if (contrast) {
      aug_luma_sum_kernel<<<dim3(std::min(bx, 128), count), 256, 0, s>>>(dsteps + stage_begin[k]);
      VDK_CUDA_OK(cudaGetLastError());
    }
    aug_stage_kernel<<<dim3(bx, count), 256, 0, s>>>(dsteps + stage_begin[k]);
    VDK_CUDA_OK(cudaGetLastError());
  }
  return resample_launch(reinterpret_cast<const PreImage*>(ws), n, max_tmp, size, mean, std_, out, s);
}

extern "C" int vdk_augment_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_aug_op), sizeof(vdk_aug_plan)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}
