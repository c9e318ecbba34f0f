// preprocess.cu — the eval-time image transform of the CBIR / face path on the device, for a batch of decoded RGB images of
// different sizes: ResizeAndPadding2Square(size) -> ToTensor -> Normalize.
//
// Replaces, per image, dataset/transforms.py:325-365 (PIL `Image.resize(..., BILINEAR)` + `ImageOps.expand` with black borders),
// :466-468 (T.ToTensor) and :474-477 (T.Normalize) — the `val.augment` list of configs/faceX/{face,cbir}.yaml that every gallery
// and query image passes through before FeatureExtractor.extract_cbir (models/faceX/face_model.py:120-144).
//
// Byte work, bit-exact: Pillow's 8-bit resampling (src/libImaging/Resample.c: separable, horizontal then vertical, uint8
// intermediate image, 22-bit fixed-point coefficients from a double-precision triangle filter whose support scales with the
// reduction factor) is restated on the host for the coefficient tables (a few hundred doubles per image) and on the device for
// the two passes; the float tail is IEEE fp32 division / subtraction exactly as torch evaluates ToTensor and Normalize.
// HBM-bound: one read of the packed uint8 images, one uint8 intermediate, one fp32 CHW write.  The resampler (resample.h) is
// shared with the training pipeline (augment.cu), which adds crop boxes and NEAREST tables.
#include "resample.h"
#include "vdk_host.h"

#include <cmath>
#include <cstring>
#include <vector>

namespace vdk {

constexpr int kPrecisionBits = 32 - 8 - 2;

// Resample.c precompute_coeffs + normalize_coeffs_8bpc for the bilinear (triangle, support 1) filter
static int resize_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& kk) {
  const double scale = static_cast<double>(in_size) / static_cast<double>(out_size);
  const double filterscale = scale > 1.0 ? scale : 1.0;
  const double support = 1.0 * filterscale;
  const int kmax = static_cast<int>(std::ceil(support)) * 2 + 1;
  bounds.assign(static_cast<size_t>(out_size) * 2, 0);
  kk.assign(static_cast<size_t>(out_size) * kmax, 0);
  std::vector<double> w(kmax);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    const int n = xmax - xmin;
    double ww = 0.0;
    for (int x = 0; x < n; ++x) {
      double a = (x + xmin - center + 0.5) * ss;
      if (a < 0.0) a = -a;
      const double v = a < 1.0 ? 1.0 - a : 0.0;
      w[x] = v;
      ww += v;
    }
    for (int x = 0; x < n; ++x) {
      if (ww != 0.0) w[x] /= ww;
      const double v = w[x] * static_cast<double>(1 << kPrecisionBits);
      kk[static_cast<size_t>(xx) * kmax + x] = w[x] < 0 ? static_cast<int>(v - 0.5) : static_cast<int>(v + 0.5);
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = n;
  }
  return kmax;
}

// Pillow's NEAREST resize (_imaging.c _resize: affine a = in_size / out_size as a float box width over an int, offset 0;
// Geometry.c ImagingScaleAffine: source index COORD(a * 0.5 + k * a), the position ACCUMULATED in double, one add per output
// pixel; an index outside the input leaves the fill, 0) as one-tap tables: a tap of weight 1 << kPrecisionBits copies the
// byte through either pass, no tap gives 0
static int nearest_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& kk) {
  const double a = static_cast<double>(static_cast<float>(in_size)) / out_size;
  bounds.assign(static_cast<size_t>(out_size) * 2, 0);
  kk.assign(static_cast<size_t>(out_size), 1 << kPrecisionBits);
  double pos = a * 0.5;
  for (int xx = 0; xx < out_size; ++xx) {
    const int xin = pos < 0.0 ? -1 : static_cast<int>(pos);
    if (xin >= 0 && xin < in_size) {
      bounds[2 * xx] = xin;
      bounds[2 * xx + 1] = 1;
    }
    pos += a;
  }
  return 1;
}

static int kmax_of(int in_size, int out_size, int filter) {
  if (filter == kResampleNearest) return 1;
  const double scale = static_cast<double>(in_size) / static_cast<double>(out_size);
  const double filterscale = scale > 1.0 ? scale : 1.0;
  return static_cast<int>(std::ceil(1.0 * filterscale)) * 2 + 1;
}

void resized_shape(int w, int h, int size, PreLayout* L) {
  const double scale_factor = static_cast<double>(size) / static_cast<double>(w > h ? w : h);
  L->new_w = static_cast<int>(w * scale_factor);
  L->new_h = static_cast<int>(h * scale_factor);
  // python's floor division for the (possibly zero) non-negative differences
  L->left = (size - L->new_w) / 2;
  L->top = (size - L->new_h) / 2;
}

size_t layout_tables(int w, int h, size_t off, PreLayout* L) {
  L->kmax_x = kmax_of(w, L->new_w, L->filter);
  L->kmax_y = kmax_of(h, L->new_h, L->filter);
  L->xb = off;  off += up256p(static_cast<size_t>(L->new_w) * 2 * sizeof(int));
  L->kx = off;  off += up256p(static_cast<size_t>(L->new_w) * L->kmax_x * sizeof(int));
  L->yb = off;  off += up256p(static_cast<size_t>(L->new_h) * 2 * sizeof(int));
  L->ky = off;  off += up256p(static_cast<size_t>(L->new_h) * L->kmax_y * sizeof(int));
  return off;
}

void fill_tables(int w, int h, const PreLayout& L, uint8_t* host_ws) {
  std::vector<int> bounds, kk;
  auto coeffs = L.filter == kResampleNearest ? nearest_coeffs : resize_coeffs;
  coeffs(w, L.new_w, bounds, kk);
  memcpy(host_ws + L.xb, bounds.data(), bounds.size() * sizeof(int));
  memcpy(host_ws + L.kx, kk.data(), kk.size() * sizeof(int));
  coeffs(h, L.new_h, bounds, kk);
  memcpy(host_ws + L.yb, bounds.data(), bounds.size() * sizeof(int));
  memcpy(host_ws + L.ky, kk.data(), kk.size() * sizeof(int));
}

PreImage describe(const PreLayout& L, const uint8_t* src, int stride, int w, int h, uint8_t* ws) {
  PreImage d;
  d.src = src;
  d.stride = stride;
  d.tmp = ws + L.tmp;
  d.xb = reinterpret_cast<const int*>(ws + L.xb);
  d.kx = reinterpret_cast<const int*>(ws + L.kx);
  d.yb = reinterpret_cast<const int*>(ws + L.yb);
  d.ky = reinterpret_cast<const int*>(ws + L.ky);
  d.w = w; d.h = h;
  d.new_w = L.new_w; d.new_h = L.new_h; d.left = L.left; d.top = L.top; d.kmax_x = L.kmax_x; d.kmax_y = L.kmax_y;
  return d;
}

__device__ __forceinline__ uint8_t clip8(int v) { return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// horizontal pass: one thread per (row, output column), 3 channels
__global__ void __launch_bounds__(256) pre_horizontal_kernel(const PreImage* __restrict__ images) {
  const PreImage im = images[blockIdx.y];
  const int64_t total = static_cast<int64_t>(im.h) * im.new_w;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / im.new_w), xx = static_cast<int>(i - static_cast<int64_t>(y) * im.new_w);
    const int xmin = im.xb[2 * xx], n = im.xb[2 * xx + 1];
    const int* k = im.kx + static_cast<size_t>(xx) * im.kmax_x;
    const uint8_t* s = im.src + (static_cast<size_t>(y) * im.stride + xmin) * 3;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int x = 0; x < n; ++x) {
      const int c = k[x];
      a0 += s[3 * x] * c;
      a1 += s[3 * x + 1] * c;
      a2 += s[3 * x + 2] * c;
    }
    uint8_t* d = im.tmp + (static_cast<size_t>(y) * im.new_w + xx) * 3;
    d[0] = clip8(a0 >> kPrecisionBits);
    d[1] = clip8(a1 >> kPrecisionBits);
    d[2] = clip8(a2 >> kPrecisionBits);
  }
}

// vertical pass + centring in the black square + ToTensor + Normalize: one thread per output pixel, CHW fp32
__global__ void __launch_bounds__(256) pre_vertical_kernel(const PreImage* __restrict__ images, int size, float m0, float m1, float m2,
                                                           float s0, float s1, float s2, float* __restrict__ out) {
  const PreImage im = images[blockIdx.y];
  const int64_t plane = static_cast<int64_t>(size) * size;
  float* o = out + static_cast<int64_t>(blockIdx.y) * 3 * plane;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int oy = static_cast<int>(i / size), ox = static_cast<int>(i - static_cast<int64_t>(oy) * size);
    const int yy = oy - im.top, xx = ox - im.left;
    int v0 = 0, v1 = 0, v2 = 0;  // the border is black BEFORE normalisation (ImageOps.expand fill (0,0,0))
    if (yy >= 0 && yy < im.new_h && xx >= 0 && xx < im.new_w) {
      const int ymin = im.yb[2 * yy], n = im.yb[2 * yy + 1];
      const int* k = im.ky + static_cast<size_t>(yy) * im.kmax_y;
      const uint8_t* s = im.tmp + (static_cast<size_t>(ymin) * im.new_w + xx) * 3;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int y = 0; y < n; ++y) {
        const int c = k[y];
        const uint8_t* r = s + static_cast<size_t>(y) * im.new_w * 3;
        a0 += r[0] * c;
        a1 += r[1] * c;
        a2 += r[2] * c;
      }
      v0 = clip8(a0 >> kPrecisionBits);
      v1 = clip8(a1 >> kPrecisionBits);
      v2 = clip8(a2 >> kPrecisionBits);
    }
    // ToTensor: uint8 -> fp32 / 255;  Normalize: (x - mean) / std — IEEE round-to-nearest, no contraction
    o[i] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v0), 255.0f), m0), s0);
    o[plane + i] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v1), 255.0f), m1), s1);
    o[2 * plane + i] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v2), 255.0f), m2), s2);
  }
}

int resample_launch(const PreImage* dimg, int n, int64_t max_tmp, int size, const float* mean, const float* std_, float* out,
                    cudaStream_t s) {
  const int bx = static_cast<int>(std::min<int64_t>((max_tmp + 255) / 256, 4096));
  pre_horizontal_kernel<<<dim3(bx, n), 256, 0, s>>>(dimg);
  VDK_CUDA_OK(cudaGetLastError());
  const int by = static_cast<int>(std::min<int64_t>((static_cast<int64_t>(size) * size + 255) / 256, 4096));
  pre_vertical_kernel<<<dim3(by, n), 256, 0, s>>>(dimg, size, mean[0], mean[1], mean[2], std_[0], std_[1], std_[2], out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// workspace = [descriptors | coefficient tables of every image | intermediate images]: the first two parts are built on the
// host and uploaded in one copy (`*tables_end` bytes), the intermediate images exist on the device only
static int plan(const vdk_image_desc* images, int n, int size, std::vector<PreLayout>* layouts, size_t* tables_end, size_t* total) {
  size_t off = up256p(static_cast<size_t>(n) * sizeof(PreImage));
  layouts->resize(n);
  for (int i = 0; i < n; ++i) {
    const int w = images[i].width, h = images[i].height;
    VDK_REQUIRE(w > 0 && h > 0 && images[i].offset >= 0, "vdk_preprocess: bad image %d (%d x %d)", i, w, h);
    PreLayout& L = (*layouts)[i];
    resized_shape(w, h, size, &L);
    VDK_REQUIRE(L.new_w > 0 && L.new_h > 0, "vdk_preprocess: image %d (%d x %d) collapses to an empty side at size %d", i, w, h, size);
    L.filter = kResampleBilinear;
    off = layout_tables(w, h, off, &L);
  }
  *tables_end = off;
  for (int i = 0; i < n; ++i) {
    PreLayout& L = (*layouts)[i];
    L.tmp = off;
    off += up256p(static_cast<size_t>(images[i].height) * L.new_w * 3);
  }
  *total = off;
  return VDK_OK;
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_preprocess_workspace_bytes(const vdk_image_desc* images, int n, int size) {
  if (!images || n <= 0 || size <= 0) return 0;
  std::vector<PreLayout> layouts;
  size_t tables_end = 0, total = 0;
  if (plan(images, n, size, &layouts, &tables_end, &total) != VDK_OK) return 0;
  return total;
}

extern "C" int vdk_preprocess_resize_pad_normalize(const uint8_t* packed, const vdk_image_desc* images, int n, int size,
                                                   const float* mean, const float* std_, float* out, void* workspace,
                                                   size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(packed && images && mean && std_ && out && n > 0 && size > 0, "vdk_preprocess: bad arguments");
  VDK_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_preprocess: workspace must be 256-byte aligned");
  std::vector<PreLayout> layouts;
  size_t tables_end = 0, total = 0;
  int rc = plan(images, n, size, &layouts, &tables_end, &total);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(workspace_bytes >= total, "vdk_preprocess: workspace too small");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  std::vector<uint8_t> host(tables_end, 0);  // descriptors + coefficient tables
  PreImage* desc = reinterpret_cast<PreImage*>(host.data());
  int64_t max_h = 0;
  for (int i = 0; i < n; ++i) {
    const PreLayout& L = layouts[i];
    const int w = images[i].width, h = images[i].height;
    desc[i] = describe(L, packed + images[i].offset, w, w, h, ws);
    fill_tables(w, h, L, host.data());
    max_h = std::max<int64_t>(max_h, static_cast<int64_t>(h) * L.new_w);
  }
  VDK_CUDA_OK(cudaMemcpyAsync(ws, host.data(), tables_end, cudaMemcpyHostToDevice, s));
  VDK_CUDA_OK(cudaStreamSynchronize(s));  // `host` is pageable and goes out of scope: the copy must have left it
  return resample_launch(reinterpret_cast<const PreImage*>(ws), n, max_h, size, mean, std_, out, s);
}
