// resample.h — Pillow's 8-bit resize of a crop box, padded into a square and written as ToTensor + Normalize, shared by the
// eval pipeline (preprocess.cu) and the training pipeline (augment.cu).
//
// One image's work is a crop box of a packed uint8 RGB image (row stride in pixels) resized to new_w x new_h and placed at
// (left, top) of a size x size black square.  BILINEAR is Pillow's separable triangle-filter resample (Resample.c);
// NEAREST is Pillow's nearest resize (_imaging.c _resize -> Geometry.c ImagingScaleAffine), expressed as one-tap tables of the
// same two passes, so both filters run through the same kernels.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace vdk {

enum ResampleFilter { kResampleBilinear = 0, kResampleNearest = 1 };

struct PreImage {          // device-side view of one image's work
  const uint8_t* src;      // first pixel of the crop box, rows `stride` pixels apart, [h][w][3]
  uint8_t* tmp;            // [h][new_w][3]   horizontal pass output
  const int* xb;           // [new_w][2] (first input column, tap count)
  const int* kx;           // [new_w][kmax_x]
  const int* yb;           // [new_h][2]
  const int* ky;           // [new_h][kmax_y]
  int w, h, new_w, new_h, left, top, kmax_x, kmax_y, stride;
};

struct PreLayout {
  int new_w, new_h, left, top, kmax_x, kmax_y, filter;
  size_t tmp, xb, kx, yb, ky;  // offsets in the workspace
};

static inline size_t up256p(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

// ResizeAndPadding2Square arithmetic (dataset/transforms.py:344-357): python float `size / max_side`, int() truncation,
// centred; sets new_w, new_h, left, top
void resized_shape(int w, int h, int size, PreLayout* L);
// Assigns the coefficient-table offsets of a w x h box resized to L->new_w x L->new_h with L->filter, from `off` on;
// returns the end offset
size_t layout_tables(int w, int h, size_t off, PreLayout* L);
// Writes those tables into the host image of the workspace
void fill_tables(int w, int h, const PreLayout& L, uint8_t* host_ws);
// The device descriptor of one image whose tables and intermediate live in the workspace `ws`
PreImage describe(const PreLayout& L, const uint8_t* src, int stride, int w, int h, uint8_t* ws);
// Horizontal pass, then vertical pass + padding + ToTensor + Normalize into out[n][3][size][size]; `max_tmp` is the largest
// h * new_w of the batch
int resample_launch(const PreImage* dimg, int n, int64_t max_tmp, int size, const float* mean, const float* std_, float* out,
                    cudaStream_t s);

}  // namespace vdk
