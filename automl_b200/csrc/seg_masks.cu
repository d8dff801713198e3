// Segmentation masks at each image's own size: per output pixel, the arg-max over the classes of
// the segmentation head's logits at the pixel's nearest cell of the letterboxed network input.
// The reference stops at the logits; its demo takes tf.argmax(pred, -1) (tf2/segmentation.py:25-27)
// at the network resolution.  Nearest sampling in integer arithmetic keeps masks bit-exact:
//   cell_y = min(((2y + 1) * scaled_h) / (2 * h * f), hs - 1)     (x alike, f = input / logits grid)
// so only cells of the scaled image, which sits top-left in the letterbox, are ever read.
// Memory-bound: at most n * hs * ws * ld * 2 bytes in (each cell is reused from L1 / L2 by the
// pixels that sample it), sum(h * w) bytes out.
#include "common.cuh"

namespace edet {

constexpr int kSegThreads = 256;   // output columns per CTA (one per thread)
constexpr int kSegRows = 16;       // output rows per CTA

struct SegImage {                  // edet_seg_mask_image
  long long offset;
  int h, w, scaled_h, scaled_w;
};
static_assert(sizeof(SegImage) == 24, "edet_seg_mask_image layout");

// First index of the maximum of C fp16 logits, np.argmax's rule: equal values keep the earlier
// class (+0 == -0), the first NaN wins outright.  `cell` is 16-byte aligned.
__device__ __forceinline__ int argmax_cell(const __half* cell, int c) {
  float best = 0.f;
  int idx = 0;
  for (int c0 = 0; c0 < c; c0 += 8) {
    float v[8];
    half8_to_float(__ldg(reinterpret_cast<const uint4*>(cell + c0)), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = c0 + j;
      if (k >= c) break;
      if (isnan(v[j])) return k;
      if (k == 0 || v[j] > best) {
        best = v[j];
        idx = k;
      }
    }
  }
  return idx;
}

// grid = (column blocks, row blocks, images); a CTA covers kSegRows rows (striding by the grid when
// the tallest image needs more than 65535 row blocks) of 256 columns of one image.  A thread walks
// down its column and recomputes the arg-max only when the sampled cell row changes.
__global__ void __launch_bounds__(kSegThreads)
seg_masks_kernel(const __half* __restrict__ logits, const SegImage* __restrict__ table,
                 uint8_t* __restrict__ out, int hs, int ws, int ld, int c, int f) {
  pdl_launch_dependents();
  pdl_wait_prior();        // the logits come from the previous kernel, the table from a copy
  __shared__ SegImage d;
  if (threadIdx.x < sizeof(SegImage) / 4)
    reinterpret_cast<int*>(&d)[threadIdx.x] =
        __ldg(reinterpret_cast<const int*>(table + blockIdx.z) + threadIdx.x);
  __syncthreads();
  const long long h = d.h, w = d.w;
  const long long x = static_cast<long long>(blockIdx.x) * kSegThreads + threadIdx.x;
  if (x >= w) return;
  const long long cx = min((2 * x + 1) * d.scaled_w / (2 * w * f), static_cast<long long>(ws - 1));
  const __half* col = logits + (static_cast<long long>(blockIdx.z) * hs * ws + cx) * ld;
  uint8_t* o = out + d.offset + x;
  for (long long y0 = static_cast<long long>(blockIdx.y) * kSegRows; y0 < h;
       y0 += static_cast<long long>(gridDim.y) * kSegRows) {
    const long long y_end = min(y0 + kSegRows, h);
    long long last = -1;
    int cls = 0;
    for (long long y = y0; y < y_end; ++y) {
      const long long cy = min((2 * y + 1) * d.scaled_h / (2 * h * f), static_cast<long long>(hs - 1));
      if (cy != last) {
        cls = argmax_cell(col + cy * ws * ld, c);
        last = cy;
      }
      o[y * w] = static_cast<uint8_t>(cls);
    }
  }
}

}  // namespace edet

extern "C" int edet_seg_masks(const edet_half* logits, int n, int hs, int ws, int ld,
                              int num_classes, int grid_factor, const edet_seg_mask_image* table,
                              int max_h, int max_w, uint8_t* out, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(logits && table && out, "seg_masks: null pointer");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && hs > 0 && ws > 0 && grid_factor > 0 && max_h > 0 && max_w > 0,
                 "seg_masks: bad shape (n=%d logits %dx%d f=%d masks up to %dx%d)", n, hs, ws,
                 grid_factor, max_h, max_w);
  EDET_CHECK_ARG(num_classes >= 1 && num_classes <= 256,
                 "seg_masks: num_classes=%d must be in [1, 256] (uint8 masks)", num_classes);
  EDET_CHECK_ARG(ld >= num_classes && ld % 8 == 0,
                 "seg_masks: ld=%d must be a multiple of 8 and >= num_classes=%d", ld, num_classes);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(logits) % 16 == 0 &&
                     reinterpret_cast<uintptr_t>(table) % 8 == 0,
                 "seg_masks: logits must be 16-byte aligned, table 8-byte aligned");
  const dim3 grid(ceil_div(max_w, kSegThreads), min(ceil_div(max_h, kSegRows), 65535), n);
  EDET_CHECK_CUDA(launch_pdl(seg_masks_kernel, grid, dim3(kSegThreads), 0, as_stream(stream),
                             reinterpret_cast<const __half*>(logits),
                             reinterpret_cast<const SegImage*>(table), out, hs, ws, ld,
                             num_classes, grid_factor));
  return EDET_OK;
}
