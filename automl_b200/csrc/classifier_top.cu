// Classification top of the EfficientNet V1 / V2 models: global average pooling of the head
// feature map and the Dense classifier (efficientnetv2/effnetv2_model.py Head.call :472-496,
// EffNetV2Model._build :571-578).  Both keep float32 from the pooled mean to the logits and sum
// in an order fixed by the shapes alone: row i of either output has the same bits whatever the
// batch size or the grid is.
#include "common.cuh"

namespace edet {

// ---- global average pooling --------------------------------------------------------------------
// One CTA per (image, slice of 32 channels).  Thread t owns the 8 channels of lane t & 3 (one
// 128-bit load per row) and the rows r, r + 64, r + 128, ... with r = t >> 2, summed in that order.
// The 64 row partials of a channel are then combined in a fixed tree: xor-shuffles over the 8 rows
// of a warp, then the 8 warps pairwise through shared memory.  Every 16-byte piece of the map is
// loaded by its own thread in at most ceil(hw / 64) rounds, so a single image (40 CTAs for 1280
// channels) already has all of its loads in flight at once.
constexpr int kPoolSlice = 32;                    // channels per CTA (64 bytes of each row)
constexpr int kPoolRows = 64;                     // row partials per channel
constexpr int kPoolThreads = kPoolRows * kPoolSlice / 8;

__global__ void __launch_bounds__(kPoolThreads)
global_avg_pool_kernel(const __half* __restrict__ x, float* __restrict__ out, int hw, int c,
                       float inv_hw) {
  pdl_launch_dependents();
  pdl_wait_prior();
  __shared__ float part[kPoolThreads / 32][kPoolSlice];
  const int img = blockIdx.y, c0 = blockIdx.x * kPoolSlice;
  const int piece = threadIdx.x & 3, row = threadIdx.x >> 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ch = c0 + piece * 8;
  float acc[8] = {};
  if (ch < c) {
    const __half* p = x + (static_cast<size_t>(img) * hw + row) * c + ch;
    for (int r = row; r < hw; r += kPoolRows, p += static_cast<size_t>(kPoolRows) * c) {
      float f[8];
      half8_to_float(ldg_nc_v4(p), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += f[i];
    }
  }
#pragma unroll
  for (int o = 4; o < 32; o <<= 1)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
  if (lane < 4) {
#pragma unroll
    for (int i = 0; i < 8; ++i) part[warp][piece * 8 + i] = acc[i];
  }
  __syncthreads();
  if (threadIdx.x < kPoolSlice && c0 + threadIdx.x < c) {
    const int j = threadIdx.x;
    const float s = ((part[0][j] + part[1][j]) + (part[2][j] + part[3][j])) +
                    ((part[4][j] + part[5][j]) + (part[6][j] + part[7][j]));
    out[static_cast<size_t>(img) * c + c0 + j] = s * inv_hw;
  }
}

// ---- Dense classifier --------------------------------------------------------------------------
// One CTA per tile of 8 classes.  Its weight rows are converted to float32 once into shared memory
// (k in chunks of 2560, one chunk for every registered model); then each warp takes two images at
// a time, lane l multiplying the input columns 128 i + 4 l .. + 3 (i ascending) into 8 class
// sums per image, which an xor-shuffle tree combines.  A later k chunk adds to what the same
// lane stored for the chunk before, so the order per (image, class) depends on k alone.
constexpr int kDenseClasses = 8;
constexpr int kDenseChunk = 2560;                 // k per shared-memory pass: 80 KB of float32
constexpr int kDenseWarps = 8;
constexpr int kDenseImages = 2;                   // images per warp pass (register blocking)

__global__ void __launch_bounds__(kDenseWarps * 32)
dense_kernel(const float* __restrict__ x, const __half* __restrict__ wt,
             const float* __restrict__ bias, float* __restrict__ out, int n, int k, int m) {
  pdl_launch_dependents();
  pdl_wait_prior();
  extern __shared__ __align__(16) float sw[];     // [kDenseClasses][len]
  const int m0 = blockIdx.x * kDenseClasses;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k0 = 0; k0 < k; k0 += kDenseChunk) {
    const int len = min(kDenseChunk, k - k0);
    if (k0 > 0) __syncthreads();                  // every warp is done with the previous chunk
    for (int i = threadIdx.x; i < kDenseClasses * (len / 8); i += blockDim.x) {
      const int cls = i / (len / 8), col = (i - cls * (len / 8)) * 8;
      float f[8] = {};
      if (m0 + cls < m)
        half8_to_float(ldg_nc_v4(wt + static_cast<size_t>(m0 + cls) * k + k0 + col), f);
      float4* dst = reinterpret_cast<float4*>(sw + cls * len + col);
      dst[0] = make_float4(f[0], f[1], f[2], f[3]);
      dst[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
    __syncthreads();
    for (int img = warp * kDenseImages; img < n; img += kDenseWarps * kDenseImages) {
      float acc[kDenseImages][kDenseClasses] = {};
      const float* xr[kDenseImages];
#pragma unroll
      for (int j = 0; j < kDenseImages; ++j)      // a missing second image re-reads the first
        xr[j] = x + static_cast<size_t>(min(img + j, n - 1)) * k + k0;
      for (int col = lane * 4; col < len; col += 128) {
        float4 a[kDenseImages];
#pragma unroll
        for (int j = 0; j < kDenseImages; ++j) a[j] = __ldg(reinterpret_cast<const float4*>(xr[j] + col));
#pragma unroll
        for (int cls = 0; cls < kDenseClasses; ++cls) {
          const float4 w = *reinterpret_cast<const float4*>(sw + cls * len + col);
#pragma unroll
          for (int j = 0; j < kDenseImages; ++j) {
            acc[j][cls] = fmaf(a[j].x, w.x, acc[j][cls]);
            acc[j][cls] = fmaf(a[j].y, w.y, acc[j][cls]);
            acc[j][cls] = fmaf(a[j].z, w.z, acc[j][cls]);
            acc[j][cls] = fmaf(a[j].w, w.w, acc[j][cls]);
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int j = 0; j < kDenseImages; ++j)
#pragma unroll
          for (int cls = 0; cls < kDenseClasses; ++cls)
            acc[j][cls] += __shfl_xor_sync(0xffffffffu, acc[j][cls], o);
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < kDenseImages; ++j)
#pragma unroll
          for (int cls = 0; cls < kDenseClasses; ++cls)
            if (img + j < n && m0 + cls < m) {
              float* o = out + static_cast<size_t>(img + j) * m + m0 + cls;
              *o = (k0 == 0 ? bias[m0 + cls] : *o) + acc[j][cls];
            }
      }
    }
  }
}

}  // namespace edet

extern "C" int edet_global_avg_pool(const edet_half* x, float* out, int n, int hw, int c,
                                    edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(x && out, "global_avg_pool: null pointer");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && hw > 0 && c > 0,
                 "global_avg_pool: bad shape (n=%d hw=%d c=%d)", n, hw, c);
  EDET_CHECK_ARG(c % 8 == 0, "global_avg_pool: c=%d must be a multiple of 8", c);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
                 "global_avg_pool: x must be 16-byte aligned, out 4-byte aligned");
  EDET_CHECK_CUDA(launch_pdl(global_avg_pool_kernel, dim3(ceil_div(c, kPoolSlice), n),
                             dim3(kPoolThreads), 0, as_stream(stream),
                             reinterpret_cast<const __half*>(x), out, hw, c,
                             1.0f / static_cast<float>(hw)));
  return EDET_OK;
}

extern "C" int edet_dense(const float* x, const edet_half* wt, const float* bias, float* out, int n,
                          int k, int num_classes, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(x && wt && bias && out, "dense: null pointer");
  EDET_CHECK_ARG(n > 0 && k > 0 && num_classes > 0, "dense: bad shape (n=%d k=%d num_classes=%d)", n,
                 k, num_classes);
  EDET_CHECK_ARG(k % 8 == 0, "dense: k=%d must be a multiple of 8", k);
  EDET_CHECK_ARG((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(wt)) % 16 == 0 &&
                     (reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(out)) % 4 == 0,
                 "dense: x and wt must be 16-byte aligned, bias and out 4-byte aligned");
  const int smem = kDenseClasses * (k < kDenseChunk ? k : kDenseChunk) * static_cast<int>(sizeof(float));
  static int smem_done[kMaxDevices];
  const int rc = ensure_dynamic_smem(dense_kernel, smem, smem_done);
  if (rc != EDET_OK) return rc;
  EDET_CHECK_CUDA(launch_pdl(dense_kernel, dim3(ceil_div(num_classes, kDenseClasses)),
                             dim3(kDenseWarps * 32), static_cast<size_t>(smem), as_stream(stream), x,
                             reinterpret_cast<const __half*>(wt), bias, out, n, k, num_classes));
  return EDET_OK;
}
