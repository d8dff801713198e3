// Classification eval pre-process of the EfficientNet V1 / V2 models on the device: uint8 HWC
// images of any size (a ragged request in one launch) -> center crop -> resize to S x S ->
// normalise, written as the float32 NHWC network input.  Two recipes:
//   bilinear (efficientnetv2/preprocessing.py:58-70, 153): tf.image.resize (half-pixel centres) of
//     the crop, then (x - 128) / 128;
//   bicubic  (efficientnetv2/preprocess_legacy.py:110-127, 184-244): TF1 resize_bicubic
//     (align_corners = half_pixel_centers = False, TF's CPU kernel: 1024-entry coefficient table,
//     a = -0.75, clamped taps) of the crop, then (x - mean) / stddev with the ImageNet statistics.
// The host computes each crop window (edet_cls_image), so the kernel has no integer rules.
// Memory-bound: the crop footprint in, 12 S^2 bytes out per image.
#include "common.cuh"

namespace edet {

constexpr int kClsCols = 128;   // output columns per CTA (one thread each)
constexpr int kClsRows = 8;     // output rows per CTA
constexpr int kBicubicTableSize = 1024;

struct ClsImage {               // edet_cls_image
  long long offset;
  int h, w, y0, x0, crop_h, crop_w;
};
static_assert(sizeof(ClsImage) == 32, "edet_cls_image layout");

__device__ __forceinline__ float px(const uint8_t* p) { return static_cast<float>(__ldg(p)); }

// grid = (column blocks, row blocks, images).  The descriptor is read once per CTA.
__global__ void __launch_bounds__(kClsCols)
cls_preprocess_kernel(const uint8_t* __restrict__ images, const ClsImage* __restrict__ desc,
                      int size, int mode, const float* __restrict__ table, float* __restrict__ out) {
  __shared__ ClsImage d;
  if (threadIdx.x < sizeof(ClsImage) / 4)
    reinterpret_cast<int*>(&d)[threadIdx.x] =
        __ldg(reinterpret_cast<const int*>(desc + blockIdx.z) + threadIdx.x);
  __syncthreads();
  const int x = blockIdx.x * kClsCols + threadIdx.x;
  if (x >= size) return;
  const int y_end = min(size, static_cast<int>(blockIdx.y + 1) * kClsRows);
  const uint8_t* base = images + d.offset;
  const size_t row_bytes = static_cast<size_t>(d.w) * 3;
  float* o = out + ((static_cast<size_t>(blockIdx.z) * size + blockIdx.y * kClsRows) * size + x) * 3;
  const float inv_out = static_cast<float>(size);
  if (mode == EDET_CLS_BILINEAR) {
    // src = (dst + 0.5) * (in / out) - 0.5, lower = max(floor, 0), upper = min(ceil, in - 1)
    const float sx = static_cast<float>(d.crop_w) / inv_out;
    const float sy = static_cast<float>(d.crop_h) / inv_out;
    const float fx = __fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(x), 0.5f), sx), 0.5f);
    const float fx0 = floorf(fx);
    const int xa = d.x0 + max(static_cast<int>(fx0), 0);
    const int xb = d.x0 + min(static_cast<int>(ceilf(fx)), d.crop_w - 1);
    const float lx = __fsub_rn(fx, fx0);
    for (int y = blockIdx.y * kClsRows; y < y_end; ++y, o += static_cast<size_t>(size) * 3) {
      const float fy = __fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(y), 0.5f), sy), 0.5f);
      const float fy0 = floorf(fy);
      const int ya = d.y0 + max(static_cast<int>(fy0), 0);
      const int yb = d.y0 + min(static_cast<int>(ceilf(fy)), d.crop_h - 1);
      const float ly = __fsub_rn(fy, fy0);
      const uint8_t* p00 = base + ya * row_bytes + xa * 3;
      const uint8_t* p01 = base + ya * row_bytes + xb * 3;
      const uint8_t* p10 = base + yb * row_bytes + xa * 3;
      const uint8_t* p11 = base + yb * row_bytes + xb * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v00 = px(p00 + c), v01 = px(p01 + c), v10 = px(p10 + c), v11 = px(p11 + c);
        const float top = __fadd_rn(v00, __fmul_rn(__fsub_rn(v01, v00), lx));
        const float bot = __fadd_rn(v10, __fmul_rn(__fsub_rn(v11, v10), lx));
        const float v = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), ly));
        o[c] = __fdiv_rn(__fsub_rn(v, 128.0f), 128.0f);      // preprocessing.py:153
      }
    }
    return;
  }
  // TF1 resize_bicubic, legacy scaler: src = dst * (in / out), i = floor(src), offset =
  // lrintf((src - i) * 1024) (round half to even), weights t[2o+1], t[2o], t[2(1024-o)],
  // t[2(1024-o)+1] on the taps i-1 .. i+2 clamped to [0, in-1].
  const float mean[3] = {static_cast<float>(0.485 * 255), static_cast<float>(0.456 * 255),
                         static_cast<float>(0.406 * 255)};
  const float stddev[3] = {static_cast<float>(0.229 * 255), static_cast<float>(0.224 * 255),
                           static_cast<float>(0.225 * 255)};
  float wx[4];
  int cx[4];
  {
    const float src = __fmul_rn(static_cast<float>(x), static_cast<float>(d.crop_w) / inv_out);
    const float fi = floorf(src);
    const int off = __float2int_rn(__fmul_rn(__fsub_rn(src, fi), static_cast<float>(kBicubicTableSize)));
    wx[0] = __ldg(table + 2 * off + 1);
    wx[1] = __ldg(table + 2 * off);
    wx[2] = __ldg(table + 2 * (kBicubicTableSize - off));
    wx[3] = __ldg(table + 2 * (kBicubicTableSize - off) + 1);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      cx[j] = (d.x0 + min(max(static_cast<int>(fi) - 1 + j, 0), d.crop_w - 1)) * 3;
  }
  const float sy = static_cast<float>(d.crop_h) / inv_out;
  for (int y = blockIdx.y * kClsRows; y < y_end; ++y, o += static_cast<size_t>(size) * 3) {
    const float src = __fmul_rn(static_cast<float>(y), sy);
    const float fi = floorf(src);
    const int off = __float2int_rn(__fmul_rn(__fsub_rn(src, fi), static_cast<float>(kBicubicTableSize)));
    const float wy[4] = {__ldg(table + 2 * off + 1), __ldg(table + 2 * off),
                         __ldg(table + 2 * (kBicubicTableSize - off)),
                         __ldg(table + 2 * (kBicubicTableSize - off) + 1)};
    const uint8_t* r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      r[j] = base + (d.y0 + min(max(static_cast<int>(fi) - 1 + j, 0), d.crop_h - 1)) * row_bytes;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float col[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {   // vertical first at each x tap, products summed left to right
        float s = __fmul_rn(px(r[0] + cx[j] + c), wy[0]);
        s = __fadd_rn(s, __fmul_rn(px(r[1] + cx[j] + c), wy[1]));
        s = __fadd_rn(s, __fmul_rn(px(r[2] + cx[j] + c), wy[2]));
        col[j] = __fadd_rn(s, __fmul_rn(px(r[3] + cx[j] + c), wy[3]));
      }
      float v = __fmul_rn(wx[0], col[0]);
      v = __fadd_rn(v, __fmul_rn(wx[1], col[1]));
      v = __fadd_rn(v, __fmul_rn(wx[2], col[2]));
      v = __fadd_rn(v, __fmul_rn(wx[3], col[3]));
      o[c] = __fdiv_rn(__fsub_rn(v, mean[c]), stddev[c]);   // preprocess_legacy.py:239-243
    }
  }
}

}  // namespace edet

extern "C" int edet_cls_preprocess(const uint8_t* images, const edet_cls_image* desc, int n,
                                   int size, int mode, const float* bicubic_table, float* out,
                                   edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(images && desc && out, "cls_preprocess: null pointer");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && size > 0, "cls_preprocess: bad shape (n=%d size=%d)", n, size);
  EDET_CHECK_ARG(mode == EDET_CLS_BILINEAR || mode == EDET_CLS_BICUBIC, "cls_preprocess: bad mode %d",
                 mode);
  EDET_CHECK_ARG(mode != EDET_CLS_BICUBIC || bicubic_table,
                 "cls_preprocess: the bicubic mode needs the coefficient table");
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(desc) % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
                 "cls_preprocess: desc must be 8-byte aligned, out 4-byte aligned");
  cls_preprocess_kernel<<<dim3(ceil_div(size, kClsCols), ceil_div(size, kClsRows), n), kClsCols, 0,
                          as_stream(stream)>>>(images, reinterpret_cast<const ClsImage*>(desc), size,
                                               mode, bicubic_table, out);
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}
