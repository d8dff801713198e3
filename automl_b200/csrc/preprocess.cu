// Serving pre-process on the device: HWC image -> (x - mean) / std -> aspect-preserving bilinear
// resize (TF2 tf.image.resize: half-pixel centres, no antialias) -> zero pad to the network input.
// Replaces inference.image_preprocess (inference.py:37-56) and EfficientDetModel._preprocessing
// (tf2/efficientdet_keras.py:920-954) -> DetectionInputProcessor.normalize_image /
// set_scale_factors_to_output_size / resize_and_crop_image (dataloader.py:59-65, 115-142), which
// cast any input to float32 first: uint8 images (serving) and float32 images (the Keras model).  A
// ragged uint8 request (images of different sizes, batch_image_preprocess inference.py:68-109) is
// one launch over a descriptor table.  The mirrored variant also writes each image flipped left to
// right (test-time augmentation, tf2/postprocess.py:560-573 un-mirrors about the network input
// width) from the same values.
// Memory-bound: 3*h*w (uint8) or 12*h*w (float32) bytes in, 12*H*W bytes out per image.
#include "common.cuh"

namespace edet {

constexpr int kPreRows = 8;   // output rows per CTA

struct PreImage {               // edet_preprocess_image
  long long offset;
  int h, w, scaled_h, scaled_w;
};
static_assert(sizeof(PreImage) == 24, "edet_preprocess_image layout");

// (x - mean) / std only takes 3 x 256 distinct values for uint8 input: each CTA builds the table
// once with the same IEEE division the reference order implies (normalise, then interpolate), so
// the twelve divisions per pixel become twelve shared-memory lookups -- bit-identical results.
__device__ __forceinline__ void build_lut(float (&lut)[3][256], float3 mean, float3 stddev) {
  const float m[3] = {mean.x, mean.y, mean.z}, sd[3] = {stddev.x, stddev.y, stddev.z};
  for (int i = threadIdx.x; i < 3 * 256; i += 256) {
    const int c = i >> 8, v = i & 255;
    lut[c][v] = __fdiv_rn(__fsub_rn(static_cast<float>(v), m[c]), sd[c]);
  }
}

// Tap loaders: the normalised value of channel c of the pixel at `p`.
struct LutTaps {                // uint8 images: the CTA's table
  using T = uint8_t;
  const float (&lut)[3][256];
  __device__ __forceinline__ float operator()(const uint8_t* p, int c) const {
    return lut[c][__ldg(p + c)];
  }
};

struct FloatTaps {              // float32 images: the operations that build the table, per tap
  using T = float;
  float m[3], sd[3];
  __device__ __forceinline__ FloatTaps(float3 mean, float3 stddev)
      : m{mean.x, mean.y, mean.z}, sd{stddev.x, stddev.y, stddev.z} {}
  __device__ __forceinline__ float operator()(const float* p, int c) const {
    return __fdiv_rn(__fsub_rn(__ldg(p + c), m[c]), sd[c]);
  }
};

// This thread's column of the CTA's kPreRows output rows of one image: `img` is the image's first
// element, `o_img` its [out_h, out_w, 3] output.  Every kernel runs exactly this, so an image gives
// the same bits whichever launch it is part of, and a float32 image of integral values 0..255 the
// bits of the same uint8 image.  kMirror: each value is also stored at column out_w - 1 - x of
// `o_mir`, the image's [out_h, out_w, 3] mirrored output.
template <bool kMirror = false, class Taps>
__device__ __forceinline__ void preprocess_rows(const Taps& taps, const typename Taps::T* img,
                                                float* o_img, int h, int w, int out_h, int out_w,
                                                int scaled_h, int scaled_w, float* o_mir = nullptr) {
  using T = typename Taps::T;
  const int x = blockIdx.x * 256 + threadIdx.x;
  if (x >= out_w) return;
  const int y_end = min(out_h, static_cast<int>(blockIdx.y + 1) * kPreRows);
  for (int y = blockIdx.y * kPreRows; y < y_end; ++y) {     // the table is shared by kPreRows rows
    float* o = o_img + (static_cast<size_t>(y) * out_w + x) * 3;
    float* om = nullptr;
    if constexpr (kMirror) om = o_mir + (static_cast<size_t>(y) * out_w + (out_w - 1 - x)) * 3;
    if (y >= scaled_h || x >= scaled_w) {   // pad_to_bounding_box zero padding
      o[0] = 0.f; o[1] = 0.f; o[2] = 0.f;
      if constexpr (kMirror) { om[0] = 0.f; om[1] = 0.f; om[2] = 0.f; }
      continue;
    }
    // tf.image.resize bilinear, half_pixel_centers: src = (dst + 0.5) * (in / out) - 0.5
    const float sy = static_cast<float>(h) / static_cast<float>(scaled_h);
    const float sx = static_cast<float>(w) / static_cast<float>(scaled_w);
    const float fy = __fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(y), 0.5f), sy), 0.5f);
    const float fx = __fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(x), 0.5f), sx), 0.5f);
    const float fy0 = floorf(fy), fx0 = floorf(fx);
    const int y0 = max(static_cast<int>(fy0), 0), y1 = min(static_cast<int>(ceilf(fy)), h - 1);
    const int x0 = max(static_cast<int>(fx0), 0), x1 = min(static_cast<int>(ceilf(fx)), w - 1);
    const float ly = __fsub_rn(fy, fy0), lx = __fsub_rn(fx, fx0);
    const T* p00 = img + (static_cast<size_t>(y0) * w + x0) * 3;
    const T* p01 = img + (static_cast<size_t>(y0) * w + x1) * 3;
    const T* p10 = img + (static_cast<size_t>(y1) * w + x0) * 3;
    const T* p11 = img + (static_cast<size_t>(y1) * w + x1) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      // normalise first (as the reference does), then interpolate
      const float v00 = taps(p00, c), v01 = taps(p01, c);
      const float v10 = taps(p10, c), v11 = taps(p11, c);
      const float top = __fadd_rn(v00, __fmul_rn(__fsub_rn(v01, v00), lx));
      const float bot = __fadd_rn(v10, __fmul_rn(__fsub_rn(v11, v10), lx));
      const float v = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), ly));
      o[c] = v;
      if constexpr (kMirror) om[c] = v;
    }
  }
}

// One thread per output column, kPreRows rows; grid = (x blocks, row blocks, images): no index
// division.  Images of one size, back to back.
__global__ void __launch_bounds__(256)
preprocess_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int h, int w,
                  int out_h, int out_w, int scaled_h, int scaled_w, float3 mean, float3 stddev) {
  __shared__ float lut[3][256];
  build_lut(lut, mean, stddev);
  __syncthreads();
  const int img = blockIdx.z;
  preprocess_rows(LutTaps{lut}, in + static_cast<size_t>(img) * h * w * 3,
                  out + static_cast<size_t>(img) * out_h * out_w * 3, h, w, out_h, out_w, scaled_h,
                  scaled_w);
}

// A ragged request: the same grid, each CTA reads its image's descriptor (byte offset into
// `packed`, size, scaled size) once into shared memory.
__global__ void __launch_bounds__(256)
preprocess_kernel(const uint8_t* __restrict__ packed, const PreImage* __restrict__ desc,
                  float* __restrict__ out, int out_h, int out_w, float3 mean, float3 stddev) {
  __shared__ float lut[3][256];
  __shared__ PreImage d;
  if (threadIdx.x < sizeof(PreImage) / 4)
    reinterpret_cast<int*>(&d)[threadIdx.x] =
        __ldg(reinterpret_cast<const int*>(desc + blockIdx.z) + threadIdx.x);
  build_lut(lut, mean, stddev);
  __syncthreads();
  preprocess_rows(LutTaps{lut}, packed + d.offset,
                  out + static_cast<size_t>(blockIdx.z) * out_h * out_w * 3, d.h, d.w, out_h, out_w,
                  d.scaled_h, d.scaled_w);
}

// A ragged request and its mirror: image i of the table to out[i] and, flipped on width, to
// out[n + i] (`mirror` = n * out_h * out_w * 3 elements further).  Same grid as the ragged launch.
__global__ void __launch_bounds__(256)
preprocess_kernel(const uint8_t* __restrict__ packed, const PreImage* __restrict__ desc,
                  float* __restrict__ out, long long mirror, int out_h, int out_w, float3 mean,
                  float3 stddev) {
  __shared__ float lut[3][256];
  __shared__ PreImage d;
  if (threadIdx.x < sizeof(PreImage) / 4)
    reinterpret_cast<int*>(&d)[threadIdx.x] =
        __ldg(reinterpret_cast<const int*>(desc + blockIdx.z) + threadIdx.x);
  build_lut(lut, mean, stddev);
  __syncthreads();
  float* o_img = out + static_cast<size_t>(blockIdx.z) * out_h * out_w * 3;
  preprocess_rows<true>(LutTaps{lut}, packed + d.offset, o_img, d.h, d.w, out_h, out_w,
                        d.scaled_h, d.scaled_w, o_img + mirror);
}

// A float32 batch of one size: the same grid as the uint8 launch, no table -- each tap is
// normalised where it is read (FloatTaps).  NaN and Inf pass through the arithmetic.
__global__ void __launch_bounds__(256)
preprocess_kernel(const float* __restrict__ in, float* __restrict__ out, int h, int w,
                  int out_h, int out_w, int scaled_h, int scaled_w, float3 mean, float3 stddev) {
  const int img = blockIdx.z;
  preprocess_rows(FloatTaps(mean, stddev), in + static_cast<size_t>(img) * h * w * 3,
                  out + static_cast<size_t>(img) * out_h * out_w * 3, h, w, out_h, out_w, scaled_h,
                  scaled_w);
}

// dataloader.py:115-127 (float32 arithmetic, truncation to int): the scale that fits an h x w
// image into out_h x out_w, and the scaled size.
static float fit_scale(int h, int w, int out_h, int out_w, int* scaled_h, int* scaled_w) {
  const float sy = static_cast<float>(out_h) / static_cast<float>(h);
  const float sx = static_cast<float>(out_w) / static_cast<float>(w);
  const float image_scale = sx < sy ? sx : sy;
  *scaled_h = static_cast<int>(static_cast<float>(h) * image_scale);
  *scaled_w = static_cast<int>(static_cast<float>(w) * image_scale);
  return image_scale;
}

}  // namespace edet

extern "C" int edet_preprocess(const uint8_t* in, float* out, int n, int h, int w, int out_h,
                               int out_w, const float* h_mean_rgb, const float* h_stddev_rgb,
                               float* h_image_scale, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(in && out && h_mean_rgb && h_stddev_rgb, "preprocess: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "preprocess: bad shape");
  int scaled_h, scaled_w;
  const float image_scale = fit_scale(h, w, out_h, out_w, &scaled_h, &scaled_w);
  EDET_CHECK_ARG(scaled_h > 0 && scaled_w > 0, "preprocess: image collapses to zero size");
  if (h_image_scale) *h_image_scale = 1.0f / image_scale;   // image_scale_to_original
  EDET_CHECK_ARG(n <= 65535, "preprocess: n must be <= 65535");
  preprocess_kernel<<<dim3(ceil_div(out_w, 256), ceil_div(out_h, kPreRows), n), 256, 0, as_stream(stream)>>>(
      in, out, h, w, out_h, out_w, scaled_h, scaled_w,
      make_float3(h_mean_rgb[0], h_mean_rgb[1], h_mean_rgb[2]),
      make_float3(h_stddev_rgb[0], h_stddev_rgb[1], h_stddev_rgb[2]));
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}

extern "C" int edet_preprocess_ragged(const uint8_t* packed, const edet_preprocess_image* desc,
                                      float* out, int n, int out_h, int out_w,
                                      const float* h_mean_rgb, const float* h_stddev_rgb,
                                      edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(packed && desc && out && h_mean_rgb && h_stddev_rgb,
                 "preprocess_ragged: null pointer");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && out_h > 0 && out_w > 0,
                 "preprocess_ragged: bad shape (n=%d out=%dx%d)", n, out_h, out_w);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(desc) % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
                 "preprocess_ragged: desc must be 8-byte aligned, out 4-byte aligned");
  preprocess_kernel<<<dim3(ceil_div(out_w, 256), ceil_div(out_h, kPreRows), n), 256, 0, as_stream(stream)>>>(
      packed, reinterpret_cast<const PreImage*>(desc), out, out_h, out_w,
      make_float3(h_mean_rgb[0], h_mean_rgb[1], h_mean_rgb[2]),
      make_float3(h_stddev_rgb[0], h_stddev_rgb[1], h_stddev_rgb[2]));
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}

extern "C" int edet_preprocess_mirrored(const uint8_t* packed, const edet_preprocess_image* desc,
                                        float* out, int n, int out_h, int out_w,
                                        const float* h_mean_rgb, const float* h_stddev_rgb,
                                        edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(packed && desc && out && h_mean_rgb && h_stddev_rgb,
                 "preprocess_mirrored: null pointer");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && out_h > 0 && out_w > 0,
                 "preprocess_mirrored: bad shape (n=%d out=%dx%d)", n, out_h, out_w);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(desc) % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
                 "preprocess_mirrored: desc must be 8-byte aligned, out 4-byte aligned");
  preprocess_kernel<<<dim3(ceil_div(out_w, 256), ceil_div(out_h, kPreRows), n), 256, 0, as_stream(stream)>>>(
      packed, reinterpret_cast<const PreImage*>(desc), out,
      static_cast<long long>(n) * out_h * out_w * 3, out_h, out_w,
      make_float3(h_mean_rgb[0], h_mean_rgb[1], h_mean_rgb[2]),
      make_float3(h_stddev_rgb[0], h_stddev_rgb[1], h_stddev_rgb[2]));
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}

extern "C" int edet_preprocess_float(const float* in, float* out, int n, int h, int w, int out_h,
                                     int out_w, const float* h_mean_rgb, const float* h_stddev_rgb,
                                     float* h_image_scale, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(in && out && h_mean_rgb && h_stddev_rgb, "preprocess_float: null pointer");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && h > 0 && w > 0 && out_h > 0 && out_w > 0,
                 "preprocess_float: bad shape (n=%d in=%dx%d out=%dx%d)", n, h, w, out_h, out_w);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(in) % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
                 "preprocess_float: in and out must be 4-byte aligned");
  int scaled_h, scaled_w;
  const float image_scale = fit_scale(h, w, out_h, out_w, &scaled_h, &scaled_w);
  EDET_CHECK_ARG(scaled_h > 0 && scaled_w > 0, "preprocess_float: image collapses to zero size");
  if (h_image_scale) *h_image_scale = 1.0f / image_scale;   // image_scale_to_original
  preprocess_kernel<<<dim3(ceil_div(out_w, 256), ceil_div(out_h, kPreRows), n), 256, 0, as_stream(stream)>>>(
      in, out, h, w, out_h, out_w, scaled_h, scaled_w,
      make_float3(h_mean_rgb[0], h_mean_rgb[1], h_mean_rgb[2]),
      make_float3(h_stddev_rgb[0], h_stddev_rgb[1], h_stddev_rgb[2]));
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}
