// Stem: Conv2D 3x3 stride 2 'SAME', 3 -> cout (24..64), + folded BN + activation.
// Reads the float32 NHWC image the reference feeds the network (efficientnet_model.py:526-527)
// and writes NHWC fp16.  bytes = 12*n*h*w + 2*n*ho*wo*cout; 27 MACs per output element, so the
// arithmetic runs as fp32 FMAs on channel pairs.
//
// One thread = two horizontally adjacent output pixels x 16 output channels (8 channel pairs);
// the [27][16] weight slab of the channel half sits in shared memory as float2 pairs and is read
// as warp-wide broadcasts, each read feeding both pixels.
#include "common.cuh"

namespace edet {

constexpr int kStemThreads = 128;
constexpr int kStemCh = 16;   // output channels per thread

template <int ACT>
__global__ void __launch_bounds__(kStemThreads)
stem_kernel(const float* __restrict__ in, __half* __restrict__ out, const __half* __restrict__ w,
            const float* __restrict__ bias, int h, int wd, int ho, int wo, int cout, int pad_t,
            int pad_l) {
  pdl_launch_dependents();
  __shared__ __align__(16) float2 ws[27][kStemCh / 2];
  __shared__ __align__(16) float2 bs[kStemCh / 2];
  const int c0 = blockIdx.y * kStemCh;
  const int cn = min(kStemCh, cout - c0);            // channels of this slab that exist (mult. of 8)
  for (int i = threadIdx.x; i < 27 * kStemCh; i += kStemThreads) {
    const int t = i / kStemCh, c = i % kStemCh;
    reinterpret_cast<float*>(&ws[t][0])[c] = c < cn ? __half2float(w[t * cout + c0 + c]) : 0.f;
  }
  for (int i = threadIdx.x; i < kStemCh; i += kStemThreads)
    reinterpret_cast<float*>(&bs[0])[i] = i < cn ? bias[c0 + i] : 0.f;
  __syncthreads();
  pdl_wait_prior();   // weights staged above; the image is read below
  const int n = blockIdx.z;
  const int wo2 = (wo + 1) >> 1;                      // pixel pairs per output row
  const float* in_n = in + static_cast<size_t>(n) * h * wd * 3;
  // grid-stride loop over pixel pairs: the weight slab is staged once per CTA
  for (int pp = blockIdx.x * kStemThreads + threadIdx.x; pp < ho * wo2;
       pp += gridDim.x * kStemThreads) {
    const int oy = pp / wo2, ox = (pp - oy * wo2) * 2;
    // input patch: 3 rows x 5 columns x 3 channels (columns 0..2 feed pixel 0, 2..4 pixel 1)
    float x[3][5][3];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy * 2 - pad_t + ky;
      const bool row_ok = iy >= 0 && iy < h;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const int ix = ox * 2 - pad_l + j;
        const bool ok = row_ok && ix >= 0 && ix < wd;
        const float* px = in_n + (static_cast<size_t>(iy) * wd + ix) * 3;
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) x[ky][j][ci] = ok ? __ldg(px + ci) : 0.f;
      }
    }
    float2 acc0[kStemCh / 2], acc1[kStemCh / 2];
#pragma unroll
    for (int p = 0; p < kStemCh / 2; ++p) {
      acc0[p] = bs[p];
      acc1[p] = bs[p];
    }
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const int t = (ky * 3 + kx) * 3 + ci;
          const float2 a0 = make_float2(x[ky][kx][ci], x[ky][kx][ci]);
          const float2 a1 = make_float2(x[ky][kx + 2][ci], x[ky][kx + 2][ci]);
#pragma unroll
          for (int q = 0; q < kStemCh / 4; ++q) {
            const float4 w4 = *reinterpret_cast<const float4*>(&ws[t][2 * q]);
            const float2 wa = make_float2(w4.x, w4.y), wb = make_float2(w4.z, w4.w);
            acc0[2 * q] = ffma2_rn(a0, wa, acc0[2 * q]);
            acc0[2 * q + 1] = ffma2_rn(a0, wb, acc0[2 * q + 1]);
            acc1[2 * q] = ffma2_rn(a1, wa, acc1[2 * q]);
            acc1[2 * q + 1] = ffma2_rn(a1, wb, acc1[2 * q + 1]);
          }
        }
      }
    }
    __half* o0 = out + ((static_cast<size_t>(n) * ho + oy) * wo + ox) * cout + c0;
#pragma unroll
    for (int g = 0; g < kStemCh / 8; ++g) {
      if (g * 8 < cn) {
        float f0[8], f1[8];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          float2 r0 = acc0[g * 4 + p], r1 = acc1[g * 4 + p];
          apply_act4<ACT>(r0, r1);
          f0[2 * p] = r0.x; f0[2 * p + 1] = r0.y;
          f1[2 * p] = r1.x; f1[2 * p + 1] = r1.y;
        }
        *reinterpret_cast<uint4*>(o0 + g * 8) = float_to_half8(f0);
        if (ox + 1 < wo) *reinterpret_cast<uint4*>(o0 + cout + g * 8) = float_to_half8(f1);
      }
    }
  }
}

namespace stemtc {   // stem_tc.cu
bool eligible(int cout);
int run(const float* in, __half* out, const __half* w, const float* bias, int n, int h, int wd,
        int cout, int act, cudaStream_t stream);
}  // namespace stemtc
}  // namespace edet

extern "C" int edet_stem_conv(const float* in, edet_half* out, const edet_half* w,
                              const float* bias, int n, int h, int wd, int cout, int act,
                              edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(in && out && w && bias, "stem: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && wd > 0, "stem: bad shape");
  EDET_CHECK_ARG(cout > 0 && cout % 8 == 0, "stem: cout must be a multiple of 8 (got %d)", cout);
  const __half* hw = reinterpret_cast<const __half*>(w);
  __half* ho_p = reinterpret_cast<__half*>(out);
  cudaStream_t s = as_stream(stream);
  // default: implicit GEMM on the tensor cores (stem_tc.cu); "stem_impl" = 1 keeps this kernel
  if (option_stem_impl() != 1 && stemtc::eligible(cout) &&
      (act == EDET_ACT_SWISH || act == EDET_ACT_RELU6 || act == EDET_ACT_NONE))
    return stemtc::run(in, ho_p, hw, bias, n, h, wd, cout, act, s);
  const int ho = ceil_div(h, 2), wo = ceil_div(wd, 2);
  const int pad_t = same_pad_before(h, 3, 2), pad_l = same_pad_before(wd, 3, 2);
  // ~8 pixel pairs per thread: staging the weights is amortised, yet there are enough CTAs
  dim3 grid(ceil_div(ceil_div(ho * ((wo + 1) / 2), kStemThreads), 8), ceil_div(cout, kStemCh), n);
  cudaError_t err = cudaSuccess;
  if (act == EDET_ACT_SWISH)
    err = launch_pdl(stem_kernel<EDET_ACT_SWISH>, grid, dim3(kStemThreads), 0, s, in, ho_p, hw, bias, h, wd, ho, wo, cout, pad_t, pad_l);
  else if (act == EDET_ACT_RELU6)
    err = launch_pdl(stem_kernel<EDET_ACT_RELU6>, grid, dim3(kStemThreads), 0, s, in, ho_p, hw, bias, h, wd, ho, wo, cout, pad_t, pad_l);
  else if (act == EDET_ACT_NONE)
    err = launch_pdl(stem_kernel<EDET_ACT_NONE>, grid, dim3(kStemThreads), 0, s, in, ho_p, hw, bias, h, wd, ho, wo, cout, pad_t, pad_l);
  else {
    set_error("stem: unsupported activation %d", act);
    return EDET_ERR_UNSUPPORTED;
  }
  EDET_CHECK_CUDA(err);
  return EDET_OK;
}
