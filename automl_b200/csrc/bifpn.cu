// BiFPN node kernel: resample each input to the node resolution (identity / TF1 nearest
// upsample / 'SAME' max-pool), fast-normalised weighted fusion, activation, depthwise 3x3 'SAME'
// -- one pass, the fused map only ever lives in shared memory.  Plus the stand-alone max-pool
// used to create the extra P6.. levels.
//
// Memory-bound (SURVEY.md 8d): bytes = 2*n*c*(sum_inputs h_i*w_i + h*w) + 2*9*c.
#include "fuse_common.cuh"

namespace edet {

constexpr int kFuseThreads = 256;
constexpr int kFuseTH = 8, kFuseTW = 16;   // output tile
constexpr int kFuseCB = 32;                // channels per CTA
// smem pixel pitch of the fused tile: 36 floats = 9 x 16 bytes.  An ODD number of 16-byte units
// makes both the phase-1 stores (lanes = 4 channel groups x 2 pixels per quarter warp) and the
// phase-2 loads (4 channel groups x 2 columns) hit 8 distinct bank groups.
constexpr int kFusePitch = kFuseCB + 4;

// SIG: compile-time input signature (fuse_common.cuh: kSigGeneric or one of the three shapes a
// BiFPN cell has).  With the modes known at compile time the loads of ALL inputs of an item
// are issued before any of them is consumed (the generic loop serialises one global round trip
// per input: the kernel is latency bound, ncu long-scoreboard 5.0 issue-slots per instruction).
template <int ACT, int SIG>
__global__ void __launch_bounds__(kFuseThreads)
fuse_dw_kernel(const FuseParams p, const float* __restrict__ dw_w, __half* __restrict__ out,
               int h, int wd, int c, int chunks) {
  pdl_launch_dependents();
  constexpr int HT = kFuseTH + 2, WT = kFuseTW + 2, G = kFuseCB / 8;
  static_assert(G == 4 && kFuseTH * kFuseTW * G == 2 * kFuseThreads, "phase-2 mapping");
  __shared__ __align__(16) float fused[HT * WT * kFusePitch];
  __shared__ __align__(16) float wsm[9 * kFuseCB];
  const int n = blockIdx.z / chunks;
  const int c0 = (blockIdx.z % chunks) * kFuseCB;
  const int y0 = blockIdx.y * kFuseTH, x0 = blockIdx.x * kFuseTW;
  const int groups = min(G, (c - c0) >> 3);
  // fp32 depthwise weights of this channel chunk (constants: fetched before the PDL wait)
  for (int i = threadIdx.x; i < 9 * kFuseCB; i += kFuseThreads) {
    const int tap = i / kFuseCB, ch = i % kFuseCB;
    wsm[i] = (c0 + ch < c) ? __ldg(dw_w + static_cast<size_t>(tap) * c + c0 + ch) : 0.f;
  }
  pdl_wait_prior();

  // ---- phase 1: fused + activated map for the tile and its 1-pixel halo -------------------
  for (int item = threadIdx.x; item < HT * WT * G; item += kFuseThreads) {
    const int g = item & (G - 1), pix = item >> 2;
    const int ty = pix / WT, tx = pix - ty * WT;
    const int y = y0 + ty - 1, x = x0 + tx - 1;
    float2 acc[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[e] = make_float2(0.f, 0.f);
    if (g < groups && y >= 0 && y < h && x >= 0 && x < wd) {
      const int ch = c0 + g * 8;
      if (SIG == kSigGeneric) {
        for (int i = 0; i < p.n_inputs; ++i) {
          const FuseIn& fi = p.in[i];
          const __half* base = fi.ptr + static_cast<size_t>(n) * fi.h * fi.w * c;
          float v[8];
          resample8(fi, base, c, y, x, ch, v);
          const float2 w2 = make_float2(fi.weight, fi.weight);
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[e] = ffma2_rn(make_float2(v[2 * e], v[2 * e + 1]), w2, acc[e]);
        }
      } else {
        // all raw loads first (same values, same accumulation order as the generic loop)
        constexpr int NI = sig_inputs(SIG);
        uint4 raw0[9], raw1[9], raw2[9];
        int taps0 = 0, taps1 = 0, taps2 = 0;
        auto img = [&](int i) { return p.in[i].ptr + static_cast<size_t>(n) * p.in[i].h * p.in[i].w * c; };
        taps0 = resample_raw<sig_mode(SIG, 0)>(p.in[0], img(0), c, y, x, ch, raw0);
        taps1 = resample_raw<sig_mode(SIG, 1)>(p.in[1], img(1), c, y, x, ch, raw1);
        if (NI == 3) taps2 = resample_raw<sig_mode(SIG, 2)>(p.in[2], img(2), c, y, x, ch, raw2);
        auto accumulate = [&](const float* v, float weight) {
          const float2 w2 = make_float2(weight, weight);
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[e] = ffma2_rn(make_float2(v[2 * e], v[2 * e + 1]), w2, acc[e]);
        };
        float v[8];
        resample_reduce<sig_mode(SIG, 0)>(raw0, taps0, v);
        accumulate(v, p.in[0].weight);
        resample_reduce<sig_mode(SIG, 1)>(raw1, taps1, v);
        accumulate(v, p.in[1].weight);
        if (NI == 3) {
          resample_reduce<sig_mode(SIG, 2)>(raw2, taps2, v);
          accumulate(v, p.in[2].weight);
        }
      }
      apply_act4<ACT>(acc[0], acc[1]);
      apply_act4<ACT>(acc[2], acc[3]);
    }
    float4* dst = reinterpret_cast<float4*>(fused + pix * kFusePitch + g * 8);
    dst[0] = make_float4(acc[0].x, acc[0].y, acc[1].x, acc[1].y);
    dst[1] = make_float4(acc[2].x, acc[2].y, acc[3].x, acc[3].y);
  }
  __syncthreads();

  // ---- phase 2: depthwise 3x3, one thread = 8 channels x 2 vertically adjacent pixels --------
  {
    const int g = threadIdx.x & (G - 1);
    const int tx = (threadIdx.x >> 2) & (kFuseTW - 1);
    const int ty = (threadIdx.x >> 6) * 2;            // rows ty, ty + 1
    const int x = x0 + tx;
    if (g >= groups || x >= wd || y0 + ty >= h) return;
    float2 acc[2][4];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[r][e] = make_float2(0.f, 0.f);
    // taps in (ky, kx) order for each output row, so the sums match the scalar fmaf chain
#pragma unroll
    for (int iy = 0; iy < 4; ++iy) {
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4* src = reinterpret_cast<const float4*>(fused + ((ty + iy) * WT + tx + kx) * kFusePitch + g * 8);
        const float4 a = src[0], b = src[1];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int ky = iy - r;
          if (ky >= 0 && ky < 3) {
            const float4* wp = reinterpret_cast<const float4*>(wsm + (ky * 3 + kx) * kFuseCB + g * 8);
            const float4 w0 = wp[0], w1 = wp[1];
            acc[r][0] = ffma2_rn(make_float2(a.x, a.y), make_float2(w0.x, w0.y), acc[r][0]);
            acc[r][1] = ffma2_rn(make_float2(a.z, a.w), make_float2(w0.z, w0.w), acc[r][1]);
            acc[r][2] = ffma2_rn(make_float2(b.x, b.y), make_float2(w1.x, w1.y), acc[r][2]);
            acc[r][3] = ffma2_rn(make_float2(b.z, b.w), make_float2(w1.z, w1.w), acc[r][3]);
          }
        }
      }
    }
    const int ch = c0 + g * 8;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int y = y0 + ty + r;
      if (y < h) {
        const float o[8] = {acc[r][0].x, acc[r][0].y, acc[r][1].x, acc[r][1].y,
                            acc[r][2].x, acc[r][2].y, acc[r][3].x, acc[r][3].y};
        *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(n) * h + y) * wd + x) * c + ch) =
            float_to_half8(o);
      }
    }
  }
}

__global__ void __launch_bounds__(256)
max_pool_kernel(const __half* __restrict__ in, __half* __restrict__ out, int h, int wd, int c,
                int ho, int wo, int pool_h, int pool_w, int stride_h, int stride_w, int pad_t,
                int pad_l, long long total) {
  pdl_launch_dependents();
  pdl_wait_prior();
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = c >> 3;
  const int g = static_cast<int>(idx % cg);
  long long r = idx / cg;
  const int ox = static_cast<int>(r % wo);
  r /= wo;
  const int oy = static_cast<int>(r % ho);
  const int n = static_cast<int>(r / ho);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = -CUDART_INF_F;
  const __half* base = in + static_cast<size_t>(n) * h * wd * c;
  for (int py = 0; py < pool_h; ++py) {
    const int sy = oy * stride_h - pad_t + py;
    if (sy < 0 || sy >= h) continue;
    for (int px = 0; px < pool_w; ++px) {
      const int sx = ox * stride_w - pad_l + px;
      if (sx < 0 || sx >= wd) continue;
      float t[8];
      load8(base, h, wd, c, sy, sx, g * 8, t);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], t[e]);
    }
  }
  *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(n) * ho + oy) * wo + ox) * c + g * 8) =
      float_to_half8(v);
}

}  // namespace edet

extern "C" int edet_fuse_dw(const edet_fuse_input* h_inputs, int n_inputs, const float* dw_w,
                            edet_half* out, int n, int h, int wd, int c, int act,
                            edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(dw_w && out, "fuse_dw: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && wd > 0 && c > 0 && c % 8 == 0, "fuse_dw: bad shape");
  FuseParams p;
  if (int rc = fill_fuse_params(h_inputs, n_inputs, h, wd, "fuse_dw", &p)) return rc;
  const int chunks = ceil_div(c, kFuseCB);
  dim3 grid(ceil_div(wd, kFuseTW), ceil_div(h, kFuseTH), n * chunks);
  const float* hw = dw_w;
  __half* ho = reinterpret_cast<__half*>(out);
  cudaStream_t s = as_stream(stream);
  cudaError_t err = cudaSuccess;
  const int sig = fuse_signature(p);
#define EDET_FUSE_DW(ACT)                                                                          \
  switch (sig) {                                                                                   \
    case kSigSameUp: err = launch_pdl(fuse_dw_kernel<ACT, kSigSameUp>, grid, dim3(kFuseThreads), 0, s, p, hw, ho, h, wd, c, chunks); break; \
    case kSigSameSameDown: err = launch_pdl(fuse_dw_kernel<ACT, kSigSameSameDown>, grid, dim3(kFuseThreads), 0, s, p, hw, ho, h, wd, c, chunks); break; \
    case kSigSameDown: err = launch_pdl(fuse_dw_kernel<ACT, kSigSameDown>, grid, dim3(kFuseThreads), 0, s, p, hw, ho, h, wd, c, chunks); break; \
    default: err = launch_pdl(fuse_dw_kernel<ACT, kSigGeneric>, grid, dim3(kFuseThreads), 0, s, p, hw, ho, h, wd, c, chunks); break; \
  }
  switch (act) {
    case EDET_ACT_SWISH: EDET_FUSE_DW(EDET_ACT_SWISH); break;
    case EDET_ACT_RELU6: EDET_FUSE_DW(EDET_ACT_RELU6); break;
    case EDET_ACT_RELU: EDET_FUSE_DW(EDET_ACT_RELU); break;
    case EDET_ACT_HSWISH: EDET_FUSE_DW(EDET_ACT_HSWISH); break;
    case EDET_ACT_NONE: EDET_FUSE_DW(EDET_ACT_NONE); break;
    default:
      set_error("fuse_dw: bad activation %d", act);
      return EDET_ERR_INVALID;
  }
#undef EDET_FUSE_DW
  EDET_CHECK_CUDA(err);
  return EDET_OK;
}

extern "C" int edet_max_pool(const edet_half* in, edet_half* out, int n, int h, int wd, int c,
                             int pool_h, int pool_w, int stride_h, int stride_w,
                             edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(in && out, "max_pool: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && wd > 0 && c > 0 && c % 8 == 0, "max_pool: bad shape");
  EDET_CHECK_ARG(pool_h > 0 && pool_w > 0 && stride_h > 0 && stride_w > 0, "max_pool: bad window");
  const int ho = ceil_div(h, stride_h), wo = ceil_div(wd, stride_w);
  const long long total = static_cast<long long>(n) * ho * wo * (c >> 3);
  const int blocks = static_cast<int>((total + 255) / 256);
  EDET_CHECK_CUDA(launch_pdl(max_pool_kernel, dim3(blocks), dim3(256), 0, as_stream(stream),
                             reinterpret_cast<const __half*>(in), reinterpret_cast<__half*>(out), h, wd,
                             c, ho, wo, pool_h, pool_w, stride_h, stride_w,
                             same_pad_before(h, pool_h, stride_h),
                             same_pad_before(wd, pool_w, stride_w), total));
  return EDET_OK;
}
