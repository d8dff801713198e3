// Depthwise k x k convolution ('SAME', NHWC fp16) + bias + activation, with the SE squeeze
// (per-image spatial sums) produced in the same pass, and the SE gate kernel.
//
// Memory-bound op (SURVEY.md 8d): algorithmic bytes per launch =
//   2 * n * c * (h*w + ho*wo) + 2 * k*k*c      (the SE squeeze adds 8*n*c bytes of atomics).
//
// Mapping: see depthwise_kernel below (register tile of 1 channel pair x 4 columns x ROWS rows,
// fp32 accumulation with FFMA on channel pairs; coalesced 128-byte warp accesses along the channel axis).
#include "common.cuh"

namespace edet {

constexpr int kDwThreads = 128;
constexpr int kDwTW = 4;  // adjacent output columns per thread
constexpr double kSeFixedScale = 1048576.0;  // 2^20: fixed-point scale of the SE squeeze sums

template <int K, int S>
struct DwCfg {
  static constexpr int ROWS = (S == 2 || K == 5) ? 4 : 8;   // output rows per thread
  static constexpr int IN_ROWS = (ROWS - 1) * S + K;        // input rows touched
  static constexpr int IN_COLS = (kDwTW - 1) * S + K;       // input columns touched
};

// Register tiling: one thread owns ONE channel pair (a half2, so a warp reads 128 contiguous
// bytes of the NHWC row), kDwTW adjacent output columns and ROWS output rows.  Every loaded
// input is converted to fp32 once and reused by up to K*K taps from registers; the arithmetic is
// fp32 FMAs on the channel pair.  Rationale: a 5x5 depthwise conv
// needs 25 MACs per output element, more than the scalar FFMA pipe can issue at the HBM rate,
// and without the column tiling the half->float conversions of the kx re-reads dominate.
template <int K, int S, int ACT, bool HAS_BIAS, bool HAS_SE>
__global__ void __launch_bounds__(kDwThreads, (K == 3 || S == 1) ? 4 : 3)
depthwise_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                 const float* __restrict__ w, const float* __restrict__ bias,
                 long long* __restrict__ se_sum, int h, int wd, int c, int ho, int wo, int pad_t,
                 int pad_l) {
  pdl_launch_dependents();
  constexpr int TW = kDwTW;
  constexpr int ROWS = DwCfg<K, S>::ROWS;
  constexpr int IN_ROWS = DwCfg<K, S>::IN_ROWS;
  constexpr int IN_COLS = DwCfg<K, S>::IN_COLS;
  const int cp_count = c >> 1;                         // channel pairs per pixel
  const int xt_count = (wo + TW - 1) / TW;
  const int e = blockIdx.x * kDwThreads + threadIdx.x;  // (x tile, channel pair) flattened
  const int n = blockIdx.z;
  const int oy0 = blockIdx.y * ROWS;
  const bool active = e < xt_count * cp_count;
  const int xt = active ? e / cp_count : 0;
  const int cp = active ? e - xt * cp_count : 0;
  const int ox0 = xt * TW;

  float2 ssum = make_float2(0.f, 0.f);
  if (!active) pdl_wait_prior();

  if (active) {
    const float2* w2 = reinterpret_cast<const float2*>(w);   // fp32 taps [k*k][c]
    float2 wreg[K * K];
#pragma unroll
    for (int t = 0; t < K * K; ++t) wreg[t] = __ldg(w2 + t * cp_count + cp);
    pdl_wait_prior();   // the (constant) weights above were fetched during the previous kernel's tail

    float2 acc[ROWS][TW];
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int tx = 0; tx < TW; ++tx) acc[r][tx] = make_float2(0.f, 0.f);

    const __half2* in2 = reinterpret_cast<const __half2*>(in) +
                         static_cast<size_t>(n) * h * wd * cp_count + cp;
    const int iy0 = oy0 * S - pad_t;
    const int ix0 = ox0 * S - pad_l;
    // Interior tiles (the vast majority) need no bounds predicate on any of their loads/stores.
    const bool interior = iy0 >= 0 && iy0 + IN_ROWS <= h && ix0 >= 0 && ix0 + IN_COLS <= wd &&
                          oy0 + ROWS <= ho && ox0 + TW <= wo;
    const int row_stride = wd * cp_count;
    const __half2* rowp = in2 + (iy0 * wd + ix0) * cp_count;   // may point outside; guarded below

    if (interior) {
      // software pipeline: the raw loads run two input rows ahead of the arithmetic, so each
      // thread keeps 3 rows of loads in flight (this kernel is latency bound otherwise)
      __half2 raw[3][IN_COLS];
#pragma unroll
      for (int pre = 0; pre < 2; ++pre) {
#pragma unroll
        for (int j = 0; j < IN_COLS; ++j) raw[pre][j] = __ldg(rowp + j * cp_count);
        rowp += row_stride;
      }
#pragma unroll
      for (int ir = 0; ir < IN_ROWS; ++ir) {
        if (ir + 2 < IN_ROWS) {
#pragma unroll
          for (int j = 0; j < IN_COLS; ++j) raw[(ir + 2) % 3][j] = __ldg(rowp + j * cp_count);
          rowp += row_stride;
        }
        float2 xv[IN_COLS];
#pragma unroll
        for (int j = 0; j < IN_COLS; ++j) xv[j] = __half22float2(raw[ir % 3][j]);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          const int ky = ir - r * S;
          if (ky >= 0 && ky < K) {
#pragma unroll
            for (int tx = 0; tx < TW; ++tx)
#pragma unroll
              for (int kx = 0; kx < K; ++kx)
                acc[r][tx] = ffma2_rn(xv[tx * S + kx], wreg[ky * K + kx], acc[r][tx]);
          }
        }
      }
    } else {
      unsigned col_ok = 0;
#pragma unroll
      for (int j = 0; j < IN_COLS; ++j)
        if (ix0 + j >= 0 && ix0 + j < wd) col_ok |= 1u << j;
#pragma unroll
      for (int ir = 0; ir < IN_ROWS; ++ir) {
        const int iy = iy0 + ir;
        const bool row_ok = (iy >= 0) && (iy < h);
        float2 xv[IN_COLS];
#pragma unroll
        for (int j = 0; j < IN_COLS; ++j) {
          __half2 v = __float2half2_rn(0.f);
          if (row_ok && ((col_ok >> j) & 1u)) v = __ldg(rowp + j * cp_count);
          xv[j] = __half22float2(v);
        }
        rowp += row_stride;
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          const int ky = ir - r * S;
          if (ky >= 0 && ky < K) {
#pragma unroll
            for (int tx = 0; tx < TW; ++tx)
#pragma unroll
              for (int kx = 0; kx < K; ++kx)
                acc[r][tx] = ffma2_rn(xv[tx * S + kx], wreg[ky * K + kx], acc[r][tx]);
          }
        }
      }
    }

    float2 bv = make_float2(0.f, 0.f);
    if (HAS_BIAS) bv = __ldg(reinterpret_cast<const float2*>(bias) + cp);
    __half2* out2 = reinterpret_cast<__half2*>(out) + static_cast<size_t>(n) * ho * wo * cp_count + cp;
    __half2* orow = out2 + (oy0 * wo + ox0) * cp_count;
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      if (interior || oy0 + r < ho) {
        float2 o[TW];
#pragma unroll
        for (int tx = 0; tx < TW; ++tx) o[tx] = fadd2_rn(acc[r][tx], bv);
#pragma unroll
        for (int tx = 0; tx + 1 < TW; tx += 2) apply_act4<ACT>(o[tx], o[tx + 1]);
        if (TW & 1) o[TW - 1] = apply_act2<ACT>(o[TW - 1]);
#pragma unroll
        for (int tx = 0; tx < TW; ++tx) {
          if (interior || ox0 + tx < wo) {
            if (HAS_SE) ssum = fadd2_rn(ssum, o[tx]);
            orow[tx * cp_count] = __floats2half2_rn(o[tx].x, o[tx].y);
          }
        }
      }
      orow += wo * cp_count;
    }
  }

  if (HAS_SE) {
    // Deterministic block reduction: every thread parks its sums, then one thread per channel
    // pair adds the contributions of the threads that own that pair, in index order.
    __shared__ float2 red[kDwThreads];
    red[threadIdx.x] = ssum;
    __syncthreads();
    // ... and adds the block's sum to the per-(image, channel) total as a 2^-20 fixed-point
    // integer: integer atomics are associative, so the squeeze is bit-reproducible run to run.
    unsigned long long* dst =
        reinterpret_cast<unsigned long long*>(se_sum) + static_cast<size_t>(n) * c;
    const int e0 = blockIdx.x * kDwThreads;
    const int touched = min(cp_count, kDwThreads);
    for (int q = threadIdx.x; q < touched; q += kDwThreads) {
      const int g = (e0 + q) % cp_count;   // the pairs this block actually owns
      int t = q;
      float2 s2 = make_float2(0.f, 0.f);
      for (; t < kDwThreads; t += cp_count) {
        s2.x += red[t].x;
        s2.y += red[t].y;
      }
      atomicAdd(dst + 2 * g, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(s2.x) * kSeFixedScale)));
      atomicAdd(dst + 2 * g + 1, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(s2.y) * kSeFixedScale)));
    }
  }
}

// SE, first FC: one WARP per (image, squeezed unit), so the n * se dot products of length c run
// on n * se / 8 CTAs with every load of a lane independent (pure latency otherwise).
//   mean[c]      = inv_hw * se_sum[n][c] / 2^20
//   hidden[n][j] = act(b1[j] + sum_c w1[j][c] * mean[c])
// Also clears `zero_buf` (the squeeze accumulator the NEXT block will use).
constexpr int kSeWarps = 8;
// SE, first FC: hidden[img][j] = act(b1[j] + sum_c w1[j][c] * mean[img][c]).  `split` warps share
// one output (each a contiguous slice of the channels; partial sums combined in warp order through
// shared memory, so the result does not depend on timing): 1 when the batch alone fills the chip
// (D0 at batch 32: 1536 outputs), up to 8 for small batches (D7x at batch 2: 320 outputs of 3840
// channels each would otherwise be 40 CTAs walking 30 dependent iterations).
__global__ void __launch_bounds__(kSeWarps * 32)
se_fc1_kernel(const long long* __restrict__ se_sum, float inv_hw, const float* __restrict__ w1,
              const float* __restrict__ b1, float* __restrict__ hidden,
              long long* __restrict__ zero_buf, long long zero_total, int n, int c, int se, int act,
              int split) {
  pdl_launch_dependents();
  pdl_wait_prior();
  __shared__ float part[kSeWarps];
  if (zero_buf != nullptr) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < zero_total;
         i += static_cast<long long>(gridDim.x) * blockDim.x)
      zero_buf[i] = 0;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per_cta = kSeWarps / split;                     // outputs per CTA
  const int unit = blockIdx.x * per_cta + warp / split;     // the warps of an output are adjacent
  const int piece = warp % split;
  const bool live = unit < n * se;
  float s = 0.f;
  int img = 0, j = 0;
  if (live) {
    img = unit / se;
    j = unit - img * se;
    const long long* sums = se_sum + static_cast<size_t>(img) * c;
    const float* wr = w1 + static_cast<size_t>(j) * c;
    const double scale = (1.0 / kSeFixedScale) * static_cast<double>(inv_hw);
    // channel slice of this warp (multiples of 32 so the lanes stay aligned)
    const int span = ((c + split * 32 - 1) / (split * 32)) * 32;
    const int c_begin = piece * span, c_end = min(c, c_begin + span);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int ch = c_begin + lane;
    for (; ch + 96 < c_end; ch += 128) {
      const long long q0 = sums[ch], q1 = sums[ch + 32], q2 = sums[ch + 64], q3 = sums[ch + 96];
      const float a0 = __ldg(wr + ch), a1 = __ldg(wr + ch + 32), a2 = __ldg(wr + ch + 64),
                  a3 = __ldg(wr + ch + 96);
      s0 = fmaf(a0, static_cast<float>(static_cast<double>(q0) * scale), s0);
      s1 = fmaf(a1, static_cast<float>(static_cast<double>(q1) * scale), s1);
      s2 = fmaf(a2, static_cast<float>(static_cast<double>(q2) * scale), s2);
      s3 = fmaf(a3, static_cast<float>(static_cast<double>(q3) * scale), s3);
    }
    for (; ch < c_end; ch += 32)
      s0 = fmaf(__ldg(wr + ch), static_cast<float>(static_cast<double>(sums[ch]) * scale), s0);
    s = (s0 + s1) + (s2 + s3);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  if (split == 1) {
    if (live && lane == 0) hidden[static_cast<size_t>(img) * se + j] = apply_act(s + b1[j], act);
    return;
  }
  if (lane == 0) part[warp] = s;
  __syncthreads();
  if (live && piece == 0 && lane == 0) {
    float t = 0.f;
    for (int k = 0; k < split; ++k) t += part[warp + k];     // fixed order
    hidden[static_cast<size_t>(img) * se + j] = apply_act(t + b1[j], act);
  }
}

// SE, second FC + excitation folded into the project weights, one CTA per (128-channel slice,
// image):
//   gate[n][c]            = sigmoid(b2[c] + sum_j w2t[j][c] * hidden[n][j])
//   wt_scaled[n][o][c]    = wt[o][c] * gate[n][c]
// blockIdx.z splits the output rows (kSeRows per CTA) so that small batches still fill the chip
// (D7x at batch 2: 640 x 3840 weights per image); every z recomputes the cheap gate slice.
constexpr int kSeSlice = 128;
constexpr int kSeRows = 64;
__global__ void __launch_bounds__(256)
se_fc2_scale_kernel(const float* __restrict__ hidden, const float* __restrict__ w2t,
                    const float* __restrict__ b2, float* __restrict__ gate,
                    const __half* __restrict__ wt, __half* __restrict__ wt_scaled, int c, int se,
                    int nout) {
  pdl_launch_dependents();
  pdl_wait_prior();
  extern __shared__ float sm[];
  float* hid = sm;              // [se]
  float* g = sm + ((se + 3) & ~3);   // [kSeSlice], 16-byte aligned
  const int n = blockIdx.y, c0 = blockIdx.x * kSeSlice;
  for (int j = threadIdx.x; j < se; j += blockDim.x) hid[j] = hidden[static_cast<size_t>(n) * se + j];
  __syncthreads();
  if (threadIdx.x < kSeSlice) {
    const int ch = c0 + threadIdx.x;
    float v = 0.f;
    if (ch < c) {
      float s0 = b2[ch], s1 = 0.f, s2 = 0.f, s3 = 0.f;
      int j = 0;
      for (; j + 3 < se; j += 4) {
        const float a0 = __ldg(w2t + static_cast<size_t>(j) * c + ch);
        const float a1 = __ldg(w2t + static_cast<size_t>(j + 1) * c + ch);
        const float a2 = __ldg(w2t + static_cast<size_t>(j + 2) * c + ch);
        const float a3 = __ldg(w2t + static_cast<size_t>(j + 3) * c + ch);
        s0 = fmaf(a0, hid[j], s0);
        s1 = fmaf(a1, hid[j + 1], s1);
        s2 = fmaf(a2, hid[j + 2], s2);
        s3 = fmaf(a3, hid[j + 3], s3);
      }
      for (; j < se; ++j) s0 = fmaf(__ldg(w2t + static_cast<size_t>(j) * c + ch), hid[j], s0);
      v = 1.0f / (1.0f + expf(-((s0 + s1) + (s2 + s3))));
      if (blockIdx.z == 0) gate[static_cast<size_t>(n) * c + ch] = v;
    }
    g[threadIdx.x] = v;
  }
  __syncthreads();
  if (wt == nullptr) return;
  // 16 x 16-byte pieces per 128-channel row slice; 256 threads cover 16 rows per pass
  const int piece = threadIdx.x & 15, row0 = threadIdx.x >> 4;
  const int ch = c0 + piece * 8;
  if (ch >= c) return;
  const float4 g0 = *reinterpret_cast<const float4*>(g + piece * 8);
  const float4 g1 = *reinterpret_cast<const float4*>(g + piece * 8 + 4);
  __half* dst = wt_scaled + static_cast<size_t>(n) * nout * c;
  const int o_end = min(nout, static_cast<int>(blockIdx.z + 1) * kSeRows);
#pragma unroll 4
  for (int o = static_cast<int>(blockIdx.z) * kSeRows + row0; o < o_end; o += 16) {
    float f[8];
    half8_to_float(__ldg(reinterpret_cast<const uint4*>(wt + static_cast<size_t>(o) * c + ch)), f);
    f[0] *= g0.x; f[1] *= g0.y; f[2] *= g0.z; f[3] *= g0.w;
    f[4] *= g1.x; f[5] *= g1.y; f[6] *= g1.z; f[7] *= g1.w;
    *reinterpret_cast<uint4*>(dst + static_cast<size_t>(o) * c + ch) = float_to_half8(f);
  }
}

template <int K, int S>
static int launch_dw(const __half* in, __half* out, const float* w, const float* bias,
                     long long* se_partial, int n, int h, int wd, int c, int act, cudaStream_t stream) {
  const int ho = ceil_div(h, S), wo = ceil_div(wd, S);
  const int pad_t = same_pad_before(h, K, S), pad_l = same_pad_before(wd, K, S);
  dim3 grid(ceil_div(ceil_div(wo, kDwTW) * (c >> 1), kDwThreads), ceil_div(ho, DwCfg<K, S>::ROWS), n);
#define EDET_DW_LAUNCH(ACT, HB, HS)                                                        \
  launch_err = launch_pdl(depthwise_kernel<K, S, ACT, HB, HS>, grid, dim3(kDwThreads), 0,  \
                          stream, in, out, w, bias, se_partial, h, wd, c, ho, wo, pad_t, pad_l)
  cudaError_t launch_err = cudaSuccess;
  const bool hb = bias != nullptr, hs = se_partial != nullptr;
  if (act == EDET_ACT_SWISH && hb && hs) EDET_DW_LAUNCH(EDET_ACT_SWISH, true, true);
  else if (act == EDET_ACT_SWISH && hb && !hs) EDET_DW_LAUNCH(EDET_ACT_SWISH, true, false);
  else if (act == EDET_ACT_RELU6 && hb && !hs) EDET_DW_LAUNCH(EDET_ACT_RELU6, true, false);
  else if (act == EDET_ACT_RELU6 && hb && hs) EDET_DW_LAUNCH(EDET_ACT_RELU6, true, true);
  else if (act == EDET_ACT_NONE && !hb && !hs) EDET_DW_LAUNCH(EDET_ACT_NONE, false, false);
  else if (act == EDET_ACT_NONE && hb && !hs) EDET_DW_LAUNCH(EDET_ACT_NONE, true, false);
  else {
    set_error("depthwise: unsupported combination act=%d bias=%d se=%d", act, (int)hb, (int)hs);
    return EDET_ERR_UNSUPPORTED;
  }
#undef EDET_DW_LAUNCH
  EDET_CHECK_CUDA(launch_err);
  return EDET_OK;
}

namespace dwt {   // depthwise_tile.cu
bool eligible(int h, int wd, int c, int k, int stride);
int run(const __half* in, __half* out, const float* w, const float* bias, long long* se_sum,
        int n, int h, int wd, int c, int k, int stride, int act, cudaStream_t stream);
}  // namespace dwt
}  // namespace edet

extern "C" int edet_depthwise_conv(const edet_half* in, edet_half* out, const float* w,
                                   const float* bias, int64_t* se_sum, int n, int h, int wd,
                                   int c, int k, int stride, int act, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(in && out && w, "depthwise: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && wd > 0 && c > 0 && c % 8 == 0, "depthwise: bad shape (c%%8)");
  EDET_CHECK_ARG((k == 3 || k == 5) && (stride == 1 || stride == 2),
                 "depthwise: k must be 3 or 5 and stride 1 or 2 (got %d, %d)", k, stride);
  const __half* hi = reinterpret_cast<const __half*>(in);
  const float* hw = w;
  __half* ho = reinterpret_cast<__half*>(out);
  long long* sp = reinterpret_cast<long long*>(se_sum);
  cudaStream_t s = as_stream(stream);
  // large maps: TMA-staged shared-memory tiles (depthwise_tile.cu); small maps: register tiles
  if (option_dw_impl() != 1 && dwt::eligible(h, wd, c, k, stride))
    return dwt::run(hi, ho, hw, bias, sp, n, h, wd, c, k, stride, act, s);
  if (k == 3 && stride == 1) return launch_dw<3, 1>(hi, ho, hw, bias, sp, n, h, wd, c, act, s);
  if (k == 3 && stride == 2) return launch_dw<3, 2>(hi, ho, hw, bias, sp, n, h, wd, c, act, s);
  if (k == 5 && stride == 1) return launch_dw<5, 1>(hi, ho, hw, bias, sp, n, h, wd, c, act, s);
  return launch_dw<5, 2>(hi, ho, hw, bias, sp, n, h, wd, c, act, s);
}

extern "C" int edet_se_fc(const int64_t* se_sum, float inv_hw, const float* w1, const float* b1,
                          const float* w2, const float* b2, float* hidden, float* gate,
                          const edet_half* wt, edet_half* wt_scaled, int64_t* zero_buf,
                          int zero_count, int n, int c, int se, int nout, int act,
                          edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(se_sum && w1 && b1 && w2 && b2 && hidden && gate, "se_fc: null pointer");
  EDET_CHECK_ARG(n > 0 && c > 0 && c % 8 == 0 && se > 0, "se_fc: bad shape");
  EDET_CHECK_ARG(!wt || (wt_scaled && nout > 0), "se_fc: wt given without wt_scaled/nout");
  const size_t smem = static_cast<size_t>(((se + 3) & ~3) + kSeSlice) * sizeof(float);
  EDET_CHECK_ARG(smem <= 48 * 1024, "se_fc: se too large");
  // warps per output: enough CTAs to cover the chip a few times, slices of >= 128 channels
  int split = 1;
  while (split < kSeWarps && n * se * split < 2048 && c / (2 * split) >= 128) split *= 2;
  EDET_CHECK_CUDA(launch_pdl(se_fc1_kernel, dim3(ceil_div(n * se, kSeWarps / split)),
                             dim3(kSeWarps * 32), 0, as_stream(stream),
                             reinterpret_cast<const long long*>(se_sum), inv_hw, w1, b1, hidden,
                             reinterpret_cast<long long*>(zero_buf),
                             static_cast<long long>(n) * zero_count, n, c, se, act, split));
  EDET_CHECK_CUDA(launch_pdl(se_fc2_scale_kernel,
                             dim3(ceil_div(c, kSeSlice), n, wt ? ceil_div(nout, kSeRows) : 1), dim3(256), smem,
                             as_stream(stream), static_cast<const float*>(hidden), w2, b2, gate,
                             reinterpret_cast<const __half*>(wt),
                             reinterpret_cast<__half*>(wt_scaled), c, se, nout));
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}
