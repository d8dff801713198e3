// Depthwise k x k convolution ('SAME', NHWC fp16) + bias + activation (+ SE squeeze), tiled
// through shared memory by TMA.
//
// The north_star design for this memory-bound op: the input tile (with its halo) of one 64-channel
// slice is fetched by ONE bulk tensor copy (cp.async.bulk.tensor, 4-D map over [N][H][W][C]),
// out-of-image pixels arrive as zeros -- exactly TF's 'SAME' zero padding -- so the kernel has no
// border predicates and a single code path; a ring of NSTAGE tiles keeps the next work units in
// flight while the current one is computed.  Compute: one lane = one channel pair (a warp reads
// the 128 contiguous bytes of a pixel, conflict-free), one thread = TR x TC outputs of that pair
// from registers (fp32 weights in registers, FFMA on channel pairs), one warp = one TR x TC patch, the 8
// warps of a CTA tile a (TR*WY) x (TC*WX) output tile.  HBM sees each input byte once per tile
// (plus the halo, served by L2) and each output byte once.
//
// Persistent CTAs (two per SM) take the work units (image, tile, 64-channel slice) from a global
// counter; the channel slice varies fastest so that concurrently running CTAs touch the same DRAM
// pages.
//
// Algorithmic HBM bytes per launch (SURVEY.md 8d): 2*n*c*(h*w + ho*wo) + 2*k*k*c (+ 8*n*c of
// int64 atomics for the SE squeeze).  Used for c >= 64 when the fixed output tile covers the map
// with <= 30 % waste (see eligible()); the register-tiled kernel of depthwise.cu keeps the rest.
#include "tc_common.cuh"

namespace edet {
namespace dwt {

using namespace pwtc;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kCB = 64;                 // channels per work unit (one 128-byte pixel row in smem)
constexpr int kPixBytes = kCB * 2;

template <int K, int S>
struct Cfg {
  // thread tile
  static constexpr int TR = (S == 2) ? 4 : (K == 3 ? 8 : 4);
  static constexpr int TC = (S == 2) ? 2 : 4;
  static constexpr int WX = 4, WY = 2;                       // warps along x / y
  static constexpr int TOH = TR * WY, TOW = TC * WX;         // output tile of a CTA
  static constexpr int IN_ROWS = (TR - 1) * S + K;           // input rows / cols a thread touches
  static constexpr int IN_COLS = (TC - 1) * S + K;
  static constexpr int TIH = (TOH - 1) * S + K;              // input tile (with halo)
  static constexpr int TIW = (TOW - 1) * S + K;
  static constexpr int TILE_BYTES = ((TIH * TIW * kPixBytes + 127) / 128) * 128;
  static constexpr int NSTAGE = TILE_BYTES <= 32 * 1024 ? 3 : 2;
};

struct Params {
  int n, h, w, c, ho, wo, pad_t, pad_l;
  int chunks, tiles_y, tiles_x, total_units;
  const float* wgt;       // fp32 taps [k*k][c]
  const float* bias;      // [c] or null
  __half* out;            // [n, ho, wo, c]
  long long* se_sum;      // [n, c] or null
  unsigned* sched;        // dynamic work-unit scheduler slot (tc_common.cuh)
};

struct Unit {
  int n, ty, tx, chunk;
};
__device__ __forceinline__ Unit decode(int u, const Params& p) {
  Unit r;
  r.chunk = u % p.chunks;
  u /= p.chunks;
  r.tx = u % p.tiles_x;
  u /= p.tiles_x;
  r.ty = u % p.tiles_y;
  r.n = u / p.tiles_y;
  return r;
}

__device__ __forceinline__ uint32_t lds_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

template <int K, int S, int ACT, bool HAS_BIAS, bool HAS_SE>
__global__ void __launch_bounds__(kThreads, 2)
dw_tile_kernel(const __grid_constant__ CUtensorMap map_x, const Params p) {
  using C = Cfg<K, S>;
  constexpr int TR = C::TR, TC = C::TC, IN_ROWS = C::IN_ROWS, IN_COLS = C::IN_COLS;
  constexpr int NSTAGE = C::NSTAGE;
  pdl_launch_dependents();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE * C::TILE_BYTES);      // [NSTAGE]
  // SE squeeze partials [2][warps][kCB]: every warp parks the fixed-point sums of its lanes'
  // channel pairs with plain stores; after the unit's barrier 64 threads add the eight warps up and
  // issue the global atomics (64-bit shared-memory atomics are CAS loops, 8-way contended here)
  unsigned long long* se_s = reinterpret_cast<unsigned long long*>(
      (reinterpret_cast<uintptr_t>(bars + NSTAGE) + 15) & ~static_cast<uintptr_t>(15));
  // [NSTAGE] x {unit index, image, tile row, tile column}: decoded once by thread 0 (three integer
  // divisions), read by everybody else with one 16-byte shared-memory load
  volatile int4* unit_s = reinterpret_cast<volatile int4*>(
      (reinterpret_cast<uintptr_t>(se_s + 2 * kWarps * kCB) + 15) & ~static_cast<uintptr_t>(15));
  int* unit_chunk_s = reinterpret_cast<int*>(const_cast<int4*>(unit_s) + NSTAGE);      // [NSTAGE]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) mbar_init(smem_u32(&bars[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_x)) : "memory");
  }
  pdl_wait_prior();      // everything above overlapped the previous kernel's tail

  auto park = [&](int u, int stage) -> Unit {   // thread 0 only: publish the unit of a stage
    Unit un;
    un.n = un.ty = un.tx = un.chunk = 0;
    if (u < p.total_units) un = decode(u, p);
    unit_chunk_s[stage] = un.chunk;
    const_cast<int4*>(unit_s)[stage] = make_int4(u, un.n, un.ty, un.tx);
    return un;
  };
  auto issue = [&](const Unit& un, int stage) {       // thread 0 only
    const uint32_t bar = smem_u32(&bars[stage]);
    mbar_expect_tx(bar, static_cast<uint32_t>(C::TIH * C::TIW * kPixBytes));
    tma_load_4d(smem_u32(smem + stage * C::TILE_BYTES), &map_x, bar, un.chunk * kCB,
                un.tx * C::TOW * S - p.pad_l, un.ty * C::TOH * S - p.pad_t, un.n);
  };
  // Work units come from a global counter (CTA i owns unit i, every further unit is fetched):
  // when another stream holds some SMs (the NMS of the previous batch) late CTAs simply find less
  // work instead of owning a full static share.  Thread 0 fetches NSTAGE units ahead and parks
  // each stage's unit index in unit_s; after the first out-of-range fetch it stops fetching.
  bool exhausted = false;    // thread 0 only
  auto next_unit = [&]() -> int {
    if (exhausted) return p.total_units;
    const int u = sched_next_tile(p.sched, p.total_units);
    if (u >= p.total_units) exhausted = true;
    return u;
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      const int u = s == 0 ? static_cast<int>(blockIdx.x) : next_unit();
      const Unit un = park(u, s);
      if (u < p.total_units) issue(un, s);
    }
  }
  __syncthreads();

  const int wx = warp % C::WX, wy = warp / C::WX;
  const int oy_t = wy * TR, ox_t = wx * TC;                      // thread's outputs inside the tile
  const uint32_t thread_off =
      static_cast<uint32_t>(((oy_t * S) * C::TIW + ox_t * S) * kPixBytes + lane * 4);
  const int cp_total = p.c >> 1;

  float2 wreg[K * K];
  float2 bv = make_float2(0.f, 0.f);
  int cur_chunk = -1;

  for (int it = 0;; ++it) {
    const int stage = it % NSTAGE;
    const int4 ui = const_cast<const int4*>(unit_s)[stage];
    if (ui.x >= p.total_units) break;       // same value for every thread of the CTA
    const uint32_t phase = static_cast<uint32_t>(it / NSTAGE) & 1u;
    Unit un;
    un.n = ui.y; un.ty = ui.z; un.tx = ui.w; un.chunk = unit_chunk_s[stage];
    const int cp = un.chunk * (kCB / 2) + lane;                  // channel pair of this lane
    const bool lane_ok = cp < cp_total;
    if (un.chunk != cur_chunk) {                                 // (re)load this slice's weights
      cur_chunk = un.chunk;
      const float2* w2 = reinterpret_cast<const float2*>(p.wgt);
#pragma unroll
      for (int t = 0; t < K * K; ++t)
        wreg[t] = lane_ok ? __ldg(w2 + t * cp_total + cp) : make_float2(0.f, 0.f);
      if (HAS_BIAS) bv = lane_ok ? __ldg(reinterpret_cast<const float2*>(p.bias) + cp) : make_float2(0.f, 0.f);
    }
    mbar_wait(smem_u32(&bars[stage]), phase);                    // the tile has landed

    float2 acc[TR][TC];
#pragma unroll
    for (int r = 0; r < TR; ++r)
#pragma unroll
      for (int tx = 0; tx < TC; ++tx) acc[r][tx] = make_float2(0.f, 0.f);
    const uint32_t base = smem_u32(smem + stage * C::TILE_BYTES) + thread_off;
#pragma unroll
    for (int ir = 0; ir < IN_ROWS; ++ir) {
      float2 xv[IN_COLS];
#pragma unroll
      for (int j = 0; j < IN_COLS; ++j) {
        const uint32_t raw = lds_b32(base + static_cast<uint32_t>((ir * C::TIW + j) * kPixBytes));
        xv[j] = __half22float2(*reinterpret_cast<const __half2*>(&raw));
      }
#pragma unroll
      for (int r = 0; r < TR; ++r) {
        const int ky = ir - r * S;
        if (ky >= 0 && ky < K) {
#pragma unroll
          for (int tx = 0; tx < TC; ++tx)
#pragma unroll
            for (int kx = 0; kx < K; ++kx)
              acc[r][tx] = ffma2_rn(xv[tx * S + kx], wreg[ky * K + kx], acc[r][tx]);
        }
      }
    }

    // epilogue: bias, activation, SE partial sums, coalesced 128-byte stores per (pixel, warp)
    const int oy0 = un.ty * C::TOH + oy_t, ox0 = un.tx * C::TOW + ox_t;
    float2 ssum = make_float2(0.f, 0.f);
    if (lane_ok) {
      __half2* orow = reinterpret_cast<__half2*>(p.out) +
                      ((static_cast<size_t>(un.n) * p.ho + oy0) * p.wo + ox0) * cp_total + cp;
#pragma unroll
      for (int r = 0; r < TR; ++r) {
        if (oy0 + r < p.ho) {
          float2 o[TC];
#pragma unroll
          for (int tx = 0; tx < TC; ++tx) o[tx] = fadd2_rn(acc[r][tx], bv);
#pragma unroll
          for (int tx = 0; tx + 1 < TC; tx += 2) apply_act4<ACT>(o[tx], o[tx + 1]);
          if (TC & 1) o[TC - 1] = apply_act2<ACT>(o[TC - 1]);
#pragma unroll
          for (int tx = 0; tx < TC; ++tx) {
            if (ox0 + tx < p.wo) {
              if (HAS_SE) ssum = fadd2_rn(ssum, o[tx]);
              orow[static_cast<size_t>(tx) * cp_total] = __floats2half2_rn(o[tx].x, o[tx].y);
            }
          }
        }
        orow += static_cast<size_t>(p.wo) * cp_total;
      }
    }
    unsigned long long* se_unit = se_s + (it & 1) * (kWarps * kCB);
    if (HAS_SE) {
      // 2^-20 fixed point, integer sums: order independent => bit-reproducible squeeze
      const unsigned long long sx = lane_ok ? static_cast<unsigned long long>(__float2ll_rn(ssum.x * 1048576.f)) : 0ull;
      const unsigned long long sy = lane_ok ? static_cast<unsigned long long>(__float2ll_rn(ssum.y * 1048576.f)) : 0ull;
      *reinterpret_cast<ulonglong2*>(se_unit + warp * kCB + 2 * lane) = make_ulonglong2(sx, sy);
    }
    __syncthreads();       // every thread has finished reading this stage (and adding to se_unit)
    if (threadIdx.x == 0) {
      const int u_next = next_unit();
      const Unit un_next = park(u_next, stage);   // read NSTAGE iterations (>= 1 barrier) later
      if (u_next < p.total_units) issue(un_next, stage);
    }
    if (HAS_SE && threadIdx.x < kCB) {
      // flush this unit's sums; the OTHER buffer takes the next unit's partials meanwhile
      const int ch = un.chunk * kCB + threadIdx.x;
      unsigned long long v = 0ull;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) v += se_unit[w * kCB + threadIdx.x];
      if (ch < p.c && v != 0ull)
        atomicAdd(reinterpret_cast<unsigned long long*>(p.se_sum) + static_cast<size_t>(un.n) * p.c + ch, v);
    }
  }
}

template <int K, int S>
static int launch_kernel(const CUtensorMap& mx, const Params& p, int grid, int act, cudaStream_t stream) {
  using C = Cfg<K, S>;
  const int smem_bytes = 1024 + C::NSTAGE * C::TILE_BYTES + C::NSTAGE * 8 + 2 * kWarps * kCB * 8 + 16 +
                         C::NSTAGE * 20 + 16;
  const bool hb = p.bias != nullptr, hs = p.se_sum != nullptr;
#define EDET_DWT(ACT, HB, HS)                                                                  \
  do {                                                                                         \
    auto kern = dw_tile_kernel<K, S, ACT, HB, HS>;                                             \
    static int configured[kMaxDevices];                                                        \
    if (int rc = ensure_dynamic_smem(kern, smem_bytes, configured)) return rc;                 \
    EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), smem_bytes, stream, mx, p));  \
    return EDET_OK;                                                                            \
  } while (0)
  if (act == EDET_ACT_SWISH && hb && hs) EDET_DWT(EDET_ACT_SWISH, true, true);
  if (act == EDET_ACT_SWISH && hb && !hs) EDET_DWT(EDET_ACT_SWISH, true, false);
  if (act == EDET_ACT_RELU6 && hb && !hs) EDET_DWT(EDET_ACT_RELU6, true, false);
  if (act == EDET_ACT_RELU6 && hb && hs) EDET_DWT(EDET_ACT_RELU6, true, true);
  if (act == EDET_ACT_NONE && !hb && !hs) EDET_DWT(EDET_ACT_NONE, false, false);
  if (act == EDET_ACT_NONE && hb && !hs) EDET_DWT(EDET_ACT_NONE, true, false);
#undef EDET_DWT
  set_error("depthwise(tile): unsupported combination act=%d bias=%d se=%d", act, (int)hb, (int)hs);
  return EDET_ERR_UNSUPPORTED;
}

// True when the tiled kernel takes this shape (otherwise the register-tiled kernel runs): at least
// one full 64-channel slice, and the fixed output tile of this (k, stride) must cover the map
// without wasting more than ~30 % of its threads on out-of-map outputs (measured: 24 x 24 maps
// under 16 x 16 tiles lose to the register kernel, 40 x 40 maps under 8 x 16 tiles win).
template <int K, int S>
static bool fits(int ho, int wo) {
  using C = Cfg<K, S>;
  const long long covered = static_cast<long long>(ceil_div(ho, C::TOH)) * C::TOH *
                            static_cast<long long>(ceil_div(wo, C::TOW)) * C::TOW;
  return static_cast<long long>(ho) * wo * 10 >= covered * 7;
}
bool eligible(int h, int wd, int c, int k, int stride) {
  const int ho = ceil_div(h, stride), wo = ceil_div(wd, stride);
  if (c < kCB) return false;
  if (k == 3 && stride == 1) return fits<3, 1>(ho, wo);
  if (k == 3 && stride == 2) return fits<3, 2>(ho, wo);
  if (k == 5 && stride == 1) return fits<5, 1>(ho, wo);
  return fits<5, 2>(ho, wo);
}

template <int K, int S>
static int run_ks(const __half* in, __half* out, const float* w, const float* bias,
                  long long* se_sum, int n, int h, int wd, int c, int act, cudaStream_t stream) {
  using C = Cfg<K, S>;
  Params p;
  p.n = n; p.h = h; p.w = wd; p.c = c;
  p.ho = ceil_div(h, S); p.wo = ceil_div(wd, S);
  p.pad_t = same_pad_before(h, K, S); p.pad_l = same_pad_before(wd, K, S);
  p.chunks = ceil_div(c, kCB);
  p.tiles_y = ceil_div(p.ho, C::TOH);
  p.tiles_x = ceil_div(p.wo, C::TOW);
  const long long total = static_cast<long long>(n) * p.tiles_y * p.tiles_x * p.chunks;
  EDET_CHECK_ARG(total < 0x7fffffffLL, "depthwise(tile): too many work units");
  p.total_units = static_cast<int>(total);
  p.wgt = w; p.bias = bias; p.out = out; p.se_sum = se_sum;
  p.sched = next_sched_slot();
  if (!p.sched) return EDET_ERR_CUDA;
  CUtensorMap mx;
  if (int rc = make_map4(&mx, in, c, wd, h, n, kCB, C::TIW, C::TIH, /*swizzle=*/false)) return rc;
  const int sms = device_sm_count();
  if (!sms) return EDET_ERR_CUDA;
  int grid = 2 * sms - option_persist_slack();
  if (grid < sms) grid = sms;
  if (p.total_units < grid) grid = p.total_units;
  return launch_kernel<K, S>(mx, p, grid, act, stream);
}

int run(const __half* in, __half* out, const float* w, const float* bias, long long* se_sum,
        int n, int h, int wd, int c, int k, int stride, int act, cudaStream_t stream) {
  if (k == 3 && stride == 1) return run_ks<3, 1>(in, out, w, bias, se_sum, n, h, wd, c, act, stream);
  if (k == 3 && stride == 2) return run_ks<3, 2>(in, out, w, bias, se_sum, n, h, wd, c, act, stream);
  if (k == 5 && stride == 1) return run_ks<5, 1>(in, out, w, bias, se_sum, n, h, wd, c, act, stream);
  return run_ks<5, 2>(in, out, w, bias, se_sum, n, h, wd, c, act, stream);
}

}  // namespace dwt
}  // namespace edet
