// Fused front half of an MBConv block:  expand 1x1 (+BN, +act)  ->  depthwise kxk 'SAME' (+BN,
// +act) (+ SE squeeze), WITHOUT the expanded tensor ever reaching HBM.
//
// Replaces, for the early high-resolution blocks, the pair
//   Conv2D 1x1 + BN + swish   backbone/efficientnet_model.py:303-317, 388
//   DepthwiseConv2D + BN + swish (+ reduce_mean for SE)  :320-333, 391, :192
// whose 6x-expanded intermediate is the largest byte mover of the network (SURVEY.md 8d:
// "plan B").  Algorithmic HBM bytes per launch: 2*N*(H*W*Cin*halo + Ho*Wo*Cmid) + weights,
// instead of 2*N*(H*W*Cin + 2*H*W*Cmid + Ho*Wo*Cmid) for the two separate kernels.
//
// One CTA works on a 16x16 INPUT patch (256 pixels = four 64-row wgmma blocks, two per warpgroup)
// and one chunk of the expanded channels:
//   1. TMA (4-D map over the NHWC input, out-of-image pixels zero-filled) -> smem A tile
//      [256 px][Cin], TMA -> smem W tile [ch][Cin]   (32B / 64B / 128B swizzle by Cin)
//   2. wgmma: E[256 px][ch] = A * W^T, fp32 accumulators in registers
//   3. every thread: its accumulator fragment -> +bias -> act -> fp16 -> smem E tile; pixels
//      outside the image become 0 (TF pads the EXPANDED tensor with zeros, not the input)
//   4. all 8 warps: depthwise kxk stride s over the smem E tile (one channel pair x one output
//      row per work item, FFMA on channel pairs), + bias + act -> global, SE sums -> int64 atomics
// The next tile's TMA loads are issued as soon as the MMAs of the current tile have retired, so
// they overlap steps 3-4.
#include "tc_common.cuh"

namespace edet {
namespace mbf {

using namespace pwtc;

constexpr int kThreads = 256;
constexpr int kPatch = 16;                 // input patch is kPatch x kPatch pixels
constexpr int kPatchPx = kPatch * kPatch;  // 256 rows of the expand GEMM
constexpr int kMaxCh = 64;                 // expanded channels per tile: 2 x 32 accumulators per thread
constexpr int kNT = kMaxCh / 16;
// bytes per pixel row of the smem E tile: (pitch / 16) odd -> conflict-free 128-bit row writes;
// a compile-time constant so that every depthwise tap is an immediate offset
constexpr int kEPitch = kMaxCh * 2 + 16;

__device__ __forceinline__ uint32_t lds_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_v4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ float2 h2_bits_to_f2(uint32_t v) {
  return __half22float2(*reinterpret_cast<const __half2*>(&v));
}

struct Params {
  int n, h, w, cin, cmid, ho, wo, pad_t, pad_l;
  int block_k, num_k_blocks, a_bytes, b_bytes, desc_sbo, desc_layout;
  int ch, num_chunks;          // expanded channels per CTA tile, number of chunks
  int oth, otw;                // output tile (rows, cols) produced from one input patch
  int tiles_y, tiles_x, total_tiles;
  const float* bias_e;         // [cmid]
  const float* wd;             // fp32 depthwise taps [k*k][cmid]
  const float* bias_d;         // [cmid]
  __half* out;                 // [n, ho, wo, cmid]
  long long* se_sum;           // [n, cmid] or null
  unsigned* sched;             // dynamic tile scheduler slot (tc_common.cuh)
};

struct Tile {
  int n, ty, tx, chunk;
};
__device__ __forceinline__ Tile decode(int t, const Params& p) {
  Tile r;
  r.chunk = t % p.num_chunks;
  t /= p.num_chunks;
  r.tx = t % p.tiles_x;
  t /= p.tiles_x;
  r.ty = t % p.tiles_y;
  r.n = t / p.tiles_y;
  return r;
}

template <int K, int S, int ACT, bool HAS_SE>
__global__ void __launch_bounds__(kThreads, 2)
mbconv_front_kernel(const __grid_constant__ CUtensorMap map_x,
                    const __grid_constant__ CUtensorMap map_w, const Params p) {
  constexpr int OTW = (kPatch - K) / S + 1;   // output columns (and rows) per patch
  constexpr int NIX = (OTW - 1) * S + K;      // input columns a full output row touches
  pdl_launch_dependents();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;                       // [256 px][block_k] swizzled
  uint8_t* smem_b = smem_a + p.a_bytes;         // [ch][block_k] swizzled
  uint8_t* smem_e = smem_b + p.b_bytes;         // [256 px][e_pitch] fp16
  unsigned long long* se_s =
      reinterpret_cast<unsigned long long*>(smem_e + kPatchPx * kEPitch);  // [ch]
  uint64_t* bars = reinterpret_cast<uint64_t*>(se_s + p.ch);
  const uint32_t full_bar = smem_u32(bars);       // TMA -> MMA
  volatile int* next_tile_s = reinterpret_cast<volatile int*>(bars + 1);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;                       // warpgroup: patch pixels 128 wg .. 128 wg + 127
  if (threadIdx.x == 0) {
    mbar_init(full_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_x)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
  }
  __syncthreads();
  pdl_wait_prior();

  const uint32_t tx_bytes = static_cast<uint32_t>(kPatchPx * p.block_k * 2 + p.ch * p.block_k * 2);
  const int pitch = p.block_k * 2;                // bytes per smem operand row
  const int nt = p.ch >> 4;
  uint32_t full_phase = 0;

  auto issue_loads = [&](const Tile& tl, int kb) {
    mbar_expect_tx(full_bar, tx_bytes);
    tma_load_4d(smem_u32(smem_a), &map_x, full_bar, kb * p.block_k, tl.tx * OTW * S - p.pad_l,
                tl.ty * OTW * S - p.pad_t, tl.n);
    tma_load_3d(smem_u32(smem_b), &map_w, full_bar, kb * p.block_k, tl.chunk * p.ch, 0);
  };

  bool prefetched = false;   // thread 0 only
  int t = blockIdx.x;
  // next_tile_s is double buffered: the slot written in iteration i is rewritten in i + 2, after
  // every thread has passed the closing barrier of i + 1 (hence its read of iteration i)
  for (int it = 0; t < p.total_tiles; ++it) {
    const Tile tl = decode(t, p);
    const int cbase = tl.chunk * p.ch;
    const int cv = min(p.ch, p.cmid - cbase);   // valid channels of this chunk (multiple of 8)
    // ---- 1+2. expand GEMM (thread 0 drives TMA; each warpgroup multiplies its 128 pixels) ----
    float acc[2][kNT][8] = {};
    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
      if (threadIdx.x == 0 && !(kb == 0 && prefetched)) issue_loads(tl, kb);
      mbar_wait(full_bar, full_phase);
      full_phase ^= 1;
      const int k_rem = p.cin - kb * p.block_k;
      const int ksteps = k_rem >= p.block_k ? p.block_k / MMA_K : (k_rem + MMA_K - 1) / MMA_K;
      const uint64_t db = make_smem_desc(smem_u32(smem_b), p.desc_sbo, p.desc_layout);
      wg_fence();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint64_t da =
            make_smem_desc(smem_u32(smem_a + (wg * 128 + h * 64) * pitch), p.desc_sbo, p.desc_layout);
        wg_mma_kblock<kNT>(acc[h], da, db, pitch, nt, ksteps, kb == 0);
      }
      wg_commit();
      wg_wait<0>();
      __syncthreads();   // every MMA of this k-block has retired: the operand buffers are free
    }
    wg_fence_acc<kNT>(acc[0]);
    wg_fence_acc<kNT>(acc[1]);
    // the operand buffers are free: fetch the next tile's first k-block under phases 3-4
    if (threadIdx.x == 0) {
      const int tn = sched_next_tile(p.sched, p.total_tiles);
      next_tile_s[it & 1] = tn;
      prefetched = tn < p.total_tiles;
      if (prefetched) issue_loads(decode(tn, p), 0);
    }
    // ---- 3. accumulator fragments -> bias, act, mask -> smem E tile ----
    {
      const int cq = 2 * (lane & 3);
      const float* be = p.bias_e + cbase;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int m = wg * 128 + h * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * r;  // patch pixel
          const int py = m / kPatch, px = m % kPatch;
          const int iy = tl.ty * OTW * S - p.pad_t + py, ix = tl.tx * OTW * S - p.pad_l + px;
          const bool inside = iy >= 0 && iy < p.h && ix >= 0 && ix < p.w;
          const uint32_t erow = smem_u32(smem_e) + m * kEPitch;
#pragma unroll
          for (int j = 0; j < kNT; ++j) {
            const int col = 16 * j + cq;
            if (16 * j >= cv) continue;
            const bool hi_ok = 16 * j + 8 < cv;     // cv is a multiple of 8
            uint32_t lo_bits = 0u, hi_bits = 0u;    // TF zero-pads the EXPANDED map
            if (inside) {
              const float2 b_lo = __ldg(reinterpret_cast<const float2*>(be + col));
              const float2 b_hi = hi_ok ? __ldg(reinterpret_cast<const float2*>(be + col + 8))
                                        : make_float2(0.f, 0.f);
              float2 lo = fadd2_rn(make_float2(acc[h][j][2 * r], acc[h][j][2 * r + 1]), b_lo);
              float2 hi = fadd2_rn(make_float2(acc[h][j][4 + 2 * r], acc[h][j][4 + 2 * r + 1]), b_hi);
              apply_act4<ACT>(lo, hi);
              const __half2 l2 = __floats2half2_rn(lo.x, lo.y), h2 = __floats2half2_rn(hi.x, hi.y);
              lo_bits = *reinterpret_cast<const uint32_t*>(&l2);
              hi_bits = *reinterpret_cast<const uint32_t*>(&h2);
            }
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(erow + col * 2), "r"(lo_bits) : "memory");
            if (hi_ok)
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(erow + (col + 8) * 2), "r"(hi_bits) : "memory");
          }
        }
      }
      if (HAS_SE)
        for (int i = threadIdx.x; i < p.ch; i += kThreads) se_s[i] = 0ull;
    }
    __syncthreads();
    // ---- 4. depthwise over the smem E tile ------------------------------------------------------
    {
      const int cpn = cv >> 1;
      const int oy0 = tl.ty * OTW, ox0 = tl.tx * OTW;
      const int rows = min(OTW, p.ho - oy0), cols = min(OTW, p.wo - ox0);
      const int cm2 = p.cmid >> 1;
      const uint32_t e_u32 = smem_u32(smem_e);
      if constexpr (K == 3 && S == 2) {
        // One work item = (pair of output columns, channel pair): the thread produces the whole
        // 7-row column pair from registers (weights loaded once, every input pixel read once per
        // thread: 15 x 5 ld.shared for 14 outputs), instead of one output row per item with the
        // weights re-read per item -- the depthwise phase was 2/3 of this kernel's instructions.
        constexpr int CG = 2;
        constexpr int NCG = (OTW + CG - 1) / CG;
        constexpr int IN_R = (OTW - 1) * S + K, IN_C = (CG - 1) * S + K;
        for (int item = threadIdx.x; item < NCG * cpn; item += kThreads) {
          const int xg = item / cpn, cp = item - xg * cpn;
          const float2* wd2 = reinterpret_cast<const float2*>(p.wd) + ((cbase >> 1) + cp);
          float2 wk[K * K];
#pragma unroll
          for (int i = 0; i < K * K; ++i) wk[i] = __ldg(wd2 + i * cm2);
          uint32_t coff[IN_C];     // the last column group reads a clamped (discarded) column
#pragma unroll
          for (int j = 0; j < IN_C; ++j)
            coff[j] = e_u32 + static_cast<uint32_t>(min(xg * CG * S + j, kPatch - 1) * kEPitch + cp * 4);
          float2 acc[OTW][CG];
#pragma unroll
          for (int r = 0; r < OTW; ++r)
#pragma unroll
            for (int tx = 0; tx < CG; ++tx) acc[r][tx] = make_float2(0.f, 0.f);
#pragma unroll
          for (int ir = 0; ir < IN_R; ++ir) {
            float2 xv[IN_C];
#pragma unroll
            for (int j = 0; j < IN_C; ++j) xv[j] = h2_bits_to_f2(lds_b32(coff[j] + ir * kPatch * kEPitch));
#pragma unroll
            for (int r = 0; r < OTW; ++r) {
              const int ky = ir - r * S;
              if (ky >= 0 && ky < K) {
#pragma unroll
                for (int tx = 0; tx < CG; ++tx)
#pragma unroll
                  for (int kx = 0; kx < K; ++kx)
                    acc[r][tx] = ffma2_rn(xv[tx * S + kx], wk[ky * K + kx], acc[r][tx]);
              }
            }
          }
          const float2 bd = __ldg(reinterpret_cast<const float2*>(p.bias_d + cbase) + cp);
          __half2* ocol = reinterpret_cast<__half2*>(p.out) +
                          ((static_cast<size_t>(tl.n) * p.ho + oy0) * p.wo + ox0 + xg * CG) * cm2 +
                          (cbase >> 1) + cp;
          float2 ssum = make_float2(0.f, 0.f);
#pragma unroll
          for (int r = 0; r < OTW; ++r) {
            float2 o0 = fadd2_rn(acc[r][0], bd), o1 = fadd2_rn(acc[r][1], bd);
            apply_act4<ACT>(o0, o1);
            if (r < rows) {
              if (xg * CG < cols) {
                if (HAS_SE) ssum = fadd2_rn(ssum, o0);
                ocol[static_cast<size_t>(r) * p.wo * cm2] = __floats2half2_rn(o0.x, o0.y);
              }
              if (xg * CG + 1 < cols) {
                if (HAS_SE) ssum = fadd2_rn(ssum, o1);
                ocol[static_cast<size_t>(r) * p.wo * cm2 + cm2] = __floats2half2_rn(o1.x, o1.y);
              }
            }
          }
          if (HAS_SE) {
            atomicAdd(&se_s[2 * cp], static_cast<unsigned long long>(__float2ll_rn(ssum.x * 1048576.f)));
            atomicAdd(&se_s[2 * cp + 1], static_cast<unsigned long long>(__float2ll_rn(ssum.y * 1048576.f)));
          }
        }
      } else {
      // one (output row, channel pair) per work item
      for (int item = threadIdx.x; item < rows * cpn; item += kThreads) {
        const int oyl = item / cpn, cp = item - oyl * cpn;
        const float2* wd2 = reinterpret_cast<const float2*>(p.wd) + ((cbase >> 1) + cp);
        const uint32_t ebase = e_u32 + (oyl * S * kPatch) * kEPitch + cp * 4;
        float2 acc[OTW];
#pragma unroll
        for (int i = 0; i < OTW; ++i) acc[i] = make_float2(0.f, 0.f);
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          float2 wk[K];
#pragma unroll
          for (int kx = 0; kx < K; ++kx) wk[kx] = __ldg(wd2 + (ky * K + kx) * cm2);
#pragma unroll
          for (int ixl = 0; ixl < NIX; ++ixl) {
            const float2 v = h2_bits_to_f2(lds_b32(ebase + (ky * kPatch + ixl) * kEPitch));
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
              if ((ixl - kx) >= 0 && (ixl - kx) % S == 0 && (ixl - kx) / S < OTW)
                acc[(ixl - kx) / S] = ffma2_rn(v, wk[kx], acc[(ixl - kx) / S]);
            }
          }
        }
        const float2 bd = __ldg(reinterpret_cast<const float2*>(p.bias_d + cbase) + cp);
        __half2* orow = reinterpret_cast<__half2*>(p.out) +
                        ((static_cast<size_t>(tl.n) * p.ho + oy0 + oyl) * p.wo + ox0) * cm2 +
                        (cbase >> 1) + cp;
#pragma unroll
        for (int i = 0; i < OTW; ++i) acc[i] = fadd2_rn(acc[i], bd);
#pragma unroll
        for (int i = 0; i + 1 < OTW; i += 2) apply_act4<ACT>(acc[i], acc[i + 1]);
        if (OTW & 1) acc[OTW - 1] = apply_act2<ACT>(acc[OTW - 1]);
        float2 ssum = make_float2(0.f, 0.f);
#pragma unroll
        for (int oxl = 0; oxl < OTW; ++oxl) {
          if (oxl < cols) {
            if (HAS_SE) ssum = fadd2_rn(ssum, acc[oxl]);
            orow[static_cast<size_t>(oxl) * cm2] = __floats2half2_rn(acc[oxl].x, acc[oxl].y);
          }
        }
        if (HAS_SE) {
          atomicAdd(&se_s[2 * cp], static_cast<unsigned long long>(__float2ll_rn(ssum.x * 1048576.f)));
          atomicAdd(&se_s[2 * cp + 1], static_cast<unsigned long long>(__float2ll_rn(ssum.y * 1048576.f)));
        }
      }
      }
      if (HAS_SE) {
        __syncthreads();
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(p.se_sum) +
                                  static_cast<size_t>(tl.n) * p.cmid + cbase;
        for (int i = threadIdx.x; i < cv; i += kThreads)
          if (se_s[i] != 0ull) atomicAdd(dst + i, se_s[i]);
      }
    }
    __syncthreads();   // E tile (and se_s) free for the next tile; next_tile_s published
    t = next_tile_s[it & 1];
  }
}

template <int K, int S>
static int launch(const CUtensorMap& mx, const CUtensorMap& mw, const Params& p, int grid,
                  int smem_bytes, int act, bool has_se, cudaStream_t stream) {
#define EDET_MBF(ACT, SE)                                                                     \
  do {                                                                                        \
    auto kern = mbconv_front_kernel<K, S, ACT, SE>;                                           \
    static int configured[kMaxDevices];                                                       \
    if (int rc = ensure_dynamic_smem(kern, 232448, configured)) return rc;                    \
    EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), smem_bytes, stream, mx, mw, p)); \
    return EDET_OK;                                                                           \
  } while (0)
  if (act == EDET_ACT_SWISH && has_se) EDET_MBF(EDET_ACT_SWISH, true);
  if (act == EDET_ACT_SWISH && !has_se) EDET_MBF(EDET_ACT_SWISH, false);
  if (act == EDET_ACT_RELU6 && has_se) EDET_MBF(EDET_ACT_RELU6, true);
  if (act == EDET_ACT_RELU6 && !has_se) EDET_MBF(EDET_ACT_RELU6, false);
#undef EDET_MBF
  set_error("mbconv_expand_dw: unsupported activation %d", act);
  return EDET_ERR_UNSUPPORTED;
}

}  // namespace mbf
}  // namespace edet

extern "C" int edet_mbconv_expand_dw(const edet_half* x, const edet_half* we, const float* bias_e,
                                     const float* wd, const float* bias_d, edet_half* out,
                                     int64_t* se_sum, int n, int h, int w, int cin, int cmid,
                                     int k, int stride, int act, edet_stream_t stream) {
  using namespace edet;
  using namespace edet::mbf;
  EDET_CHECK_ARG(x && we && bias_e && wd && bias_d && out, "mbconv_expand_dw: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && w > 0 && cin % 8 == 0 && cmid % 8 == 0,
                 "mbconv_expand_dw: cin %% 8 and cmid %% 8 required (got %d, %d)", cin, cmid);
  EDET_CHECK_ARG((k == 3 || k == 5) && (stride == 1 || stride == 2), "mbconv_expand_dw: k/stride");
  Params p;
  p.n = n; p.h = h; p.w = w; p.cin = cin; p.cmid = cmid;
  p.ho = ceil_div(h, stride); p.wo = ceil_div(w, stride);
  p.pad_t = same_pad_before(h, k, stride); p.pad_l = same_pad_before(w, k, stride);
  // channel chunks: <= kMaxCh accumulator columns (2 x kMaxCh / 2 registers per thread), so that
  // two CTAs share an SM; the last chunk may be partial (weights beyond cmid are TMA zero-fill and
  // never read back)
  p.num_chunks = ceil_div(cmid, kMaxCh);
  p.ch = ((ceil_div(cmid, p.num_chunks) + 15) / 16) * 16;
  p.oth = p.otw = (kPatch - k) / stride + 1;
  p.tiles_y = ceil_div(p.ho, p.oth); p.tiles_x = ceil_div(p.wo, p.otw);
  p.total_tiles = n * p.tiles_y * p.tiles_x * p.num_chunks;
  int smem_bytes = 0;
  for (int bk = cin <= 16 ? 16 : (cin <= 32 ? 32 : 64); bk >= 16; bk >>= 1) {
    p.block_k = bk;
    p.a_bytes = kPatchPx * bk * 2;
    p.b_bytes = ((p.ch * bk * 2 + 1023) / 1024) * 1024;
    smem_bytes = 1024 + p.a_bytes + p.b_bytes + kPatchPx * kEPitch + p.ch * 8 + 64;
    if (smem_bytes <= 113 * 1024 || bk == 32) break;   // two CTAs per SM, else settle for 32
  }
  p.num_k_blocks = ceil_div(cin, p.block_k);
  p.desc_layout = desc_layout_for(p.block_k);
  p.desc_sbo = 8 * p.block_k * 2;
  p.bias_e = bias_e; p.bias_d = bias_d;
  p.wd = wd;
  p.out = reinterpret_cast<__half*>(out);
  p.se_sum = reinterpret_cast<long long*>(se_sum);
  p.sched = next_sched_slot();
  if (!p.sched) return EDET_ERR_CUDA;
  EDET_CHECK_ARG(smem_bytes <= 232448, "mbconv_expand_dw: tile needs %d bytes of smem", smem_bytes);
  CUtensorMap mx, mw;
  int rc;
  if ((rc = make_map4(&mx, x, cin, w, h, n, p.block_k, kPatch, kPatch))) return rc;
  if ((rc = make_map(&mw, we, cin, cmid, 1, cin, static_cast<uint64_t>(cmid) * cin, p.ch, p.block_k)))
    return rc;
  const int sm_count = device_sm_count();
  if (!sm_count) return EDET_ERR_CUDA;
  // CTAs per SM the shared memory allows
  int per_sm = 232448 / (smem_bytes + 1024);
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 2) per_sm = 2;
  const int grid = p.total_tiles < per_sm * sm_count ? p.total_tiles : per_sm * sm_count;
  const bool has_se = se_sum != nullptr;
  cudaStream_t s = as_stream(stream);
  if (k == 3 && stride == 1) return launch<3, 1>(mx, mw, p, grid, smem_bytes, act, has_se, s);
  if (k == 3 && stride == 2) return launch<3, 2>(mx, mw, p, grid, smem_bytes, act, has_se, s);
  if (k == 5 && stride == 1) return launch<5, 1>(mx, mw, p, grid, smem_bytes, act, has_se, s);
  return launch<5, 2>(mx, mw, p, grid, smem_bytes, act, has_se, s);
}
