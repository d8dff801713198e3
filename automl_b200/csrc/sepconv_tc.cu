// Separable convolution of a head tower layer as ONE kernel:
//   depthwise 3x3 'SAME'  ->  pointwise 1x1 on the tensor cores (+ bias, BN folded) (+ act)
// The depthwise result never reaches HBM: it is written as fp16 straight into the 128B-swizzled
// K-major shared-memory tile that wgmma reads as its A operand.
//
// Replaces, per tower layer, efficientdet_arch.py:149-191 / 206-249 (SeparableConv2D, per-level
// BN, activation).  Algorithmic HBM bytes per launch: 2*N*h*w*(c + nout) + weights -- the
// [N,h,w,c] depthwise output (written and read back by a depthwise + pointwise pair) is gone.
//
// One CTA (one warpgroup) = one 8x16 output tile (128 pixels), persistent over tiles:
//   1. all warps: depthwise 3x3 -> fp16 A tile [128 px][c] (swizzled K-major atoms)
//   2. the warpgroup, per 64-pixel half: wgmma  D[64 px][nout] = A * W^T into registers
//      (W loaded once per CTA by TMA)
//   3. every thread: its accumulator fragment -> +bias, act -> fp16 -> global
//
// The whole-BiFPN-node form of this kernel (resample + weighted fusion + activation in front of
// the depthwise) was removed in round 2: measured on the D0 step it was slower than the
// fuse_dw + pointwise pair in both rounds (4.21 vs 3.76 ms per step with the pipelined engine):
// fusion, depthwise, MMA and epilogue serialise inside a CTA whose 100 KB of staging leaves two
// CTAs per SM.
#include "fuse_common.cuh"
#include "tc_common.cuh"

namespace edet {
namespace sepc {

using namespace pwtc;

constexpr int TH = 8, TW = 16;            // output tile: 128 pixels
constexpr int HT = TH + 2, WT = TW + 2;   // with halo
constexpr int kMaxC = 128, kMaxN = 128;
constexpr int kAtomBytesA = 128 * 128;    // [128 rows][64 halves]

struct Params {
  FuseParams fuse;
  const float* dw_w;      // fp32 taps [9][c]
  const float* bias;      // [nout]
  __half* out;            // [n, h, w, ldo]
  int n, h, w, c, nout, ldo;
  int katoms, kpad, npad, b_atom_bytes;
  int tiles_x, tiles_y, total_tiles;
  unsigned* sched;        // dynamic tile scheduler slot (direct kernel)
};

// ---- single-input form (head tower layers): depthwise straight from global memory ------------
// No fusion and no pre-activation, so the input tile needs no staging: each thread owns one
// channel pair x 4 columns x the 8 rows of the tile (the register tiling of depthwise.cu: fp32
// weights in registers, FFMA on channel pairs, loads software-pipelined two rows ahead), and drops its 32
// fp16 pairs into the swizzled A tile.  128 threads per CTA, up to 4 CTAs per SM.
constexpr int kDirectThreads = 128;

// Steps 2 + 3 of both kernels: D = A * W^T for the two 64-pixel halves of the tile in turn (64
// accumulator registers per thread), each followed by its epilogue straight from the fragments.
// A: katoms atoms of [128 px][64] halves (128B swizzle), B: katoms atoms of [npad][64].
template <int ACT_POST>
__device__ __forceinline__ void mma_epilogue(const Params& p, uint32_t a_u32, uint32_t b_u32,
                                             int katoms, int n, int y0, int x0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = p.npad >> 4;
  const int cq = 2 * (lane & 3);
#pragma unroll 1
  for (int mb = 0; mb < 2; ++mb) {
    float acc[kMaxN / 16][8] = {};
    wg_fence();
    for (int kb = 0; kb < katoms; ++kb) {
      const uint64_t da = make_smem_desc(a_u32 + kb * kAtomBytesA + mb * 64 * 128, 1024, 1);
      const uint64_t db = make_smem_desc(b_u32 + kb * p.b_atom_bytes, 1024, 1);
      wg_mma_kblock<kMaxN / 16>(acc, da, db, 128, nt, min(4, (p.kpad - kb * 64) >> 4), kb == 0);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc<kMaxN / 16>(acc);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = mb * 64 + 16 * warp + (lane >> 2) + 8 * r;
      const int y = y0 + row / TW, x = x0 + row % TW;
      if (y >= p.h || x >= p.w) continue;
      __half* orow = p.out + ((static_cast<size_t>(n) * p.h + y) * p.w + x) * p.ldo;
#pragma unroll
      for (int j = 0; j < kMaxN / 16; ++j) {
        const int col = 16 * j + cq;
        if (col >= p.nout) continue;
        const bool hi_ok = col + 8 < p.nout;
        const float2 b_lo = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        const float2 b_hi = hi_ok ? __ldg(reinterpret_cast<const float2*>(p.bias + col + 8))
                                  : make_float2(0.f, 0.f);
        float2 lo = fadd2_rn(make_float2(acc[j][2 * r], acc[j][2 * r + 1]), b_lo);
        float2 hi = fadd2_rn(make_float2(acc[j][4 + 2 * r], acc[j][4 + 2 * r + 1]), b_hi);
        if (ACT_POST != EDET_ACT_NONE) apply_act4<ACT_POST>(lo, hi);
        *reinterpret_cast<__half2*>(orow + col) = __floats2half2_rn(lo.x, lo.y);
        if (hi_ok) *reinterpret_cast<__half2*>(orow + col + 8) = __floats2half2_rn(hi.x, hi.y);
      }
    }
  }
}

template <int ACT_POST>
__global__ void __launch_bounds__(kDirectThreads, 4)
sepconv_direct_kernel(const __grid_constant__ CUtensorMap map_w, const Params p) {
  pdl_launch_dependents();
  constexpr int IN_ROWS = TH + 2, IN_COLS = 4 + 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + p.katoms * kAtomBytesA;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + p.katoms * p.b_atom_bytes);
  const uint32_t w_bar = smem_u32(bars);

  if (threadIdx.x == 0) {
    mbar_init(w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
  }
  // the K-padding channels of A multiply TMA-zero-filled weights: they must be finite -> zero A once
  for (int i = threadIdx.x; i < p.katoms * kAtomBytesA / 16; i += kDirectThreads)
    reinterpret_cast<uint4*>(smem_a)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(w_bar, static_cast<uint32_t>(p.katoms * p.npad * 128));
    for (int kb = 0; kb < p.katoms; ++kb)
      tma_load_3d(smem_u32(smem_b + kb * p.b_atom_bytes), &map_w, w_bar, kb * 64, 0, 0);
  }
  const int c = p.c, h = p.h, wd = p.w;
  const int cp_count = c >> 1;
  const int items = 4 * cp_count;   // (4-column group, channel pair)
  const FuseIn& src = p.fuse.in[0];
  const float2* w2 = reinterpret_cast<const float2*>(p.dw_w);
  pdl_wait_prior();

  const uint32_t a_u32 = smem_u32(smem_a);
  bool weights_ready = false;

  __shared__ int next_tile_s[2];   // double buffered: slot (it & 1) is rewritten two iterations later
  int t = blockIdx.x;
  for (int it = 0; t < p.total_tiles; ++it) {
    if (threadIdx.x == 0) next_tile_s[it & 1] = sched_next_tile(p.sched, p.total_tiles);
    const int tx_i = t % p.tiles_x;
    const int ty_i = (t / p.tiles_x) % p.tiles_y;
    const int n = t / (p.tiles_x * p.tiles_y);
    const int y0 = ty_i * TH, x0 = tx_i * TW;

    // ---- depthwise 3x3 -> A tile ---------------------------------------------------------------
    for (int e = threadIdx.x; e < items; e += kDirectThreads) {
      const int xg = e / cp_count, cp = e - xg * cp_count;
      float2 wreg[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) wreg[i] = __ldg(w2 + i * cp_count + cp);
      float2 acc[TH][4];
#pragma unroll
      for (int r = 0; r < TH; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[r][j] = make_float2(0.f, 0.f);
      const int ox0 = x0 + xg * 4;
      const int iy0 = y0 - 1, ix0 = ox0 - 1;
      const __half2* in2 = reinterpret_cast<const __half2*>(src.ptr) +
                           static_cast<size_t>(n) * h * wd * cp_count + cp;
      const int row_stride = wd * cp_count;
      const __half2* rowp = in2 + (iy0 * wd + ix0) * cp_count;
      const bool interior = iy0 >= 0 && iy0 + IN_ROWS <= h && ix0 >= 0 && ix0 + IN_COLS <= wd;
      if (interior) {
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
          for (int r = 0; r < TH; ++r) {
            const int ky = ir - r;
            if (ky >= 0 && ky < 3) {
#pragma unroll
              for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx)
                  acc[r][j] = ffma2_rn(xv[j + kx], wreg[ky * 3 + kx], acc[r][j]);
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
          for (int r = 0; r < TH; ++r) {
            const int ky = ir - r;
            if (ky >= 0 && ky < 3) {
#pragma unroll
              for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx)
                  acc[r][j] = ffma2_rn(xv[j + kx], wreg[ky * 3 + kx], acc[r][j]);
            }
          }
        }
      }
      // row = r * 16 + xg * 4 + j; 16-byte piece (cp >> 2) of the atom (cp >> 5), xor-swizzled
      const uint32_t abase = a_u32 + (cp >> 5) * kAtomBytesA + (cp & 3) * 4;
      const int piece = (cp >> 2) & 7;
#pragma unroll
      for (int r = 0; r < TH; ++r) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int row = r * TW + xg * 4 + j;
          const __half2 hv = __floats2half2_rn(acc[r][j].x, acc[r][j].y);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(abase + row * 128 + ((piece ^ (row & 7)) << 4)),
                       "r"(*reinterpret_cast<const uint32_t*>(&hv))
                       : "memory");
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (!weights_ready) {
      mbar_wait(w_bar, 0);
      weights_ready = true;
    }
    mma_epilogue<ACT_POST>(p, a_u32, smem_u32(smem_b), p.katoms, n, y0, x0);
    __syncthreads();
    t = next_tile_s[it & 1];
  }

  if (threadIdx.x == 0 && !weights_ready) mbar_wait(w_bar, 0);
}

// ---- single-input form, c <= 64, input tile staged by TMA --------------------------------------
// Same arithmetic and thread mapping as sepconv_direct_kernel, but the (8+2) x (16+2) x 64-channel
// input tile is fetched by one bulk tensor copy (out-of-image pixels arrive as zeros = 'SAME'
// padding, so there is no border path), double buffered: the NEXT tile's copy is issued as soon as
// its index is known and overlaps this tile's depthwise, MMA and epilogue.  The depthwise reads
// come from shared memory (128 contiguous bytes per warp and pixel, conflict free).
constexpr int kInTileBytes = HT * WT * 128;

// NBUF = 1 (default): one input buffer, refilled as soon as the depthwise phase has consumed it
// (the copy overlaps the MMA and the epilogue), which leaves room for four CTAs per SM;
// NBUF = 2 (sepconv_impl = 2): the next tile's copy is issued at the top of the iteration, three
// CTAs per SM.
template <int ACT_POST, int NBUF>
__global__ void __launch_bounds__(kDirectThreads, NBUF == 1 ? 4 : 3)
sepconv_direct_tma_kernel(const __grid_constant__ CUtensorMap map_w,
                          const __grid_constant__ CUtensorMap map_x, const Params p) {
  pdl_launch_dependents();
  constexpr int IN_ROWS = TH + 2, IN_COLS = 4 + 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;                                  // [128][64] halves, swizzled
  uint8_t* smem_b = smem_a + kAtomBytesA;                  // [npad][64] halves, swizzled
  uint8_t* smem_in = smem_b + p.b_atom_bytes;              // 2 x [HT][WT][64] halves, dense
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_in + NBUF * kInTileBytes);
  const uint32_t w_bar = smem_u32(bars);
  // [2] x {tile, image, tile row, tile column}: thread 0 decodes the next tile (its divisions)
  // when it fetches it; everybody reads the coordinates with one 16-byte load
  volatile int4* next_tile_s = reinterpret_cast<volatile int4*>(bars + 4);

  if (threadIdx.x == 0) {
    mbar_init(w_bar, 1);
    mbar_init(smem_u32(bars + 2), 1);
    mbar_init(smem_u32(bars + 3), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_x)) : "memory");
  }
  // the K-padding channels of A multiply TMA-zero-filled weights: they must be finite -> zero A once
  for (int i = threadIdx.x; i < kAtomBytesA / 16; i += kDirectThreads)
    reinterpret_cast<uint4*>(smem_a)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(w_bar, static_cast<uint32_t>(p.npad * 128));
    tma_load_3d(smem_u32(smem_b), &map_w, w_bar, 0, 0, 0);
  }
  const int c = p.c, h = p.h, wd = p.w;
  const int cp_count = c >> 1;
  const int items = 4 * cp_count;   // (4-column group, channel pair)
  const float2* w2 = reinterpret_cast<const float2*>(p.dw_w);
  pdl_wait_prior();

  auto decode = [&](int tile) -> int4 {                // {tile, image, tile row, tile column}
    if (tile >= p.total_tiles) return make_int4(tile, 0, 0, 0);
    const int tx_i = tile % p.tiles_x;
    const int rest = tile / p.tiles_x;
    return make_int4(tile, rest / p.tiles_y, rest % p.tiles_y, tx_i);
  };
  auto fetch_tile = [&](const int4& tc, int slot) {    // thread 0 only
    const uint32_t bar = smem_u32(bars + 2 + slot);
    mbar_expect_tx(bar, static_cast<uint32_t>(kInTileBytes));
    tma_load_4d(smem_u32(smem_in + slot * kInTileBytes), &map_x, bar, 0, tc.w * TW - 1, tc.z * TH - 1, tc.y);
  };

  const uint32_t a_u32 = smem_u32(smem_a);
  bool weights_ready = false;

  int4 cur = decode(blockIdx.x);
  if (threadIdx.x == 0 && cur.x < p.total_tiles) fetch_tile(cur, 0);
  for (int it = 0; cur.x < p.total_tiles; ++it) {
    if (threadIdx.x == 0) {
      // slot (it + 1) & 1 was last read in iteration it - 1, which ended with a CTA barrier
      const int4 nx = decode(sched_next_tile(p.sched, p.total_tiles));
      const_cast<int4*>(next_tile_s)[it & 1] = nx;
      if (NBUF == 2 && nx.x < p.total_tiles) fetch_tile(nx, (it + 1) & 1);
    }
    const int n = cur.y;
    const int y0 = cur.z * TH, x0 = cur.w * TW;

    // ---- depthwise 3x3 from the shared-memory tile -> A tile -----------------------------------
    mbar_wait(smem_u32(bars + 2 + (it % NBUF)), static_cast<uint32_t>(it / NBUF) & 1u);
    const uint32_t in_u32 = smem_u32(smem_in + (it % NBUF) * kInTileBytes);
    for (int e = threadIdx.x; e < items; e += kDirectThreads) {
      const int xg = e / cp_count, cp = e - xg * cp_count;
      float2 wreg[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) wreg[i] = __ldg(w2 + i * cp_count + cp);
      float2 acc[TH][4];
#pragma unroll
      for (int r = 0; r < TH; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[r][j] = make_float2(0.f, 0.f);
      const uint32_t base = in_u32 + static_cast<uint32_t>((xg * 4) * 128 + cp * 4);
#pragma unroll
      for (int ir = 0; ir < IN_ROWS; ++ir) {
        float2 xv[IN_COLS];
#pragma unroll
        for (int j = 0; j < IN_COLS; ++j) {
          uint32_t raw;
          asm volatile("ld.shared.b32 %0, [%1];" : "=r"(raw) : "r"(base + static_cast<uint32_t>((ir * WT + j) * 128)));
          xv[j] = __half22float2(*reinterpret_cast<const __half2*>(&raw));
        }
#pragma unroll
        for (int r = 0; r < TH; ++r) {
          const int ky = ir - r;
          if (ky >= 0 && ky < 3) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int kx = 0; kx < 3; ++kx)
                acc[r][j] = ffma2_rn(xv[j + kx], wreg[ky * 3 + kx], acc[r][j]);
          }
        }
      }
      // row = r * 16 + xg * 4 + j; 16-byte piece (cp >> 2), xor-swizzled
      const uint32_t abase = a_u32 + (cp & 3) * 4;
      const int piece = (cp >> 2) & 7;
#pragma unroll
      for (int r = 0; r < TH; ++r) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int row = r * TW + xg * 4 + j;
          const __half2 hv = __floats2half2_rn(acc[r][j].x, acc[r][j].y);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(abase + row * 128 + ((piece ^ (row & 7)) << 4)),
                       "r"(*reinterpret_cast<const uint32_t*>(&hv))
                       : "memory");
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (NBUF == 1 && threadIdx.x == 0) {       // the input buffer is free again: prefetch the next tile
      const int4 nx = const_cast<const int4*>(next_tile_s)[it & 1];
      if (nx.x < p.total_tiles) fetch_tile(nx, 0);
    }
    if (!weights_ready) {
      mbar_wait(w_bar, 0);
      weights_ready = true;
    }
    mma_epilogue<ACT_POST>(p, a_u32, smem_u32(smem_b), 1, n, y0, x0);
    __syncthreads();
    cur = const_cast<const int4*>(next_tile_s)[it & 1];
  }

  if (threadIdx.x == 0 && !weights_ready) mbar_wait(w_bar, 0);
}

template <int POST, int NBUF>
static int launch_direct_tma(const CUtensorMap& mw, const CUtensorMap& mx, const Params& p, int grid,
                             int smem_bytes, cudaStream_t stream) {
  auto kern = sepconv_direct_tma_kernel<POST, NBUF>;
  static int configured[kMaxDevices];
  if (int rc = ensure_dynamic_smem(kern, smem_bytes, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kDirectThreads), smem_bytes, stream, mw, mx, p));
  return EDET_OK;
}

template <int POST>
static int launch_direct(const CUtensorMap& mw, const Params& p, int grid, int smem_bytes,
                         cudaStream_t stream) {
  auto kern = sepconv_direct_kernel<POST>;
  static int configured[kMaxDevices];   // the kernel also has a few bytes of static shared memory
  if (int rc = ensure_dynamic_smem(kern, 232448 - 1024, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kDirectThreads), smem_bytes, stream, mw, p));
  return EDET_OK;
}

}  // namespace sepc
}  // namespace edet

extern "C" int edet_sepconv(const edet_fuse_input* h_inputs, int n_inputs, int pre_act,
                            const float* dw_w, const edet_half* pw_wt, const float* bias,
                            edet_half* out, int ldo, int n, int h, int wd, int c, int nout,
                            int post_act, edet_stream_t stream) {
  using namespace edet;
  using namespace edet::sepc;
  EDET_CHECK_ARG(dw_w && pw_wt && bias && out, "sepconv: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && wd > 0 && c > 0 && c % 8 == 0 && c <= kMaxC,
                 "sepconv: c must be a multiple of 8 and <= %d (got %d)", kMaxC, c);
  EDET_CHECK_ARG(nout > 0 && nout % 8 == 0 && nout <= kMaxN && ldo >= nout && ldo % 8 == 0,
                 "sepconv: nout must be a multiple of 8 and <= %d, ldo >= nout (got %d, %d)", kMaxN,
                 nout, ldo);
  Params p;
  if (int rc = fill_fuse_params(h_inputs, n_inputs, h, wd, "sepconv", &p.fuse)) return rc;
  p.dw_w = dw_w;
  p.bias = bias;
  p.out = reinterpret_cast<__half*>(out);
  p.n = n; p.h = h; p.w = wd; p.c = c; p.nout = nout; p.ldo = ldo;
  p.katoms = ceil_div(c, 64);
  p.kpad = ((c + 15) / 16) * 16;
  p.npad = ((nout + 15) / 16) * 16;
  p.b_atom_bytes = ((p.npad * 128 + 1023) / 1024) * 1024;
  p.tiles_x = ceil_div(wd, TW); p.tiles_y = ceil_div(h, TH);
  p.total_tiles = n * p.tiles_x * p.tiles_y;
  CUtensorMap mw;
  if (int rc = make_map(&mw, pw_wt, c, nout, 1, c, static_cast<uint64_t>(nout) * c, p.npad, 64))
    return rc;
  cudaStream_t s = as_stream(stream);
  if (int rc = next_sched_slot(&p.sched)) return rc;
  const bool direct = n_inputs == 1 && p.fuse.in[0].mode == EDET_RS_SAME &&
                      p.fuse.in[0].weight == 1.0f && pre_act == EDET_ACT_NONE;
  const int smem_bytes = 1024 + p.katoms * (kAtomBytesA + p.b_atom_bytes) + 64;
  int per_sm = 232448 / (smem_bytes + 1024);
  const int cap = 4;
  if (per_sm > cap) per_sm = cap;
  if (per_sm < 1) per_sm = 1;
  const int grid = persistent_grid(p.total_tiles, per_sm);
  if (!grid) return EDET_ERR_CUDA;
  if (direct && p.katoms == 1 && option_sepconv_impl() != 1) {
    // c <= 64: the input tile comes through TMA, double buffered (sepconv_direct_tma_kernel)
    CUtensorMap mx;
    if (int rc = make_map4(&mx, p.fuse.in[0].ptr, c, wd, h, n, 64, WT, HT, /*swizzle=*/false)) return rc;
    // one input buffer / four CTAs per SM by default (measured on the D0 step: 3.74 vs 3.765 ms)
    const int nbuf = option_sepconv_impl() == 2 ? 2 : 1;
    const int smem_tma = 1024 + kAtomBytesA + p.b_atom_bytes + nbuf * kInTileBytes + 128;
    int per = 232448 / (smem_tma + 1024);
    if (per > (nbuf == 1 ? 4 : 3)) per = nbuf == 1 ? 4 : 3;
    const int grid_tma = persistent_grid(p.total_tiles, per);
#define EDET_SEPC_TMA(POST)                                                                   \
  if (post_act == POST)                                                                       \
    return nbuf == 1 ? launch_direct_tma<POST, 1>(mw, mx, p, grid_tma, smem_tma, s)           \
                     : launch_direct_tma<POST, 2>(mw, mx, p, grid_tma, smem_tma, s)
    EDET_SEPC_TMA(EDET_ACT_SWISH);
    EDET_SEPC_TMA(EDET_ACT_RELU6);
    EDET_SEPC_TMA(EDET_ACT_NONE);
#undef EDET_SEPC_TMA
    set_error("sepconv: unsupported activation %d", post_act);
    return EDET_ERR_UNSUPPORTED;
  }
  if (direct) {
    if (post_act == EDET_ACT_SWISH) return launch_direct<EDET_ACT_SWISH>(mw, p, grid, smem_bytes, s);
    if (post_act == EDET_ACT_RELU6) return launch_direct<EDET_ACT_RELU6>(mw, p, grid, smem_bytes, s);
    if (post_act == EDET_ACT_NONE) return launch_direct<EDET_ACT_NONE>(mw, p, grid, smem_bytes, s);
    set_error("sepconv: unsupported activation %d", post_act);
    return EDET_ERR_UNSUPPORTED;
  }
  set_error("sepconv: only the single-input form (one RS_SAME input, weight 1, no pre-activation) "
            "exists; BiFPN nodes run edet_fuse_dw + edet_pointwise_conv");
  return EDET_ERR_UNSUPPORTED;
}
