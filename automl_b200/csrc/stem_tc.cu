// Stem on the tensor cores: Conv2D 3x3 stride 2 'SAME', 3 -> cout, + folded BN + activation, as an
// implicit GEMM  D[128 px][cout] = A[128 px][64] * W'[cout][64]^T  per 8 x 16 output tile.
//
// The image arrives as float32 (what the reference feeds the network, efficientnet_model.py:
// 526-527).  To keep its precision on the fp16 tensor-core path every input value is split into
// two fp16 terms, x = hi + lo (hi = fp16(x), lo = fp16(x - hi): ~22 significant bits), and the 27
// taps become K = 54 (padded to 64 = one 128-byte swizzled K atom): columns 0..26 hold hi, 27..53
// hold lo, and W' repeats the 27 fp16 weights for both halves.  fp32 accumulation in registers.
// The 27-MAC-per-output CUDA-core kernel (stem.cu) was FFMA-issue bound at 0.21 of the HBM
// roofline; here the arithmetic is 2 x 4 wgmma per tile and the CUDA cores only build the A
// tile (27 loads + 27 splits per pixel) and run the epilogue.
//
// One CTA (128 threads = one warpgroup, one thread per output pixel of the tile when the A tile
// is built) per tile, persistent with the dynamic tile scheduler, up to 4 CTAs per SM:
//   1. all threads: the (17 x 33 x 3) float32 input patch -> shared memory with cp.async (coalesced,
//      zero filled outside the image = 'SAME' padding), double buffered: the NEXT tile's patch is
//      in flight while this tile is converted, multiplied and written out
//   2. thread m: its 27 inputs -> hi / lo halves -> row m of the swizzled A tile
//   3. the warpgroup: wgmma (two M 64 halves, N cout rounded to 16, K 16) into registers
//   4. every thread: its accumulator fragment -> + bias -> activation -> fp16 -> global
// Bytes per launch (SURVEY.md 8d): 12*n*h*w + 2*n*ho*wo*cout.
#include "tc_common.cuh"

namespace edet {
namespace stemtc {

using namespace pwtc;

constexpr int kThreads = 128;
constexpr int TH = 8, TW = 16;                       // output tile: 128 pixels = two wgmma M blocks
constexpr int IH = 2 * TH + 1, IW = 2 * TW + 1;      // input patch (stride 2, 3 x 3 window)
constexpr int kRowFloats = IW * 3;                   // 99 floats per patch row
constexpr int kInFloats = IH * kRowFloats;           // 1683
constexpr int kInPad = (kInFloats + 3) & ~3;         // floats per (double-buffered) patch slot
constexpr int kABytes = 128 * 128;                   // [128 rows][64 halves]
constexpr int kMaxN = 64;
constexpr int kBBytes = kMaxN * 128;

__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
// 4-byte asynchronous global -> shared copy; src_bytes == 0 writes a zero (the 'SAME' padding)
__device__ __forceinline__ void cp_async_f32(uint32_t dst, const float* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src),
               "r"(valid ? 4 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

struct Params {
  const float* in;      // [n, h, w, 3]
  __half* out;          // [n, ho, wo, cout]
  const __half* wgt;    // [27][cout]  (ky, kx, cin major; BN scale folded)
  const float* bias;    // [cout]
  int n, h, w, ho, wo, cout, npad, pad_t, pad_l;
  int tiles_x, tiles_y, total_tiles;
  unsigned* sched;
};

template <int ACT>
__global__ void __launch_bounds__(kThreads, 4)
stem_tc_kernel(const Params p) {
  pdl_launch_dependents();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + kABytes;
  float* in_s = reinterpret_cast<float*>(smem_b + kBBytes);                 // [2][IH][IW][3]
  // [2] x {tile, image, tile row, tile column}: thread 0 decodes the next tile once (the integer
  // divisions); everybody reads the coordinates with one 16-byte load
  volatile int4* next_tile_s = reinterpret_cast<volatile int4*>(in_s + 2 * kInPad);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // W' tile [npad][64] (K-major, 128B swizzle): k < 27 -> w[k], 27 <= k < 54 -> w[k - 27], else 0;
  // rows >= cout are zero.  Constants: built before the PDL wait.
  for (int i = threadIdx.x; i < p.npad * 64; i += kThreads) {
    const int nrow = i >> 6, k = i & 63;
    __half v = __float2half_rn(0.f);
    if (nrow < p.cout && k < 54) v = __ldg(p.wgt + (k < 27 ? k : k - 27) * p.cout + nrow);
    *reinterpret_cast<__half*>(smem_b + nrow * 128 + ((((k >> 3) ^ (nrow & 7))) << 4) + (k & 7) * 2) = v;
  }
  fence_proxy_async_smem();
  __syncthreads();
  pdl_wait_prior();

  const uint32_t a_u32 = smem_u32(smem_a);
  const uint32_t in_u32 = smem_u32(in_s);
  const int nt = p.npad >> 4;
  const int m = threadIdx.x;                         // this thread's pixel of the tile
  const int mr = m / TW, mc = m % TW;
  const int row_floats = p.w * 3;

  // The input patch of the NEXT tile is fetched with cp.async (4-byte copies, zero fill outside the
  // image) into the other half of a double buffer while the current tile is converted, multiplied
  // and written out, so its global-memory latency is off the critical path.
  auto decode = [&](int tile) -> int4 {              // {tile, image, tile row, tile column}
    if (tile >= p.total_tiles) return make_int4(tile, 0, 0, 0);
    const int rest = tile / p.tiles_x;
    return make_int4(tile, rest / p.tiles_y, rest % p.tiles_y, tile % p.tiles_x);
  };
  auto fetch_patch = [&](const int4& tc, int slot) {
    const int tx_i = tc.w, ty_i = tc.z, n = tc.y;
    const int iy0 = ty_i * TH * 2 - p.pad_t;
    const int xf0 = (tx_i * TW * 2 - p.pad_l) * 3;     // first float of the patch inside an image row
    const float* img = p.in + static_cast<size_t>(n) * p.h * row_floats;
    const uint32_t dst = in_u32 + slot * kInPad * 4;
    int r = 0, cf = threadIdx.x;                      // kThreads (128) = kRowFloats (99) + 29
    if (cf >= kRowFloats) { cf -= kRowFloats; r = 1; }
    for (int i = threadIdx.x; i < kInFloats; i += kThreads) {
      const int iy = iy0 + r, xf = xf0 + cf;
      const bool ok = iy >= 0 && iy < p.h && xf >= 0 && xf < row_floats;
      cp_async_f32(dst + i * 4, ok ? img + static_cast<size_t>(iy) * row_floats + xf : p.in, ok);
      r += 1; cf += kThreads - kRowFloats;
      if (cf >= kRowFloats) { cf -= kRowFloats; r += 1; }
    }
    cp_async_commit();
  };

  int4 cur = decode(blockIdx.x);
  if (cur.x < p.total_tiles) fetch_patch(cur, 0);
  for (int it = 0; cur.x < p.total_tiles; ++it) {
    if (threadIdx.x == 0)
      const_cast<int4*>(next_tile_s)[it & 1] = decode(sched_next_tile(p.sched, p.total_tiles));
    const int n = cur.y;
    const int y0 = cur.z * TH, x0 = cur.w * TW;

    // ---- 1. this tile's patch has landed; start fetching the next tile's ------------------------
    cp_async_wait_all();
    __syncthreads();                                   // patch + next_tile_s visible to everyone
    const int4 nxt = const_cast<const int4*>(next_tile_s)[it & 1];
    if (nxt.x < p.total_tiles) fetch_patch(nxt, (it + 1) & 1);
    const uint32_t patch_u32 = in_u32 + (it & 1) * kInPad * 4;
    // ---- 2. A row m: 27 hi halves, 27 lo halves, 10 zeros -> 8 swizzled 16-byte pieces ----------
    {
      const uint32_t src = patch_u32 + (2 * mr * IW + 2 * mc) * 3 * 4;
      __half hv[64];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
        for (int j = 0; j < 9; ++j) {                // (kx, ci) are contiguous in the patch row
          const float x = lds_f32(src + (ky * kRowFloats + j) * 4);
          const __half hi = __float2half_rn(x);
          hv[ky * 9 + j] = hi;
          hv[27 + ky * 9 + j] = __float2half_rn(x - __half2float(hi));
        }
      }
#pragma unroll
      for (int k = 54; k < 64; ++k) hv[k] = __float2half_rn(0.f);
      const uint32_t arow = a_u32 + m * 128;
#pragma unroll
      for (int piece = 0; piece < 8; ++piece) {
        uint32_t w0, w1, w2, w3;
        auto pack = [&](int k) {
          const __half2 h2 = __halves2half2(hv[k], hv[k + 1]);
          return *reinterpret_cast<const uint32_t*>(&h2);
        };
        w0 = pack(piece * 8); w1 = pack(piece * 8 + 2); w2 = pack(piece * 8 + 4); w3 = pack(piece * 8 + 6);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(arow + ((piece ^ (m & 7)) << 4)),
                     "r"(w0), "r"(w1), "r"(w2), "r"(w3)
                     : "memory");
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    // ---- 3. D = A * W'^T: rows 64 mb .. 64 mb + 63 into acc[mb] -----------------------------------
    float acc[2][kMaxN / 16][8] = {};
    {
      const uint64_t db = make_smem_desc(smem_u32(smem_b), 1024, 1);
      wg_fence();
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
        wg_mma_kblock<kMaxN / 16>(acc[mb], make_smem_desc(a_u32 + mb * 64 * 128, 1024, 1), db, 128,
                                  nt, 4, true);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc<kMaxN / 16>(acc[0]);
      wg_fence_acc<kMaxN / 16>(acc[1]);
    }
    // ---- 4. epilogue from the accumulator fragments: rows r0, r0 + 8 of each M block ------------
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = mb * 64 + 16 * warp + (lane >> 2) + 8 * r;
        const int y = y0 + row / TW, x = x0 + row % TW;
        if (y >= p.ho || x >= p.wo) continue;
        __half* orow = p.out + ((static_cast<size_t>(n) * p.ho + y) * p.wo + x) * p.cout;
#pragma unroll
        for (int j = 0; j < kMaxN / 16; ++j) {
          const int col = 16 * j + 2 * (lane & 3);
          if (col >= p.cout) continue;
          const bool hi_ok = col + 8 < p.cout;
          const float2 b_lo = __ldg(reinterpret_cast<const float2*>(p.bias + col));
          const float2 b_hi = hi_ok ? __ldg(reinterpret_cast<const float2*>(p.bias + col + 8))
                                    : make_float2(0.f, 0.f);
          float2 lo = fadd2_rn(make_float2(acc[mb][j][2 * r], acc[mb][j][2 * r + 1]), b_lo);
          float2 hi = fadd2_rn(make_float2(acc[mb][j][4 + 2 * r], acc[mb][j][4 + 2 * r + 1]), b_hi);
          apply_act4<ACT>(lo, hi);
          *reinterpret_cast<__half2*>(orow + col) = __floats2half2_rn(lo.x, lo.y);
          if (hi_ok) *reinterpret_cast<__half2*>(orow + col + 8) = __floats2half2_rn(hi.x, hi.y);
        }
      }
    }
    __syncthreads();       // A and the input patch are free for the next tile
    cur = nxt;
  }
}

template <int ACT>
static int launch(const Params& p, int grid, int smem_bytes, cudaStream_t stream) {
  auto kern = stem_tc_kernel<ACT>;
  static int configured[kMaxDevices];
  if (int rc = ensure_dynamic_smem(kern, smem_bytes, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), smem_bytes, stream, p));
  return EDET_OK;
}

bool eligible(int cout) { return cout % 8 == 0 && cout <= kMaxN; }

int run(const float* in, __half* out, const __half* w, const float* bias, int n, int h, int wd,
        int cout, int act, cudaStream_t stream) {
  Params p;
  p.in = in; p.out = out; p.wgt = w; p.bias = bias;
  p.n = n; p.h = h; p.w = wd; p.cout = cout;
  p.ho = ceil_div(h, 2); p.wo = ceil_div(wd, 2);
  p.npad = ((cout + 15) / 16) * 16;
  p.pad_t = same_pad_before(h, 3, 2); p.pad_l = same_pad_before(wd, 3, 2);
  p.tiles_x = ceil_div(p.wo, TW); p.tiles_y = ceil_div(p.ho, TH);
  const long long total = static_cast<long long>(n) * p.tiles_x * p.tiles_y;
  EDET_CHECK_ARG(total < 0x7fffffffLL, "stem: too many tiles");
  p.total_tiles = static_cast<int>(total);
  p.sched = next_sched_slot();
  if (!p.sched) return EDET_ERR_CUDA;
  const int sms = device_sm_count();
  if (!sms) return EDET_ERR_CUDA;
  const int smem_bytes = 1024 + kABytes + kBBytes + 2 * kInPad * 4 + 32;
  int per_sm = 232448 / (smem_bytes + 1024);
  if (per_sm > 4) per_sm = 4;
  const int grid = p.total_tiles < per_sm * sms ? p.total_tiles : per_sm * sms;
  if (act == EDET_ACT_SWISH) return launch<EDET_ACT_SWISH>(p, grid, smem_bytes, stream);
  if (act == EDET_ACT_RELU6) return launch<EDET_ACT_RELU6>(p, grid, smem_bytes, stream);
  if (act == EDET_ACT_NONE) return launch<EDET_ACT_NONE>(p, grid, smem_bytes, stream);
  set_error("stem: unsupported activation %d", act);
  return EDET_ERR_UNSUPPORTED;
}

}  // namespace stemtc
}  // namespace edet
