// k x k convolution ('SAME', stride 1 or 2, NHWC fp16) as an implicit GEMM on the Hopper tensor
// cores (wgmma): the Fused-MBConv convolutions of EfficientNetV2
// (efficientnetv2/effnetv2_model.py:331-341 expand k x k + BN + act, :355-364 the single k x k conv
// of expand_ratio == 1 blocks, :387-404 their use).
//
//   out[n, y, x, :] = act( sum_{ky,kx,c} in[n, y*s + ky - pt, x*s + kx - pl, c] * W[ky*k+kx][:, c] + bias )
//                     (+ residual[n, y, x, :])
//
// Same persistent, warp-specialised structure as pointwise_tc.cu (TMA producer warp, two consumer
// warpgroups taking tiles in turn, each with a stage ring of its own: wgmma main loop with fp32 accumulators in registers, then a
// TMA-store epilogue, one CTA per SM).  The M tile is a 4 x 16 block of output pixels; the K loop
// runs over (tap, 64-channel block): for each tap the A operand is the SAME input tensor fetched
// by a 4-D TMA box {64 ch, 16, 4, 1} shifted by the tap offset -- out-of-image pixels are
// zero-filled by TMA, which is exactly the zero padding of 'SAME' -- so im2col never exists
// anywhere.  Stride 2 uses four tensor maps, one per (row parity, column parity) sub-image of the
// input, so every tap is again a dense box.
// Algorithmic HBM bytes per launch: 2*N*(H*W*Cin + Ho*Wo*Cout [+ residual]) + 2*k*k*Cout*Cin.
#include "tc_common.cuh"

namespace edet {
namespace convtc {

using namespace pwtc;   // PTX wrappers and tensor-map encoders of tc_common.cuh

constexpr int TH = 4, TW = 16;   // output pixel tile = the 64 rows of one wgmma
constexpr int BLOCK_M = TH * TW;
constexpr int kConsumers = 2;
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kMaxBlockN = 128;
constexpr int kNT = kMaxBlockN / 16;
constexpr int kStoreCols = 64;
constexpr int kSlabBytes = BLOCK_M * kStoreCols * 2;   // [64 px][64 cols] fp16, 128B swizzle
constexpr int kSlabsPerTeam = kMaxBlockN / kStoreCols;
constexpr int kMaxStages = 8;
constexpr int kSmemLimit = 227 * 1024;                 // one CTA per SM

struct Maps {
  CUtensorMap a[4];   // input (stride 1: a[0]) or its four (row parity, column parity) sub-images
  CUtensorMap w;      // weights [taps][cout][cin]
  CUtensorMap o;      // output [n][ho][wo][cout]
};

struct Params {
  int batch, k, nout, nout_pad8;   // k = cin
  int ho, wo, ksize, stride, pad_t, pad_l, tiles_x, tiles_y, taps;
  int block_n, num_m_blocks, num_n_blocks, num_k_blocks, num_stages;
  int team_stages;    // stages of each consumer's own ring: num_stages / kConsumers
  int block_k;        // 64 / 32 / 16 halves per k-block == 128B / 64B / 32B swizzled smem rows
  int a_stage_bytes, b_stage_bytes;
  int desc_sbo;       // byte distance between 8-row groups in smem (8 * row pitch)
  int desc_layout;    // wgmma layout type: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B
  int ldr;
  int no_odd_col, no_odd_row;   // stride 2 on a 1-wide / 1-high input: that sub-image is empty
  int total_tiles;
  const float* bias;
  const __half* residual;
};

struct TileCoord {
  int b, ty, tx, n_blk;
};
__device__ __forceinline__ TileCoord decode_tile(int t, const Params& p) {
  TileCoord c;
  c.n_blk = t % p.num_n_blocks;
  t /= p.num_n_blocks;
  c.tx = t % p.tiles_x;
  t /= p.tiles_x;
  c.ty = t % p.tiles_y;
  c.b = t / p.tiles_y;
  return c;
}

template <int ACT, bool HAS_RES>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ Maps maps, const Params p) {
  const CUtensorMap& map_w = maps.w;
  const CUtensorMap& map_o = maps.o;
  pdl_launch_dependents();   // the next kernel may start its prologue while this one runs
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for the swizzle atoms.
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = p.a_stage_bytes + p.b_stage_bytes;
  uint8_t* smem_store = smem + p.num_stages * stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_store + kConsumers * kSlabsPerTeam * kSlabBytes);
  uint64_t* full_bar = bars;                       // [kMaxStages]
  uint64_t* empty_bar = bars + kMaxStages;         // [kMaxStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 4);       // one arrive per warp of the consumer
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.a[0])) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_o)) : "memory");
  }
  __syncthreads();
  pdl_wait_prior();          // everything above overlapped the previous kernel's tail

  const int kk_per_tile = p.taps * p.num_k_blocks;
  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage_of[kConsumers] = {}, phase_of[kConsumers] = {};   // per consumer ring
      // bytes the two TMA boxes deliver (the B slot may be padded to 1 KiB)
      const uint32_t tx_bytes = static_cast<uint32_t>(p.a_stage_bytes + p.block_n * p.block_k * 2);
      int iter = 0;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++iter) {
        const TileCoord tc = decode_tile(t, p);
        const int team = iter % kConsumers;
        int stage = stage_of[team];
        uint32_t phase = static_cast<uint32_t>(phase_of[team]);
        for (int kk = 0; kk < kk_per_tile; ++kk) {
          const int tap = kk / p.num_k_blocks, kb = kk - tap * p.num_k_blocks;
          const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
          // input pixel of output (y, x) for this tap: (y*s + ry, x*s + rx)
          const int ry = ky - p.pad_t, rx = kx - p.pad_l;
          int map_id = 0, cy = tc.ty * TH + ry, cx = tc.tx * TW + rx;
          if (p.stride == 2) {   // sub-image (ry mod 2, rx mod 2), shifted by floor(r / 2)
            const int py = ry & 1, px = rx & 1;
            map_id = py * 2 + px;
            cy = tc.ty * TH + ((ry - py) >> 1);
            cx = tc.tx * TW + ((rx - px) >> 1);
            // an empty sub-image has a stand-in map whose one column (row) is real memory: move
            // the box off it, where TMA reads the zeros of the 'SAME' padding
            if (px && p.no_odd_col) cx = -TW;
            if (py && p.no_odd_row) cy = -TH;
          }
          const int s = team * p.team_stages + stage;
          mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
          const uint32_t fb = smem_u32(&full_bar[s]);
          mbar_expect_tx(fb, tx_bytes);
          uint8_t* sa = smem + s * stage_bytes;
          tma_load_4d(smem_u32(sa), &maps.a[map_id], fb, kb * p.block_k, cx, cy, tc.b);
          tma_load_3d(smem_u32(sa + p.a_stage_bytes), &map_w, fb, kb * p.block_k,
                      tc.n_blk * p.block_n, tap);
          if (++stage == p.team_stages) {
            stage = 0;
            phase ^= 1;
          }
        }
        stage_of[team] = stage;
        phase_of[team] = static_cast<int>(phase);
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: MMA + epilogue =====================
    const int team = (warp >> 2) - 1;
    const int wtid = threadIdx.x & 127;
    const int r0 = 16 * (warp & 3) + (lane >> 2);   // tile rows (pixels) r0 and r0 + 8
    const int cq = 2 * (lane & 3);
    uint8_t* my_slabs = smem_store + team * kSlabsPerTeam * kSlabBytes;
    const int b_chunk = p.block_k * 2;
    int stage = 0;
    uint32_t phase = 0;
    int iter = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++iter) {
      if (iter % kConsumers != team) continue;   // the other consumer's tile (and ring)
      const TileCoord tc = decode_tile(t, p);
      const int n0 = tc.n_blk * p.block_n;
      const int n_valid = min(p.block_n, ((p.nout - n0 + 15) >> 4) << 4);
      const int nt = n_valid >> 4;
      float acc[kNT][8];
#pragma unroll
      for (int j = 0; j < kNT; ++j)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[j][q] = 0.f;
      for (int kk = 0; kk < kk_per_tile; ++kk) {
        const int kb = kk % p.num_k_blocks;
        const int s = team * p.team_stages + stage;
        mbar_wait(smem_u32(&full_bar[s]), phase);
        uint8_t* sa = smem + s * stage_bytes;
        const uint64_t da = make_smem_desc(smem_u32(sa), p.desc_sbo, p.desc_layout);
        const uint64_t db = make_smem_desc(smem_u32(sa + p.a_stage_bytes), p.desc_sbo, p.desc_layout);
        const int k_rem = p.k - kb * p.block_k;
        const int ksteps = k_rem >= p.block_k ? p.block_k / MMA_K : (k_rem + MMA_K - 1) / MMA_K;
        wg_fence();
        wg_mma_kblock<kNT>(acc, da, db, b_chunk, nt, ksteps, kk == 0);
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));
        if (++stage == p.team_stages) { stage = 0; phase ^= 1; }
      }
      wg_fence_acc<kNT>(acc);
      bool ok[2];
      const __half* res_row[2] = {nullptr, nullptr};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int m = r0 + 8 * r;
        const int oy = tc.ty * TH + m / TW, ox = tc.tx * TW + m % TW;
        ok[r] = oy < p.ho && ox < p.wo;
        if (HAS_RES)
          res_row[r] = p.residual +
                       ((static_cast<size_t>(tc.b) * p.ho + (ok[r] ? oy : 0)) * p.wo + (ok[r] ? ox : 0)) * p.ldr;
      }
      if (wtid == 0) tma_store_wait_read<0>();
      named_sync(1 + team, 128);
#pragma unroll
      for (int j = 0; j < kNT; ++j) {
        if (j < nt) {
          const int colt = 16 * j + cq;
          float b[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {     // columns colt, colt + 1, colt + 8, colt + 9
            const int col = n0 + colt + (e >> 1) * 8 + (e & 1);
            b[e] = col < p.nout ? __ldg(p.bias + col) : 0.f;
          }
          uint8_t* slab = my_slabs + (colt >> 6) * kSlabBytes;
          const int piece = (colt & 63) >> 3;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float2 lo = fadd2_rn(make_float2(acc[j][2 * r], acc[j][2 * r + 1]), make_float2(b[0], b[1]));
            float2 hi = fadd2_rn(make_float2(acc[j][4 + 2 * r], acc[j][4 + 2 * r + 1]), make_float2(b[2], b[3]));
            apply_act4<ACT>(lo, hi);
            if (HAS_RES && ok[r]) {
              const int col = n0 + colt;
              if (col < p.nout)
                lo = fadd2_rn(lo, __half22float2(*reinterpret_cast<const __half2*>(res_row[r] + col)));
              if (col + 8 < p.nout)
                hi = fadd2_rn(hi, __half22float2(*reinterpret_cast<const __half2*>(res_row[r] + col + 8)));
            }
            const int row = r0 + 8 * r;
            uint8_t* rb = slab + row * 128 + cq * 2;
            *reinterpret_cast<__half2*>(rb + ((piece ^ (row & 7)) << 4)) = __floats2half2_rn(lo.x, lo.y);
            *reinterpret_cast<__half2*>(rb + (((piece + 1) ^ (row & 7)) << 4)) = __floats2half2_rn(hi.x, hi.y);
          }
        }
      }
      fence_proxy_async_smem();
      named_sync(1 + team, 128);
      if (wtid == 0) {
        // the 64 rows are four tile rows of 16 pixels: one 4-D box {64, 16, 4, 1} per 64 columns
        for (int c = 0; c * kStoreCols < n_valid; ++c)
          tma_store_4d(&map_o, smem_u32(my_slabs + c * kSlabBytes), n0 + c * kStoreCols, tc.tx * TW,
                       tc.ty * TH, tc.b);
        tma_store_commit();
      }
    }
    if (wtid == 0) tma_store_wait_all();
  }
}

// N tile: the whole width up to 128 columns, else tiles of 128 (a multiple of the 64-column
// store box); the A tile of the extra tiles comes from L2.
static int pick_block_n(int nout) {
  if (nout <= kMaxBlockN) return ((nout + 15) / 16) * 16;
  return kMaxBlockN;
}

template <int ACT, bool HAS_RES>
static int launch(const Maps& maps, const Params& p, int grid, int smem_bytes, cudaStream_t stream) {
  auto kern = conv_tc_kernel<ACT, HAS_RES>;
  static int configured[kMaxDevices];
  if (int rc = ensure_dynamic_smem(kern, kSmemLimit, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), smem_bytes, stream, maps, p));
  return EDET_OK;
}

}  // namespace convtc
}  // namespace edet

extern "C" int edet_conv2d(const edet_half* in, const edet_half* wt, const float* bias,
                           const edet_half* residual, edet_half* out, int n, int h, int w, int cin,
                           int cout, int ksize, int stride, int act, edet_stream_t stream) {
  using namespace edet;
  using namespace edet::convtc;
  EDET_CHECK_ARG(in && wt && bias && out, "conv2d: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && w > 0 && cin > 0 && cin % 8 == 0 && cout > 0 && cout % 8 == 0,
                 "conv2d: cin and cout must be multiples of 8 (got %d, %d)", cin, cout);
  EDET_CHECK_ARG((ksize == 1 || ksize == 3 || ksize == 5) && (stride == 1 || stride == 2),
                 "conv2d: ksize in {1,3,5}, stride in {1,2} (got %d, %d)", ksize, stride);
  Params p;
  p.batch = n; p.k = cin; p.nout = cout; p.nout_pad8 = cout & ~7;
  p.ksize = ksize; p.stride = stride; p.taps = ksize * ksize;
  p.ho = ceil_div(h, stride); p.wo = ceil_div(w, stride);
  p.pad_t = same_pad_before(h, ksize, stride); p.pad_l = same_pad_before(w, ksize, stride);
  p.tiles_x = ceil_div(p.wo, TW); p.tiles_y = ceil_div(p.ho, TH);
  p.block_n = pick_block_n(cout);
  p.num_m_blocks = p.tiles_x * p.tiles_y;
  p.num_n_blocks = ceil_div(cout, p.block_n);
  p.block_k = cin <= 16 ? 16 : (cin <= 32 ? 32 : 64);
  p.desc_layout = desc_layout_for(p.block_k);
  p.desc_sbo = 8 * p.block_k * 2;
  p.num_k_blocks = ceil_div(cin, p.block_k);
  p.a_stage_bytes = BLOCK_M * p.block_k * 2;
  p.b_stage_bytes = ((p.block_n * p.block_k * 2 + 1023) / 1024) * 1024;
  p.ldr = cout;
  p.no_odd_col = stride == 2 && w == 1;
  p.no_odd_row = stride == 2 && h == 1;
  p.bias = bias;
  p.residual = reinterpret_cast<const __half*>(residual);
  p.total_tiles = n * p.num_m_blocks * p.num_n_blocks;
  const int stage_bytes = p.a_stage_bytes + p.b_stage_bytes;
  const int fixed = kConsumers * kSlabsPerTeam * kSlabBytes + 2 * kMaxStages * 8;
  int stages = (kSmemLimit - 1024 - fixed) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.team_stages = stages / kConsumers;       // each consumer's own ring
  EDET_CHECK_ARG(p.team_stages >= 2, "conv2d: block_n %d leaves <2 pipeline stages per consumer",
                 p.block_n);
  stages = p.team_stages * kConsumers;
  p.num_stages = stages;
  const int smem_bytes = 1024 + stages * stage_bytes + fixed;

  Maps maps;
  int rc;
  const __half* x = reinterpret_cast<const __half*>(in);
  if (stride == 1) {
    if ((rc = make_map4(&maps.a[0], x, cin, w, h, n, p.block_k, TW, TH))) return rc;
    for (int i = 1; i < 4; ++i) maps.a[i] = maps.a[0];
  } else {
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        // sub-image rows py, py+2, ... and columns px, px+2, ...; a 1-wide image has no odd column:
        // give that map one column so that the encoder accepts it (the producer never reads it:
        // no_odd_col / no_odd_row move those boxes out of bounds)
        const int sh = (h - py + 1) / 2, sw = (w - px + 1) / 2;
        if ((rc = make_map4_strided(&maps.a[py * 2 + px], x + (static_cast<size_t>(py) * w + px) * cin,
                                    cin, sw > 0 ? sw : 1, sh > 0 ? sh : 1, n,
                                    2ull * cin, 2ull * w * cin, static_cast<uint64_t>(h) * w * cin,
                                    p.block_k, TW, TH)))
          return rc;
      }
  }
  if ((rc = make_map(&maps.w, wt, cin, cout, p.taps, cin, static_cast<uint64_t>(cout) * cin,
                     p.block_n, p.block_k)))
    return rc;
  if ((rc = make_map4(&maps.o, out, cout, p.wo, p.ho, n, kStoreCols, TW, TH))) return rc;

  const int grid = persistent_grid(p.total_tiles, 1);
  if (!grid) return EDET_ERR_CUDA;
  const bool has_res = residual != nullptr;
  cudaStream_t s = as_stream(stream);
#define EDET_CONV_CASE(A)                                                \
  return has_res ? launch<A, true>(maps, p, grid, smem_bytes, s)         \
                 : launch<A, false>(maps, p, grid, smem_bytes, s)
  switch (act) {
    case EDET_ACT_NONE: EDET_CONV_CASE(EDET_ACT_NONE);
    case EDET_ACT_SWISH: EDET_CONV_CASE(EDET_ACT_SWISH);
    case EDET_ACT_RELU6: EDET_CONV_CASE(EDET_ACT_RELU6);
    default:
      set_error("conv2d: unsupported activation %d", act);
      return EDET_ERR_UNSUPPORTED;
  }
#undef EDET_CONV_CASE
}
