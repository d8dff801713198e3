// Conv2DTranspose 3 x 3, stride 2, 'SAME' (NHWC fp16) as a sub-pixel implicit GEMM on the Hopper
// tensor cores (wgmma): the upsampling stages of the EfficientDet segmentation head
// (tf2/efficientdet_keras.py:676-706, SegmentationHead).
//
// TF's conv2d_transpose with 'SAME' padding is the adjoint of the k3 s2 'SAME' conv2d, whose extra
// padding cell lies after the data, so per axis  out[y] = sum_i x[i] * w[y - 2i]  for
// y - 2i in {0, 1, 2}, output size 2H.  Split by output parity: an even row 2a takes ky = 0 from row
// a and ky = 2 from row a - 1, an odd row 2a + 1 takes ky = 1 from row a (columns alike).  So
// output pixel (2a + py, 2b + px) is a 2 x 2 stride-1 convolution of the input at (a, b), window
// rows {a - 1, a} x columns {b - 1, b} (tap (ty, tx), top / left padding 1), with phase
// (py, px)'s own weights:
//
//   out[n, 2a+py, 2b+px, co] = act( sum_{(ty,tx) in taps(py,px), c} x[n, a-1+ty, b-1+tx, c]
//                                   * W[ty*2+tx][(py*2+px)*C8 + co][c] + bias[co] )
//
// taps(py, px): ty in {0, 1} for py = 0, {1} for py = 1 (tx alike), i.e. 9 (tap, phase) pairs of
// 16; W holds zeros for the other 7, and the kernel never reads them.  ky = 1 for py = 1, else
// 2 for ty = 0 and 0 for ty = 1 (kx alike).  No zero-inserted or im2col tensor exists.
//
// K has one or two sources: channels [0, c0) from a0 and [c0, c0 + c1) from a1 (the previous
// stage's output and the BiFPN level of the reference's concat, which is never written).  Each
// source has a 4-D TMA map of its own (pixel stride lda_s); a box past the source's channels or
// the image is zero-filled by TMA, which gives both the top / left padding and the zero K padding
// up to the k-block.  W columns [woff_s, woff_s + c_s) belong to source s (woff_1 = round8(c0)).
//
// Structure of conv_tc.cu: persistent, warp-specialised (one TMA producer warp, two consumer
// warpgroups taking tiles in turn, each with a stage ring of its own), W streamed with A.  The M
// tile is a 4 x 16 block of input-grid positions, the N tile up to 128 channels of ONE phase, so
// a tile runs only its phase's taps.  The epilogue adds the bias and applies the activation in
// fp32, rounds to fp16 into a swizzled smem slab, and TMA-stores it through the phase's strided
// view of the output (rows 2a + py, columns 2b + px): the depth-to-space is the store's
// addressing.  The views are C8 = round8(cout) channels wide, so columns >= C8 (up to ld) and
// pixels outside the image are never written; columns cout..C8 are written as zero.
// Every output sums its products in a fixed order (taps, then sources, then k), whatever the grid.
// Algorithmic HBM bytes per launch: 2*N*H*W*(c0 + c1) + 2*N*4*H*W*C8 + 2*W bytes.
#include "tc_common.cuh"

namespace edet {
namespace convttc {

using namespace pwtc;   // PTX wrappers and tensor-map encoders of tc_common.cuh

constexpr int TH = 4, TW = 16;   // input-grid tile = the 64 rows of one wgmma
constexpr int BLOCK_M = TH * TW;
constexpr int kConsumers = 2;
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kMaxBlockN = 128;
constexpr int kStoreCols = 64;
constexpr int kSlabBytes = BLOCK_M * kStoreCols * 2;   // [64 px][64 cols] fp16, 128B swizzle
constexpr int kSlabsPerTeam = kMaxBlockN / kStoreCols;
constexpr int kMaxStages = 8;
constexpr int kSmemLimit = 227 * 1024;                 // one CTA per SM

struct Maps {
  CUtensorMap a[2];   // the K sources
  CUtensorMap w;      // weights [4 taps][4 * C8][kw]
  CUtensorMap o[4];   // output seen as the phase (py, px) sub-image [n][h][w][C8]
};

struct Params {
  int h, w, cout, c8;
  int nsrc, nkb0, nkb1, woff1;   // k-blocks of each source; W column of source 1
  int c0, c1;
  int tiles_x, tiles_y, n_per_phase, num_n_blocks, total_tiles;
  int block_n, block_k, num_stages, team_stages;
  int a_stage_bytes, b_stage_bytes;
  int desc_sbo, desc_layout;
  const float* bias;
};

struct TileCoord {
  int b, ty, tx, py, px, nb;
};
__device__ __forceinline__ TileCoord decode_tile(int t, const Params& p) {
  TileCoord c;
  const int n_blk = t % p.num_n_blocks;   // N fastest: the phases of one M tile share its A in L2
  t /= p.num_n_blocks;
  const int ph = n_blk / p.n_per_phase;
  c.nb = n_blk - ph * p.n_per_phase;
  c.py = ph >> 1;
  c.px = ph & 1;
  c.tx = t % p.tiles_x;
  t /= p.tiles_x;
  c.ty = t % p.tiles_y;
  c.b = t / p.tiles_y;
  return c;
}
// k-iterations of a tile: its phase's taps x (source 0's k-blocks, then source 1's)
__device__ __forceinline__ int tile_iters(const TileCoord& c, const Params& p) {
  return (2 - c.py) * (2 - c.px) * (p.nkb0 + p.nkb1);
}
struct KStep {
  int ty, tx, src, kb;
};
__device__ __forceinline__ KStep decode_k(int kk, const TileCoord& c, const Params& p) {
  const int per_tap = p.nkb0 + p.nkb1;
  const int tap = kk / per_tap, rem = kk - tap * per_tap;
  const int ntx = 2 - c.px;
  KStep s;
  s.ty = c.py + tap / ntx;
  s.tx = c.px + tap % ntx;
  s.src = rem >= p.nkb0 ? 1 : 0;
  s.kb = rem - s.src * p.nkb0;
  return s;
}

template <int ACT, int NT>
__global__ void __launch_bounds__(kThreads, 1)
convt_tc_kernel(const __grid_constant__ Maps maps, const Params p) {
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

  // Broadcast from lane 0: a role ptxas cannot prove warp-uniform puts every wgmma on a divergent
  // path, and ptxas then serialises them (C7520).
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 4);       // one arrive per warp of the consumer
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait_prior();          // everything above overlapped the previous kernel's tail

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage_of[kConsumers] = {}, phase_of[kConsumers] = {};   // per consumer ring
      const uint32_t tx_bytes = static_cast<uint32_t>(p.a_stage_bytes + p.block_n * p.block_k * 2);
      int iter = 0;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++iter) {
        const TileCoord tc = decode_tile(t, p);
        const int team = iter % kConsumers;
        int stage = stage_of[team];
        uint32_t phase = static_cast<uint32_t>(phase_of[team]);
        const int iters = tile_iters(tc, p);
        const int wrow = (tc.py * 2 + tc.px) * p.c8 + tc.nb * p.block_n;
        for (int kk = 0; kk < iters; ++kk) {
          const KStep ks = decode_k(kk, tc, p);
          const int s = team * p.team_stages + stage;
          mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
          const uint32_t fb = smem_u32(&full_bar[s]);
          mbar_expect_tx(fb, tx_bytes);
          uint8_t* sa = smem + s * stage_bytes;
          // window rows a - 1 + ty, columns b - 1 + tx (row / column -1 is TMA's zero fill)
          tma_load_4d(smem_u32(sa), &maps.a[ks.src], fb, ks.kb * p.block_k, tc.tx * TW - 1 + ks.tx,
                      tc.ty * TH - 1 + ks.ty, tc.b);
          tma_load_3d(smem_u32(sa + p.a_stage_bytes), &maps.w, fb,
                      ks.src * p.woff1 + ks.kb * p.block_k, wrow, ks.ty * 2 + ks.tx);
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
    const int r0 = 16 * (warp & 3) + (lane >> 2);   // tile rows (positions) r0 and r0 + 8
    const int cq = 2 * (lane & 3);
    uint8_t* my_slabs = smem_store + team * kSlabsPerTeam * kSlabBytes;
    int stage = 0;
    uint32_t phase = 0;
    int iter = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++iter) {
      if (iter % kConsumers != team) continue;   // the other consumer's tile (and ring)
      const TileCoord tc = decode_tile(t, p);
      const int iters = tile_iters(tc, p);
      float acc[NT][8];
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[j][q] = 0.f;
      for (int kk = 0; kk < iters; ++kk) {
        const KStep ks = decode_k(kk, tc, p);
        const int s = team * p.team_stages + stage;
        mbar_wait(smem_u32(&full_bar[s]), phase);
        uint8_t* sa = smem + s * stage_bytes;
        const uint64_t da = make_smem_desc(smem_u32(sa), p.desc_sbo, p.desc_layout);
        const uint64_t db = make_smem_desc(smem_u32(sa + p.a_stage_bytes), p.desc_sbo, p.desc_layout);
        const int k_rem = (ks.src ? p.c1 : p.c0) - ks.kb * p.block_k;
        const int ksteps = k_rem >= p.block_k ? p.block_k / MMA_K : (k_rem + MMA_K - 1) / MMA_K;
        wg_fence();
        wg_mma_kblock_wide<NT>(acc, da, db, ksteps, kk == 0);
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));
        if (++stage == p.team_stages) { stage = 0; phase ^= 1; }
      }
      wg_fence_acc<NT>(acc);
      const int n0 = tc.nb * p.block_n;   // first output channel of the tile within its phase
      if (wtid == 0) tma_store_wait_read<0>();
      named_sync(1 + team, 128);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const int colt = 16 * j + cq;
        float b[4];
        bool live[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {     // columns colt, colt + 1, colt + 8, colt + 9
          const int col = n0 + colt + (e >> 1) * 8 + (e & 1);
          live[e] = col < p.cout;
          b[e] = live[e] ? __ldg(p.bias + col) : 0.f;
        }
        uint8_t* slab = my_slabs + (colt >> 6) * kSlabBytes;
        const int piece = (colt & 63) >> 3;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float2 lo = fadd2_rn(make_float2(acc[j][2 * r], acc[j][2 * r + 1]), make_float2(b[0], b[1]));
          float2 hi = fadd2_rn(make_float2(acc[j][4 + 2 * r], acc[j][4 + 2 * r + 1]), make_float2(b[2], b[3]));
          apply_act4<ACT>(lo, hi);
          // channels cout .. C8 of the output are zero
          if (!live[0]) lo.x = 0.f;
          if (!live[1]) lo.y = 0.f;
          if (!live[2]) hi.x = 0.f;
          if (!live[3]) hi.y = 0.f;
          const int row = r0 + 8 * r;
          uint8_t* rb = slab + row * 128 + cq * 2;
          *reinterpret_cast<__half2*>(rb + ((piece ^ (row & 7)) << 4)) = __floats2half2_rn(lo.x, lo.y);
          *reinterpret_cast<__half2*>(rb + (((piece + 1) ^ (row & 7)) << 4)) = __floats2half2_rn(hi.x, hi.y);
        }
      }
      fence_proxy_async_smem();
      named_sync(1 + team, 128);
      if (wtid == 0) {
        // one 4-D box {64, 16, 4, 1} per 64 columns into the phase's view; the view's bounds
        // (C8 channels, h x w positions) clip what lies outside
        const CUtensorMap* map_o = &maps.o[tc.py * 2 + tc.px];
        for (int c = 0; c * kStoreCols < p.block_n; ++c)
          tma_store_4d(map_o, smem_u32(my_slabs + c * kSlabBytes), n0 + c * kStoreCols, tc.tx * TW,
                       tc.ty * TH, tc.b);
        tma_store_commit();
      }
    }
    if (wtid == 0) tma_store_wait_all();
  }
}

template <int ACT, int NT>
static int launch(const Maps& maps, const Params& p, int grid, int smem_bytes, cudaStream_t stream) {
  auto kern = convt_tc_kernel<ACT, NT>;
  static int configured[kMaxDevices];
  if (int rc = ensure_dynamic_smem(kern, kSmemLimit, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), smem_bytes, stream, maps, p));
  return EDET_OK;
}

template <int ACT>
static int launch_nt(const Maps& maps, const Params& p, int grid, int smem_bytes, cudaStream_t s) {
  switch (p.block_n) {
    case 32: return launch<ACT, 2>(maps, p, grid, smem_bytes, s);
    case 64: return launch<ACT, 4>(maps, p, grid, smem_bytes, s);
    case 96: return launch<ACT, 6>(maps, p, grid, smem_bytes, s);
    default: return launch<ACT, 8>(maps, p, grid, smem_bytes, s);
  }
}

static int round_up(int x, int m) { return (x + m - 1) / m * m; }

}  // namespace convttc
}  // namespace edet

extern "C" int edet_conv2d_transpose(const edet_half* a0, int c0, int lda0, const edet_half* a1,
                                     int c1, int lda1, const edet_half* wt, const float* bias,
                                     int act, edet_half* out, int ldo, int n, int h, int w,
                                     int cout, edet_stream_t stream) {
  using namespace edet;
  using namespace edet::convttc;
  EDET_CHECK_ARG(a0 && wt && bias && out, "conv2d_transpose: null pointer");
  EDET_CHECK_ARG(n > 0 && h > 0 && w > 0 && cout > 0, "conv2d_transpose: empty shape");
  EDET_CHECK_ARG(c0 > 0 && lda0 >= c0 && lda0 % 8 == 0,
                 "conv2d_transpose: source 0 needs 0 < c0 <= lda0, lda0 %% 8 == 0 (got %d, %d)", c0, lda0);
  EDET_CHECK_ARG(a1 == nullptr || (c1 > 0 && lda1 >= c1 && lda1 % 8 == 0),
                 "conv2d_transpose: source 1 needs 0 < c1 <= lda1, lda1 %% 8 == 0 (got %d, %d)", c1, lda1);
  const int c8 = round_up(cout, 8);
  EDET_CHECK_ARG(ldo >= c8 && ldo % 8 == 0,
                 "conv2d_transpose: ldo must be >= round8(cout) and a multiple of 8 (got %d)", ldo);
  Params p;
  p.h = h; p.w = w; p.cout = cout; p.c8 = c8;
  p.nsrc = a1 ? 2 : 1;
  p.c0 = c0; p.c1 = a1 ? c1 : 0;
  // k-block: the one that pads the sources' K least (the larger on a tie)
  int best = 0;
  for (int bk : {64, 32, 16}) {
    const int padded = round_up(p.c0, bk) + (p.c1 ? round_up(p.c1, bk) : 0);
    if (best == 0 || padded < best) { best = padded; p.block_k = bk; }
  }
  p.nkb0 = ceil_div(p.c0, p.block_k);
  p.nkb1 = p.c1 ? ceil_div(p.c1, p.block_k) : 0;
  p.woff1 = round_up(c0, 8);
  const int kw = p.woff1 + round_up(p.c1, 8);   // W row length
  // N tile: the phase's C8 channels rounded to a wgmma width of 32 / 64 / 96 / 128, else tiles of 128
  p.block_n = c8 <= kMaxBlockN ? round_up(c8, 32) : kMaxBlockN;
  p.n_per_phase = ceil_div(c8, p.block_n);
  p.num_n_blocks = 4 * p.n_per_phase;
  p.tiles_x = ceil_div(w, TW); p.tiles_y = ceil_div(h, TH);
  const long long tiles = static_cast<long long>(n) * p.tiles_x * p.tiles_y * p.num_n_blocks;
  EDET_CHECK_ARG(tiles < (1ll << 31), "conv2d_transpose: too many tiles");
  p.total_tiles = static_cast<int>(tiles);
  p.desc_layout = desc_layout_for(p.block_k);
  p.desc_sbo = 8 * p.block_k * 2;
  p.a_stage_bytes = BLOCK_M * p.block_k * 2;
  p.b_stage_bytes = ((p.block_n * p.block_k * 2 + 1023) / 1024) * 1024;
  p.bias = bias;
  const int stage_bytes = p.a_stage_bytes + p.b_stage_bytes;
  const int fixed = kConsumers * kSlabsPerTeam * kSlabBytes + 2 * kMaxStages * 8;
  int stages = (kSmemLimit - 1024 - fixed) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.team_stages = stages / kConsumers;       // each consumer's own ring
  EDET_CHECK_ARG(p.team_stages >= 2, "conv2d_transpose: block_n %d leaves <2 pipeline stages per consumer",
                 p.block_n);
  p.num_stages = p.team_stages * kConsumers;
  const int smem_bytes = 1024 + p.num_stages * stage_bytes + fixed;

  Maps maps;
  int rc;
  if ((rc = make_map4_strided(&maps.a[0], a0, c0, w, h, n, lda0, static_cast<uint64_t>(w) * lda0,
                              static_cast<uint64_t>(h) * w * lda0, p.block_k, TW, TH)))
    return rc;
  if (a1) {
    if ((rc = make_map4_strided(&maps.a[1], a1, c1, w, h, n, lda1, static_cast<uint64_t>(w) * lda1,
                                static_cast<uint64_t>(h) * w * lda1, p.block_k, TW, TH)))
      return rc;
  } else {
    maps.a[1] = maps.a[0];   // never addressed
  }
  if ((rc = make_map(&maps.w, wt, kw, 4 * c8, 4, kw, static_cast<uint64_t>(4) * c8 * kw, p.block_n,
                     p.block_k)))
    return rc;
  const __half* o = reinterpret_cast<const __half*>(out);
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px)
      if ((rc = make_map4_strided(&maps.o[py * 2 + px], o + (static_cast<size_t>(py) * 2 * w + px) * ldo,
                                  c8, w, h, n, 2ull * ldo, 4ull * w * ldo,
                                  4ull * h * w * ldo, kStoreCols, TW, TH)))
        return rc;

  const int grid = persistent_grid(p.total_tiles, 1);
  if (!grid) return EDET_ERR_CUDA;
  cudaStream_t s = as_stream(stream);
  switch (act) {
    case EDET_ACT_NONE: return launch_nt<EDET_ACT_NONE>(maps, p, grid, smem_bytes, s);
    case EDET_ACT_SWISH: return launch_nt<EDET_ACT_SWISH>(maps, p, grid, smem_bytes, s);
    case EDET_ACT_RELU6: return launch_nt<EDET_ACT_RELU6>(maps, p, grid, smem_bytes, s);
    default:
      set_error("conv2d_transpose: unsupported activation %d", act);
      return EDET_ERR_UNSUPPORTED;
  }
}
