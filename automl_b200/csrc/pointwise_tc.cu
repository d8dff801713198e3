// Pointwise (1x1) convolution as an NHWC GEMM on the Hopper tensor cores (wgmma, sm_90a).
//
//   out[b, r, n] = act( sum_k A[b, r, k] * Wt[b|0, n, k] + bias[n] ) (+ residual[b, r, n])
//
// Structure (persistent CTAs, one per SM, warp-specialised):
//   warpgroup 0        : warp 0 / lane 0 is the TMA producer -- cp.async.bulk.tensor (3-D maps,
//                        128B / 64B / 32B swizzle) of the A tile [64 x block_k] and the W tile
//                        [block_n x block_k] into the smem stage ring of the consumer that owns
//                        the tile (mbarrier complete_tx).  Each consumer has a ring of its own, so
//                        it sees every phase of its stage barriers (a consumer that skipped the
//                        other's stages could meet a barrier two phases behind, whose parity looks
//                        complete).  Out-of-bounds rows / K tail are zero-filled by TMA.
//   warpgroups 1..TEAMS: consumers.  Tile i of the CTA belongs to consumer i % TEAMS, which runs
//                        the wgmma main loop (m64 x n16 x k16, fp32 accumulators in registers) and
//                        then its own epilogue: +bias -> activation -> (+residual) -> fp16 ->
//                        128B-swizzled staging slab -> TMA store (clips the ragged M / N edges).
//                        While one consumer is in its MUFU-bound epilogue the other one's MMAs run.
//
// Replaces Conv2D 1x1 (+BN, +swish, +skip) at the reference call sites listed in
// include/automl_b200.h (edet_pointwise_conv).  Algorithmic HBM bytes per launch:
//   2*(batch*rows*k + batch*rows*nout [+ same for residual]) + 2*wbatch*nout*k   (SURVEY 8d).
#include <math_constants.h>

#include "tc_common.cuh"

namespace edet {
namespace pwtc {

constexpr int BLOCK_M = 64;         // rows per tile = the M of one wgmma
constexpr int kMaxBlockN = 128;     // accumulator columns per consumer thread: kMaxBlockN / 2
constexpr int kNT = kMaxBlockN / 16;
template <int TEAMS>
struct Epi {
  static constexpr int kThreads = 128 * (1 + TEAMS);
};
constexpr int kStoreCols = 64;
constexpr int kSlabBytes = BLOCK_M * kStoreCols * 2;   // [64 rows][64 cols] fp16, 128B swizzle
constexpr int kSlabsPerTeam = kMaxBlockN / kStoreCols;
constexpr int kMaxStages = 9;   // 4 + 4 (two consumers) or 3 + 3 + 3
constexpr int kRing = 4;          // tile-index ring entries (power of two)
constexpr int kSmemLimit = 227 * 1024;                   // one CTA per SM

struct Params {
  int batch, rows, k, nout, nout_pad8;
  int block_n, num_m_blocks, num_n_blocks, num_k_blocks, num_stages;
  int team_stages;    // stages of each consumer's own ring: num_stages / TEAMS
  int block_k;        // 64 / 32 / 16 halves per k-block == 128B / 64B / 32B swizzled smem rows
  int a_stage_bytes, b_stage_bytes;
  int desc_sbo;       // byte distance between 8-row groups in smem (8 * row pitch)
  int desc_layout;    // wgmma layout type: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B
  int wbatch, ldr;
  int total_tiles;
  int bias_floats;    // floats of the zero-padded bias staged in shared memory: whole N tiles
  const float* bias;
  const __half* residual;
  unsigned* sched;    // dynamic tile scheduler slot (tc_common.cuh)
  // EPI_ARGMAX (class head -> pre-NMS): N tile n_blk = anchor n_blk, rows = pixels of one level
  float* am_scores;       // [batch][am_total] sigmoid of the best class logit
  int32_t* am_classes;    // [batch][am_total] its class index
  int am_anchor_begin, am_total, am_num_anchors;
};
constexpr int EPI_STORE = 0, EPI_ARGMAX = 1;
constexpr int kArgmaxCols = 96;   // columns per anchor in the padded class-head weights

struct TileCoord {
  int b, m_blk, n_blk;
};
constexpr int kMaxBiasSmem = 8192;

__device__ __forceinline__ TileCoord decode_tile(int t, const Params& p) {
  TileCoord c;
  c.n_blk = 0;
  if (p.num_n_blocks != 1) {       // (uniform) most layers are one N tile wide ...
    c.n_blk = t % p.num_n_blocks;
    t /= p.num_n_blocks;
  }
  c.m_blk = t;
  c.b = 0;
  if (p.batch != 1) {              // ... and one batch entry long: no division at all
    c.m_blk = t % p.num_m_blocks;
    c.b = t / p.num_m_blocks;
  }
  return c;
}

// Running arg-max key of a pair of adjacent logits (columns col, col + 1): each logit is rounded
// to fp16 exactly as the storing epilogue would store it and mapped to an order-preserving uint16,
// << 16 | (0xFFFF - column), so that one unsigned max gives the maximum AND its first column
// (equal logits: the lower column has the larger key).  -0 is canonicalised to +0 first (the
// float compare of the stored-logits path treats them as equal).
__device__ __forceinline__ uint32_t argmax_pair_key(float2 s, uint32_t col) {
  const __half2 h = __hadd2(__floats2half2_rn(s.x, s.y), __float2half2_rn(0.f));
  const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h);
  uint32_t sgn;      // 0xFFFF in the halves that are negative
  asm("prmt.b32 %0, %1, %2, 0xBB99;" : "=r"(sgn) : "r"(hb), "r"(0u));
  const uint32_t ord = hb ^ (sgn | 0x80008000u);       // order-preserving uint16 x 2
  const uint32_t codes = ((0xFFFFu - (col + 1u)) << 16) | (0xFFFFu - col);
  uint32_t k0, k1;
  asm("prmt.b32 %0, %1, %2, 0x1054;" : "=r"(k0) : "r"(ord), "r"(codes));
  asm("prmt.b32 %0, %1, %2, 0x3276;" : "=r"(k1) : "r"(ord), "r"(codes));
  return max(k0, k1);
}

template <int ACT, bool HAS_RES, int TEAMS, int EPI>
__global__ void __launch_bounds__(Epi<TEAMS>::kThreads, 1)
pointwise_tc_kernel(const __grid_constant__ CUtensorMap map_a,
                    const __grid_constant__ CUtensorMap map_w,
                    const __grid_constant__ CUtensorMap map_o, const Params p) {
  pdl_launch_dependents();   // the next kernel may start its prologue while this one runs
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for the swizzle atoms.
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = p.a_stage_bytes + p.b_stage_bytes;
  uint8_t* smem_store = smem + p.num_stages * stage_bytes;   // [TEAMS][kSlabsPerTeam] slabs
  float* smem_bias = reinterpret_cast<float*>(smem_store + TEAMS * kSlabsPerTeam * kSlabBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_bias + p.bias_floats);
  uint64_t* full_bar = bars;                       // [kMaxStages]
  uint64_t* empty_bar = bars + kMaxStages;         // [kMaxStages]
  // Tile indices travel from the producer to the consumers through a small ring: CTA i owns tile
  // i, every further tile comes from a global counter (sched_next_tile), so a CTA that gets its
  // SM late -- another stream's kernel, e.g. the NMS of the previous batch, was holding it --
  // simply finds less work instead of owning a full static share.
  uint64_t* ring_full = bars + 2 * kMaxStages;     // [kRing] producer -> consumers
  uint64_t* ring_empty = ring_full + kRing;        // [kRing] consumers -> producer
  // [kRing] x {tile, batch entry, M block, N block}: the producer decodes each tile once (its two
  // integer divisions) and the consumers read the coordinates with one 16-byte load
  volatile int4* tile_ring = reinterpret_cast<volatile int4*>(ring_empty + kRing);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 4);       // one arrive per warp of the consumer
    }
    for (int s = 0; s < kRing; ++s) {
      mbar_init(smem_u32(&ring_full[s]), 1);
      mbar_init(smem_u32(&ring_empty[s]), TEAMS);  // one arrive per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_o)) : "memory");
  }
  // bias (a constant, like the weights: read before the PDL wait) -> shared memory, zero padded
  for (int i = threadIdx.x; i < p.bias_floats; i += blockDim.x)
    smem_bias[i] = i < p.nout ? __ldg(p.bias + i) : 0.f;
  __syncthreads();
  pdl_wait_prior();          // everything above overlapped the previous kernel's tail

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage_of[TEAMS] = {}, phase_of[TEAMS] = {};   // per consumer ring
      // bytes the two TMA boxes deliver (the B slot may be padded to 1 KiB)
      const uint32_t tx_bytes = static_cast<uint32_t>(p.a_stage_bytes + p.block_n * p.block_k * 2);
      bool exhausted = false;
      for (int i = 0;; ++i) {
        int t = p.total_tiles;
        if (i == 0) {
          t = blockIdx.x;
        } else if (!exhausted) {
          t = sched_next_tile(p.sched, p.total_tiles);
          exhausted = t >= p.total_tiles;
        }
        const int slot = i & (kRing - 1);
        mbar_wait(smem_u32(&ring_empty[slot]), (static_cast<uint32_t>(i / kRing) & 1u) ^ 1u);
        TileCoord tc;
        tc.b = tc.m_blk = tc.n_blk = 0;
        if (t < p.total_tiles) tc = decode_tile(t, p);
        const_cast<int4*>(tile_ring)[slot] = make_int4(t, tc.b, tc.m_blk, tc.n_blk);
        mbar_arrive(smem_u32(&ring_full[slot]));     // release: the entry is visible to waiters
        if (t >= p.total_tiles) break;
        const int wb = (p.wbatch > 1) ? tc.b : 0;
        const int team = i % TEAMS;
        int stage = stage_of[team];
        uint32_t phase = static_cast<uint32_t>(phase_of[team]);
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          const int s = team * p.team_stages + stage;
          mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
          const uint32_t fb = smem_u32(&full_bar[s]);
          mbar_expect_tx(fb, tx_bytes);
          uint8_t* sa = smem + s * stage_bytes;
          tma_load_3d(smem_u32(sa), &map_a, fb, kb * p.block_k, tc.m_blk * BLOCK_M, tc.b);
          tma_load_3d(smem_u32(sa + p.a_stage_bytes), &map_w, fb, kb * p.block_k,
                      tc.n_blk * p.block_n, wb);
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
    const int r0 = 16 * (warp & 3) + (lane >> 2);   // rows r0 and r0 + 8 of the tile
    const int cq = 2 * (lane & 3);                  // column pair inside each 8-column group
    uint8_t* my_slabs = smem_store + team * kSlabsPerTeam * kSlabBytes;
    const int b_chunk = p.block_k * 2;              // descriptor units between 16-row B chunks
    int stage = 0;            // in this consumer's ring: stages team * team_stages ..
    uint32_t phase = 0;
    auto advance = [&]() {
      if (++stage == p.team_stages) {
        stage = 0;
        phase ^= 1;
      }
    };
    for (int iter = 0;; ++iter) {
      const int slot = iter & (kRing - 1);
      mbar_wait(smem_u32(&ring_full[slot]), static_cast<uint32_t>(iter / kRing) & 1u);
      const int4 e = const_cast<const int4*>(tile_ring)[slot];
      named_sync(1 + team, 128);
      if (wtid == 0) mbar_arrive(smem_u32(&ring_empty[slot]));
      const int t = e.x;
      if (t >= p.total_tiles) break;
      if (iter % TEAMS != team) continue;   // another consumer's tile (and ring)
      TileCoord tc;
      tc.b = e.y;
      tc.m_blk = e.z;
      tc.n_blk = e.w;
      const int n0 = tc.n_blk * p.block_n;
      // only the columns that exist in the output are worth MMAs and an epilogue (rounded up to
      // the 16-column MMA granule); the rest of a ragged last N tile is skipped
      const int n_valid = min(p.block_n, ((p.nout - n0 + 15) >> 4) << 4);
      const int nt = n_valid >> 4;
      float acc[kNT][8];
#pragma unroll
      for (int j = 0; j < kNT; ++j)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[j][q] = 0.f;
      for (int kb = 0; kb < p.num_k_blocks; ++kb) {
        const int s = team * p.team_stages + stage;
        mbar_wait(smem_u32(&full_bar[s]), phase);
        uint8_t* sa = smem + s * stage_bytes;
        const uint64_t da = make_smem_desc(smem_u32(sa), p.desc_sbo, p.desc_layout);
        const uint64_t db = make_smem_desc(smem_u32(sa + p.a_stage_bytes), p.desc_sbo, p.desc_layout);
        const int k_rem = p.k - kb * p.block_k;
        const int ksteps = k_rem >= p.block_k ? p.block_k / MMA_K : (k_rem + MMA_K - 1) / MMA_K;
        wg_fence();
        wg_mma_kblock<kNT>(acc, da, db, b_chunk, nt, ksteps, kb == 0);
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));   // this warp is done with it
        advance();
      }
      wg_fence_acc<kNT>(acc);
      const int row0 = tc.m_blk * BLOCK_M + r0;
      if constexpr (EPI == EPI_ARGMAX) {
        // Class head fused with the class half of pre-NMS (tf2/postprocess.py:88-156 with
        // max_nms_inputs == 0): an N tile is ONE anchor (90 class columns + 6 pad columns whose
        // bias is -inf).  Each logit is rounded to fp16 exactly as the storing epilogue would
        // store it, then max / first arg-max / sigmoid as pre_nms_kernel does -> bit-identical
        // scores and classes, without the [N, H, W, 810] logits ever reaching HBM.
        const float* bias = smem_bias + tc.n_blk * kArgmaxCols;
        uint32_t best[2] = {0u, 0u};                  // rows r0, r0 + 8
#pragma unroll
        for (int j = 0; j < kArgmaxCols / 16; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int col = 16 * j + 8 * h + cq;
            const float2 b = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const float2 s = fadd2_rn(make_float2(acc[j][4 * h + 2 * r], acc[j][4 * h + 2 * r + 1]), b);
              best[r] = max(best[r], argmax_pair_key(s, static_cast<uint32_t>(col)));
            }
          }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {      // the four lanes of a quad hold the same row
          best[r] = max(best[r], __shfl_xor_sync(0xffffffffu, best[r], 1));
          best[r] = max(best[r], __shfl_xor_sync(0xffffffffu, best[r], 2));
          const uint32_t ord_best = best[r] >> 16;
          const unsigned short hbits = static_cast<unsigned short>(
              (ord_best & 0x8000u) ? (ord_best ^ 0x8000u) : (~ord_best & 0xFFFFu));
          const float bv = __half2float(__ushort_as_half(hbits));
          const int best_c = static_cast<int>(0xFFFFu - (best[r] & 0xFFFFu));
          const int row = row0 + 8 * r;
          if ((lane & 3) == 0 && row < p.rows) {
            const size_t o = static_cast<size_t>(tc.b) * p.am_total + p.am_anchor_begin +
                             static_cast<size_t>(row) * p.am_num_anchors + tc.n_blk;
            p.am_scores[o] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-bv)));
            p.am_classes[o] = best_c;
          }
        }
      } else {
        const bool ok[2] = {row0 < p.rows, row0 + 8 < p.rows};
        const __half* res_row[2] = {nullptr, nullptr};
        if (HAS_RES) {
#pragma unroll
          for (int r = 0; r < 2; ++r)
            res_row[r] = p.residual +
                         (static_cast<size_t>(tc.b) * p.rows + (ok[r] ? row0 + 8 * r : 0)) * p.ldr;
        }
        // the slabs are free once this consumer's previous stores have read them
        if (wtid == 0) tma_store_wait_read<0>();
        named_sync(1 + team, 128);
#pragma unroll
        for (int j = 0; j < kNT; ++j) {
          if (j < nt) {
            const int colt = 16 * j + cq;            // tile column of acc[j][0]
            const float2 b_lo = *reinterpret_cast<const float2*>(smem_bias + n0 + colt);
            const float2 b_hi = *reinterpret_cast<const float2*>(smem_bias + n0 + colt + 8);
            uint8_t* slab = my_slabs + (colt >> 6) * kSlabBytes;
            const int piece = (colt & 63) >> 3;      // 16-byte piece of the 128-byte slab row
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              float2 lo = fadd2_rn(make_float2(acc[j][2 * r], acc[j][2 * r + 1]), b_lo);
              float2 hi = fadd2_rn(make_float2(acc[j][4 + 2 * r], acc[j][4 + 2 * r + 1]), b_hi);
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
          for (int c = 0; c * kStoreCols < n_valid; ++c)
            tma_store_3d(&map_o, smem_u32(my_slabs + c * kSlabBytes), n0 + c * kStoreCols,
                         tc.m_blk * BLOCK_M, tc.b);
          tma_store_commit();
        }
      }
    }
    if (wtid == 0) tma_store_wait_all();
  }
}

// N tile: the whole width up to kMaxBlockN (one tile, A read once); wider layers use tiles of
// 128 columns (a multiple of the 64-column store box, so that a tile's stores never reach into
// the next tile), the A tile of the extra tiles comes from L2.  The class-head arg-max epilogue
// needs one anchor (kArgmaxCols columns) per tile.
static int pick_block_n(int nout) {
  if (nout <= kMaxBlockN) return ((nout + 15) / 16) * 16;
  return kMaxBlockN;
}

template <int ACT, bool HAS_RES, int TEAMS, int EPI = EPI_STORE>
static int launch(const CUtensorMap& ma, const CUtensorMap& mw, const CUtensorMap& mo,
                  const Params& p, int grid, int smem_bytes, cudaStream_t stream) {
  auto kern = pointwise_tc_kernel<ACT, HAS_RES, TEAMS, EPI>;
  static int configured[kMaxDevices];   // per instantiation and device; no API call once set
  if (int rc = ensure_dynamic_smem(kern, kSmemLimit, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(Epi<TEAMS>::kThreads), smem_bytes, stream, ma,
                             mw, mo, p));
  return EDET_OK;
}

int run(const __half* a, int lda, const __half* wt, int wbatch, const float* bias,
        const __half* residual, int ldr, __half* out, int ldo, int batch, int rows, int k, int nout,
        int act, cudaStream_t stream, const ArgmaxArgs* am) {
  Params p;
  p.am_scores = nullptr; p.am_classes = nullptr;
  p.am_anchor_begin = p.am_total = p.am_num_anchors = 0;
  if (am) {
    EDET_CHECK_ARG(nout == am->num_anchors * kArgmaxCols && !residual && act == EDET_ACT_NONE,
                   "class_argmax: nout must be num_anchors * %d", kArgmaxCols);
    p.am_scores = am->scores; p.am_classes = am->classes;
    p.am_anchor_begin = am->anchor_begin; p.am_total = am->total_anchors;
    p.am_num_anchors = am->num_anchors;
  }
  p.batch = batch;
  p.rows = rows;
  p.k = k;
  p.nout = nout;
  p.nout_pad8 = nout & ~7;   // whole float4 pairs of bias that are in bounds
  // Consumer warpgroups: two by default (one in its epilogue while the other one's MMAs run);
  // edet_set_option("pw_teams", 2 | 3) forces a variant for A/B measurements.
  const int opt_teams = option_pw_teams();
  const int teams = opt_teams ? opt_teams : 2;
  p.block_n = am ? kArgmaxCols : pick_block_n(nout);
  p.num_m_blocks = ceil_div(rows, BLOCK_M);
  p.num_n_blocks = ceil_div(nout, p.block_n);
  p.wbatch = wbatch;
  p.ldr = ldr;
  p.bias = bias;
  p.residual = residual;
  p.total_tiles = batch * p.num_m_blocks * p.num_n_blocks;
  p.sched = next_sched_slot();
  if (!p.sched) return EDET_ERR_CUDA;

  // every column the epilogue can touch: whole N tiles (n_valid is rounded up to 16 inside a tile)
  const int bias_cols = p.num_n_blocks * p.block_n;
  EDET_CHECK_ARG(bias_cols <= kMaxBiasSmem, "pointwise_tc: nout %d too wide", nout);
  p.bias_floats = bias_cols;
  // k-block / smem row pitch: 16 halves (32B swizzle) for K <= 16, 32 (64B) for K <= 32, else 64
  // (128B), so that a stage only holds bytes that exist.
  p.block_k = k <= 16 ? 16 : (k <= 32 ? 32 : 64);
  p.a_stage_bytes = BLOCK_M * p.block_k * 2;
  p.b_stage_bytes = ((p.block_n * p.block_k * 2 + 1023) / 1024) * 1024;
  const int stage_bytes = p.a_stage_bytes + p.b_stage_bytes;
  const int fixed = teams * kSlabsPerTeam * kSlabBytes + p.bias_floats * 4 +
                    (2 * kMaxStages + 2 * kRing) * 8 + 16 * kRing;
  const int opt_kb = option_pw_smem_kb();
  const int limit = opt_kb ? opt_kb * 1024 : kSmemLimit;
  int stages = (limit - 1024 - fixed) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.team_stages = stages / teams;            // each consumer's own ring
  EDET_CHECK_ARG(p.team_stages >= 2, "pointwise_tc: block_n %d leaves <2 pipeline stages per consumer",
                 p.block_n);
  stages = p.team_stages * teams;
  p.num_stages = stages;
  p.desc_layout = desc_layout_for(p.block_k);
  p.desc_sbo = 8 * p.block_k * 2;
  p.num_k_blocks = ceil_div(k, p.block_k);
  const int smem_bytes = 1024 + stages * stage_bytes + fixed;

  CUtensorMap ma, mw, mo;
  int rc;
  if ((rc = make_map(&ma, a, k, rows, batch, lda, static_cast<uint64_t>(rows) * lda, BLOCK_M,
                     p.block_k)))
    return rc;
  if ((rc = make_map(&mw, wt, k, nout, wbatch, k, static_cast<uint64_t>(nout) * k, p.block_n,
                     p.block_k)))
    return rc;
  // store box: [64 rows] x 64 columns, 128B swizzle
  if (am) {
    mo = mw;   // the arg-max epilogue stores nothing through TMA
  } else if ((rc = make_map(&mo, out, nout, rows, batch, ldo, static_cast<uint64_t>(rows) * ldo,
                            BLOCK_M, kStoreCols))) {
    return rc;
  }

  const int sm_count = device_sm_count();
  if (!sm_count) return EDET_ERR_CUDA;
  int grid = sm_count - option_persist_slack();
  if (grid < 1) grid = 1;
  if (p.total_tiles < grid) grid = p.total_tiles;
  const bool has_res = residual != nullptr;
  if (am) return launch<EDET_ACT_NONE, false, 2, EPI_ARGMAX>(ma, mw, mo, p, grid, smem_bytes, stream);

#define EDET_PW_CASE(A)                                                                       \
  if (teams == 3)                                                                             \
    return has_res ? launch<A, true, 3>(ma, mw, mo, p, grid, smem_bytes, stream)              \
                   : launch<A, false, 3>(ma, mw, mo, p, grid, smem_bytes, stream);            \
  return has_res ? launch<A, true, 2>(ma, mw, mo, p, grid, smem_bytes, stream)                \
                 : launch<A, false, 2>(ma, mw, mo, p, grid, smem_bytes, stream)
  switch (act) {
    case EDET_ACT_NONE: EDET_PW_CASE(EDET_ACT_NONE);
    case EDET_ACT_SWISH: EDET_PW_CASE(EDET_ACT_SWISH);
    case EDET_ACT_RELU: EDET_PW_CASE(EDET_ACT_RELU);
    case EDET_ACT_RELU6: EDET_PW_CASE(EDET_ACT_RELU6);
    case EDET_ACT_HSWISH: EDET_PW_CASE(EDET_ACT_HSWISH);
    case EDET_ACT_SIGMOID: EDET_PW_CASE(EDET_ACT_SIGMOID);
    default:
      set_error("pointwise_tc: bad activation %d", act);
      return EDET_ERR_INVALID;
  }
#undef EDET_PW_CASE
}

}  // namespace pwtc
}  // namespace edet
