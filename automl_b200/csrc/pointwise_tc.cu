// Pointwise (1x1) convolution as an NHWC GEMM on the Hopper tensor cores (wgmma, sm_90a).
//
//   out[b, r, n] = act( sum_k A[b, r, k] * Wt[b|0, n, k] + bias[n] ) (+ residual[b, r, n])
//
// Structure (persistent CTAs, one per SM, warp-specialised):
//   warpgroup 0        : warp 0 / lane 0 is the TMA producer -- cp.async.bulk.tensor (3-D maps,
//                        128B / 64B / 32B swizzle) of the A tile [64 x block_k] and, unless all
//                        of W is resident in smem (kResidentWBytes), the W tile
//                        [block_n x block_k] into the smem stage ring of the consumer that owns
//                        the tile (mbarrier complete_tx).  Each consumer has a ring of its own, so
//                        it sees every phase of its stage barriers (a consumer that skipped the
//                        other's stages could meet a barrier two phases behind, whose parity looks
//                        complete).  Out-of-bounds rows / K tail are zero-filled by TMA.
//   warpgroups 1..TEAMS: consumers.  Work unit i of the CTA (up to 8 consecutive 64-row M blocks
//                        of one image, see Params) belongs to consumer i % TEAMS, which runs, per
//                        tile of the unit, the wgmma main loop (one m64 x block_n x k16 per
//                        k-step, fp32 accumulators in registers, one k-block of MMAs in flight)
//                        and then its own epilogue: +bias -> activation -> (+residual) -> fp16 ->
//                        128B-swizzled staging slab -> TMA store (clips the ragged M / N edges).
//                        A residual tile is loaded by TMA into that tile's staging slabs while its
//                        MMAs run, and the epilogue adds it in place: the element it reads is the
//                        one it overwrites, at the same swizzled address.
//                        While one consumer is in its MUFU-bound epilogue the other one's MMAs run.
//   shared-W plan (share_w, two consumers): where W streams, a tile is 128 rows (two consecutive
//                        64-row M blocks of one image) and a stage holds A [128 x block_k] plus ONE
//                        W tile, in a single ring that both consumers read: consumer c multiplies
//                        rows 64c .. 64c + 63 against the same W smem, so each streamed W tile
//                        leaves L2 once per 128 rows instead of once per 64.  Every unit belongs to
//                        both consumers, both wait on every "full" phase of the ring and each stage's
//                        "empty" barrier expects the arrivals of both, so neither can meet a phase it
//                        skipped.  Rows past the image are TMA zero fill, the stores clip them, and a
//                        consumer whose 64 rows all lie past the image stores nothing.
//
// Replaces Conv2D 1x1 (+BN, +swish, +skip) at the reference call sites listed in
// include/automl_b200.h (edet_pointwise_conv).  Algorithmic HBM bytes per launch:
//   2*(batch*rows*k + batch*rows*nout [+ same for residual]) + 2*wbatch*nout*k   (SURVEY 8d).
#include <math_constants.h>

#include <algorithm>
#include <climits>
#include <type_traits>

#include "tc_common.cuh"

namespace edet {
namespace pwtc {

constexpr int BLOCK_M = 64;         // rows per consumer and tile = the M of one wgmma
constexpr int kMaxBlockN = 128;     // accumulator columns per consumer thread: kMaxBlockN / 2
template <int TEAMS>
struct Epi {
  static constexpr int kThreads = 128 * (1 + TEAMS);
};
constexpr int kStoreCols = 64;
constexpr int kSlabBytes = BLOCK_M * kStoreCols * 2;   // [64 rows][64 cols] fp16, 128B swizzle
// Stages are sized from bytes: each consumer gets enough for kTeamInFlightBytes of loads (16
// stages of a thin-K 2 KB A tile, 4 of a 128B-swizzled 8 KB one), at least kMinTeamStages and the
// stages of one work unit, and no more than the shared memory left after W, slabs and bias holds.
// Not deeper: the producer claims units as far ahead as its stages reach, and units claimed early
// by one CTA cannot go to another, which on launches with few units per CTA undoes the dynamic
// schedule.
constexpr int kTeamInFlightBytes = 32 * 1024;
constexpr int kMinTeamStages = 4;
constexpr int kMaxStages = 3 * 16;   // mbarrier storage: three consumers of 16 stages
constexpr int kRing = 4;          // work-unit ring entries (power of two)
constexpr int kResBars = 2 * 3;   // residual-landed barriers: one per slab set of each consumer
constexpr int kSmemLimit = 227 * 1024;                   // one CTA per SM
// Weights of at most this many (padded, swizzled) bytes stay in shared memory for the life of the
// CTA: every D0 layer up to blocks_8, the BiFPN layers and both predict layers (the class head,
// 9 anchors x 96 x 64 halves, is exactly this size).  What is left still holds the staging slabs
// and at least two A stages per consumer.
constexpr int kResidentWBytes = 108 * 1024;
constexpr int kUnitsPerCta = 8;                  // work-unit size policy (run())
// Shared-W plan (run()): with a residual only from this many k-blocks.  Both consumers reach their
// epilogues together.  D0 batch 32 on H100, with the residual still read in the epilogue, measured
// blocks_6/7 project (K 480: 8 k-blocks) 3 us slower with the plan, blocks_9/10 project (11) level
// and blocks_12-14 project (18) 12 us faster.  Not measured again since the residual tile comes
// through TMA.
constexpr int kShareResMinKBlocks = 10;
constexpr int kMaxUnitBytes = 128 * 1024;

struct Params {
  int batch, rows, k, nout, nout_pad8;
  int block_n, num_m_blocks, num_n_blocks, num_k_blocks, num_stages;
  int tile_m;         // rows per tile (an "M block" below): BLOCK_M, or 2 * BLOCK_M with share_w
  int share_w;        // 1: both consumers work on every tile, one ring (TEAMS == 2 only)
  int team_stages;    // stages of each ring: num_stages / TEAMS, or num_stages with share_w
  int block_k;        // 64 / 32 / 16 halves per k-block == 128B / 64B / 32B swizzled smem rows
  int a_stage_bytes, b_stage_bytes;
  int stage_bytes;    // ring bytes per stage: A, plus the W tile unless W is resident
  int w_resident;     // 1: all of W (wbatch == 1) lives in smem, loaded once per CTA
  int slab_sets;      // staging-slab sets per consumer (2: a tile's stores overlap the next epilogue)
  int slab_set_bytes; // one set: ceil(block_n / 64) slabs of [64 rows][64 cols]
  int desc_sbo;       // byte distance between 8-row groups in smem (8 * row pitch)
  int desc_layout;    // wgmma layout type: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B
  int wbatch, ldr;
  // Work unit: unit_m consecutive M blocks of one image (the last unit of an image may be
  // shorter) x one N tile, or x every N tile when hold_a is set.  One tile-ring entry and one
  // scheduler claim cover the whole unit.
  int unit_m, units_per_image;
  int hold_a;         // 1: W resident, one k-block, several N tiles: A is loaded once per M block
  int total_units;
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
// Bias floats staged in shared memory: whole 128-column N tiles of the widest registered layer,
// the 8256-channel expand of efficientnet-l2 (65 tiles).  Narrower launches stage only their own.
constexpr int kMaxBiasSmem = 65 * kMaxBlockN;

// Work unit u -> batch entry, first M block, N tile (the first one when the unit holds A).
__device__ __forceinline__ TileCoord decode_unit(int u, const Params& p) {
  TileCoord c;
  c.n_blk = 0;
  if (p.num_n_blocks != 1 && !p.hold_a) {   // (uniform) most layers are one N tile wide ...
    c.n_blk = u % p.num_n_blocks;
    u /= p.num_n_blocks;
  }
  c.m_blk = u;
  c.b = 0;
  if (p.batch != 1) {              // ... and one batch entry long: no division at all
    c.m_blk = u % p.units_per_image;
    c.b = u / p.units_per_image;
  }
  c.m_blk *= p.unit_m;
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
                    const __grid_constant__ CUtensorMap map_o,
                    const __grid_constant__ CUtensorMap map_r, const Params p) {
  pdl_launch_dependents();   // the next kernel may start its prologue while this one runs
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for the swizzle atoms.
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = p.stage_bytes;
  // false at compile time for three consumers and the arg-max epilogue, which never share a ring
  const bool share = TEAMS == 2 && EPI == EPI_STORE && p.share_w;
  // resident W: [num_n_blocks][num_k_blocks] boxes of b_stage_bytes (empty unless w_resident)
  uint8_t* smem_w = smem + p.num_stages * stage_bytes;
  const int w_bytes = p.w_resident ? p.num_n_blocks * p.num_k_blocks * p.b_stage_bytes : 0;
  uint8_t* smem_store = smem_w + w_bytes;   // [TEAMS][slab_sets] slab sets
  float* smem_bias = reinterpret_cast<float*>(smem_store + TEAMS * p.slab_sets * p.slab_set_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_bias + p.bias_floats);
  uint64_t* full_bar = bars;                       // [kMaxStages]
  uint64_t* empty_bar = bars + kMaxStages;         // [kMaxStages]
  // Work-unit indices travel from the producer to the consumers through a small ring: CTA i owns
  // unit i, every further unit comes from a global counter (sched_claim), so a CTA that gets its
  // SM late -- another stream's kernel, e.g. the NMS of the previous batch, was holding it --
  // simply finds less work instead of owning a full static share.
  uint64_t* ring_full = bars + 2 * kMaxStages;     // [kRing] producer -> consumers
  uint64_t* ring_empty = ring_full + kRing;        // [kRing] consumers -> producer
  // [kRing] x {unit, batch entry, first M block, N block}: the producer decodes each unit once
  // (its two integer divisions) and the consumers read the coordinates with one 16-byte load
  uint64_t* w_full = ring_empty + kRing;          // [2]: [0] resident W landed, [1] padding
  uint64_t* res_bars = w_full + 2;                // [kResBars]: [team * 2 + slab set]
  volatile int4* tile_ring = reinterpret_cast<volatile int4*>(res_bars + kResBars);

  // warp-uniform as far as ptxas can tell (see the tile-ring broadcast below)
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), share ? 4 * TEAMS : 4);   // one arrive per warp of each
                                                                   // consumer reading the ring
    }
    for (int s = 0; s < kRing; ++s) {
      mbar_init(smem_u32(&ring_full[s]), 1);
      mbar_init(smem_u32(&ring_empty[s]), TEAMS);  // one arrive per consumer warpgroup
    }
    mbar_init(smem_u32(&w_full[0]), 1);
    for (int s = 0; s < kResBars; ++s) mbar_init(smem_u32(&res_bars[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_o)) : "memory");
    if (HAS_RES)
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_r)) : "memory");
  }
  // bias (a constant, like the weights: read before the PDL wait) -> shared memory, zero padded
  for (int i = threadIdx.x; i < p.bias_floats; i += blockDim.x)
    smem_bias[i] = i < p.nout ? __ldg(p.bias + i) : 0.f;
  __syncthreads();
  // after the wait: with batch 1 the SE-scaled weights are a single [nout][K] matrix (wbatch 1)
  // that the previous kernel writes
  pdl_wait_prior();          // everything above overlapped the previous kernel's tail

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      const uint32_t w_box_bytes = static_cast<uint32_t>(p.block_n * p.block_k * 2);
      if (p.w_resident) {
        const uint32_t wb = smem_u32(&w_full[0]);
        mbar_expect_tx(wb, w_box_bytes * p.num_n_blocks * p.num_k_blocks);
        for (int nb = 0; nb < p.num_n_blocks; ++nb)
          for (int kb = 0; kb < p.num_k_blocks; ++kb)
            tma_load_3d(smem_u32(smem_w + (nb * p.num_k_blocks + kb) * p.b_stage_bytes), &map_w,
                        wb, kb * p.block_k, nb * p.block_n, 0);
      }
      int stage_of[TEAMS] = {}, phase_of[TEAMS] = {};   // per ring
      // bytes the TMA boxes of one stage deliver (the B slot may be padded to 1 KiB)
      const uint32_t tx_bytes =
          static_cast<uint32_t>(p.a_stage_bytes) + (p.w_resident ? 0u : w_box_bytes);
      int u = blockIdx.x;   // the CTA's first unit; the grid is never larger than total_units
      for (int i = 0;; ++i) {
        // Claim the next unit before this one's loads: the returning atomic on the counter all
        // CTAs share is only waited for at the end of this iteration.
        const int next = u < p.total_units ? sched_claim(p.sched) : p.total_units;
        const int slot = i & (kRing - 1);
        mbar_wait(smem_u32(&ring_empty[slot]), (static_cast<uint32_t>(i / kRing) & 1u) ^ 1u);
        TileCoord tc;
        tc.b = tc.m_blk = tc.n_blk = 0;
        if (u < p.total_units) tc = decode_unit(u, p);
        const_cast<int4*>(tile_ring)[slot] = make_int4(u, tc.b, tc.m_blk, tc.n_blk);
        mbar_arrive(smem_u32(&ring_full[slot]));     // release: the entry is visible to waiters
        if (u >= p.total_units) break;
        const int wb = (p.wbatch > 1) ? tc.b : 0;
        const int team = share ? 0 : i % TEAMS;   // the ring the unit's stages go to
        int stage = stage_of[team];
        uint32_t phase = static_cast<uint32_t>(phase_of[team]);
        const int m_end = min(tc.m_blk + p.unit_m, p.num_m_blocks);
        for (int m_blk = tc.m_blk; m_blk < m_end; ++m_blk) {
          for (int kb = 0; kb < p.num_k_blocks; ++kb) {
            const int s = team * p.team_stages + stage;
            mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
            const uint32_t fb = smem_u32(&full_bar[s]);
            mbar_expect_tx(fb, tx_bytes);
            uint8_t* sa = smem + s * stage_bytes;
            tma_load_3d(smem_u32(sa), &map_a, fb, kb * p.block_k, m_blk * p.tile_m, tc.b);
            if (!p.w_resident)
              tma_load_3d(smem_u32(sa + p.a_stage_bytes), &map_w, fb, kb * p.block_k,
                          tc.n_blk * p.block_n, wb);
            if (++stage == p.team_stages) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
        stage_of[team] = stage;
        phase_of[team] = static_cast<int>(phase);
        u = next;
        if (u >= p.total_units) sched_retire(p.sched);   // this CTA's last claim
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: MMA + epilogue =====================
    const int team = (warp >> 2) - 1;
    const int wtid = threadIdx.x & 127;
    const int r0 = 16 * (warp & 3) + (lane >> 2);   // rows r0 and r0 + 8 of the tile
    const int cq = 2 * (lane & 3);                  // column pair inside each 8-column group
    uint8_t* team_slabs = smem_store + team * p.slab_sets * p.slab_set_bytes;
    const int ring = share ? 0 : team;
    // with share_w this consumer's 64 rows of the 128-row tile: its A rows in a stage, and in the image
    const uint32_t a_off = share ? static_cast<uint32_t>(team * BLOCK_M * p.block_k * 2) : 0u;
    const int team_row = share ? team * BLOCK_M : 0;
    if (p.w_resident) mbar_wait(smem_u32(&w_full[0]), 0);
    // The tile loop for NT 16-column groups: one wgmma of N = 16 NT per k-step over the whole N
    // tile.  W rows of a ragged last tile past nout are TMA zero fill; their columns are computed
    // but not stored.
    auto consume = [&](auto nt_const) {
    constexpr int NT = decltype(nt_const)::value;
    int my_tiles = 0;         // tiles this consumer has run: selects the staging-slab set
    int stage = 0;            // in this consumer's ring: stages ring * team_stages ..
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
      int4 e = const_cast<const int4*>(tile_ring)[slot];
      // Broadcast from lane 0: a value ptxas cannot prove warp-uniform puts the tile loop, and
      // with it every wgmma, on a divergent path, and ptxas then serialises the wgmmas (C7520).
      e.x = __shfl_sync(0xffffffffu, e.x, 0);
      e.y = __shfl_sync(0xffffffffu, e.y, 0);
      e.z = __shfl_sync(0xffffffffu, e.z, 0);
      e.w = __shfl_sync(0xffffffffu, e.w, 0);
      named_sync(1 + team, 128);
      if (wtid == 0) mbar_arrive(smem_u32(&ring_empty[slot]));
      if (e.x >= p.total_units) break;
      if (!share && iter % TEAMS != team) continue;   // another consumer's unit (and ring)
      // The unit's tiles, N tile fastest, with no handshake between them.  With hold_a the A stage
      // of an M block serves every N tile against the resident W and is released after the last.
      const int m_end = min(e.z + p.unit_m, p.num_m_blocks);
      const int n_end = p.hold_a ? p.num_n_blocks : e.w + 1;
      TileCoord tc;
      tc.b = e.y;
      for (tc.m_blk = e.z; tc.m_blk < m_end; ++tc.m_blk) {
        for (tc.n_blk = e.w; tc.n_blk < n_end; ++tc.n_blk) {
          const bool last_n = tc.n_blk + 1 == n_end;
          const int n0 = tc.n_blk * p.block_n;
          // only the columns that exist in the output are worth an epilogue (rounded up to 16); the
          // rest of a ragged last N tile is skipped
          const int n_valid = min(p.block_n, ((p.nout - n0 + 15) >> 4) << 4);
          const int nt = n_valid >> 4;
          const int row_base = tc.m_blk * p.tile_m + team_row;   // first row of this consumer
          // the staging slabs of this tile (a set is free once the stores that last read it --
          // this consumer's previous tile, or the one before that with two sets -- have read it)
          // and the barrier its residual tile lands on
          const int slab_set = my_tiles % p.slab_sets;
          uint8_t* my_slabs = team_slabs + slab_set * p.slab_set_bytes;
          const uint32_t res_bar = smem_u32(&res_bars[team * 2 + slab_set]);
          if constexpr (HAS_RES && EPI == EPI_STORE) {
            // the residual of the tile's rows and stored columns, loaded while the MMAs run (rows
            // past the image and columns past nout are zero fill and are not stored)
            if (row_base < p.rows && wtid == 0) {
              if (p.slab_sets == 2)
                tma_store_wait_read<1>();
              else
                tma_store_wait_read<0>();
              const int boxes = (n_valid + kStoreCols - 1) / kStoreCols;
              mbar_expect_tx(res_bar, static_cast<uint32_t>(boxes * kSlabBytes));
              for (int c = 0; c < boxes; ++c)
                tma_load_3d(smem_u32(my_slabs + c * kSlabBytes), &map_r, res_bar,
                            n0 + c * kStoreCols, row_base, tc.b);
            }
          }
          float acc[NT][8];
#pragma unroll
          for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[j][q] = 0.f;
          // One k-block of MMAs stays in flight: the stage of k-block kb - 1 is released once the
          // MMAs of kb are issued and those of kb - 1 have completed.
          int prev_s = -1;
          for (int kb = 0; kb < p.num_k_blocks; ++kb) {
            const int s = ring * p.team_stages + stage;
            if (tc.n_blk == e.w) mbar_wait(smem_u32(&full_bar[s]), phase);
            uint8_t* sa = smem + s * stage_bytes;
            uint8_t* sb = p.w_resident
                              ? smem_w + (tc.n_blk * p.num_k_blocks + kb) * p.b_stage_bytes
                              : sa + p.a_stage_bytes;
            const uint64_t da = make_smem_desc(smem_u32(sa) + a_off, p.desc_sbo, p.desc_layout);
            const uint64_t db = make_smem_desc(smem_u32(sb), p.desc_sbo, p.desc_layout);
            const int k_rem = p.k - kb * p.block_k;
            const int ksteps = k_rem >= p.block_k ? p.block_k / MMA_K : (k_rem + MMA_K - 1) / MMA_K;
            wg_fence();
            wg_mma_kblock_wide<NT>(acc, da, db, ksteps, kb == 0);
            wg_commit();
            wg_wait<1>();
            if (prev_s >= 0) {
              __syncwarp();
              if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_s]));   // this warp is done with it
            }
            prev_s = s;
            if (last_n) advance();   // hold_a (one k-block): the stage stays for the next N tile
          }
          wg_wait<0>();
          if (last_n) {
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_s]));
          }
          wg_fence_acc<NT>(acc);
          const int row0 = row_base + r0;
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
          } else if (row_base < p.rows) {   // (share_w) rows all past the image: nothing to store
            const uint32_t res_parity = static_cast<uint32_t>(my_tiles / p.slab_sets) & 1u;
            ++my_tiles;
            if (HAS_RES) {
              mbar_wait(res_bar, res_parity);   // the slabs hold the residual tile
            } else {
              if (wtid == 0) {
                if (p.slab_sets == 2)
                  tma_store_wait_read<1>();
                else
                  tma_store_wait_read<0>();
              }
              named_sync(1 + team, 128);
            }
#pragma unroll
            for (int j = 0; j < NT; ++j) {
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
                  const int row = r0 + 8 * r;
                  uint8_t* rb = slab + row * 128 + cq * 2;
                  if (HAS_RES) {
                    lo = fadd2_rn(lo, __half22float2(
                                          *reinterpret_cast<const __half2*>(rb + ((piece ^ (row & 7)) << 4))));
                    hi = fadd2_rn(hi, __half22float2(*reinterpret_cast<const __half2*>(
                                          rb + (((piece + 1) ^ (row & 7)) << 4))));
                  }
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
                             row_base, tc.b);
              tma_store_commit();
            }
          }
        }
      }
    }
    };
    // block_n is a multiple of 32 (pick_block_n); the width is uniform over the kernel
    if constexpr (EPI == EPI_ARGMAX) {
      consume(std::integral_constant<int, kArgmaxCols / 16>{});
    } else {
      switch (p.block_n >> 5) {
        case 1: consume(std::integral_constant<int, 2>{}); break;
        case 2: consume(std::integral_constant<int, 4>{}); break;
        case 3: consume(std::integral_constant<int, 6>{}); break;
        default: consume(std::integral_constant<int, 8>{}); break;
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
  if (nout <= kMaxBlockN) return ((nout + 31) / 32) * 32;   // a wgmma width (wg_mma_kblock_wide)
  return kMaxBlockN;
}

template <int ACT, bool HAS_RES, int TEAMS, int EPI = EPI_STORE>
static int launch(const CUtensorMap& ma, const CUtensorMap& mw, const CUtensorMap& mo,
                  const CUtensorMap& mr, const Params& p, int grid, int smem_bytes,
                  cudaStream_t stream) {
  auto kern = pointwise_tc_kernel<ACT, HAS_RES, TEAMS, EPI>;
  static int configured[kMaxDevices];   // per instantiation and device; no API call once set
  if (int rc = ensure_dynamic_smem(kern, kSmemLimit, configured)) return rc;
  EDET_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(Epi<TEAMS>::kThreads), smem_bytes, stream, ma,
                             mw, mo, mr, p));
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
  // edet_set_option("pw_teams", 2 | 3) forces a variant for A/B measurements.  The arg-max
  // epilogue is only instantiated with two, so its rings are planned for two.
  const int opt_teams = option_pw_teams();
  const int teams = (opt_teams && !am) ? opt_teams : 2;
  p.block_n = am ? kArgmaxCols : pick_block_n(nout);
  p.num_n_blocks = ceil_div(nout, p.block_n);
  p.wbatch = wbatch;
  p.ldr = ldr;
  p.bias = bias;
  p.residual = residual;
  if (int rc = next_sched_slot(&p.sched)) return rc;

  // every column the epilogue can touch: whole N tiles (n_valid is rounded up to 16 inside a tile)
  const int bias_cols = p.num_n_blocks * p.block_n;
  EDET_CHECK_ARG(bias_cols <= kMaxBiasSmem, "pointwise_tc: nout %d too wide", nout);
  p.bias_floats = bias_cols;
  // k-block / smem row pitch: 16 halves (32B swizzle) for K <= 16, 32 (64B) for K <= 32, else 64
  // (128B), so that a stage only holds bytes that exist.  A shared W that the K padding of 64-wide
  // k-blocks alone pushes over kResidentWBytes takes 32-wide ones (blocks_6-8 expand, K 80 x N 480:
  // 96 instead of 128 padded columns, 96 instead of 128 KB), so it stays resident.  Shapes only:
  // the k16 steps of every output, and so its bits, do not depend on the options.
  auto w_bytes_for = [&](int bk) {
    return p.num_n_blocks * ceil_div(k, bk) * (((p.block_n * bk * 2 + 1023) / 1024) * 1024);
  };
  p.block_k = k <= 16 ? 16 : (k <= 32 ? 32 : 64);
  if (p.block_k == 64 && wbatch == 1 && w_bytes_for(64) > kResidentWBytes &&
      w_bytes_for(32) <= kResidentWBytes)
    p.block_k = 32;
  p.a_stage_bytes = BLOCK_M * p.block_k * 2;
  p.b_stage_bytes = ((p.block_n * p.block_k * 2 + 1023) / 1024) * 1024;
  p.num_k_blocks = ceil_div(k, p.block_k);
  // Shared weights small enough stay resident: the ring then carries only A, and the class head
  // reads each A tile from L2 once per anchor instead of once per anchor AND W tile.  Per-image
  // (SE-scaled) weights keep streaming with A.
  const int w_bytes = w_bytes_for(p.block_k);
  p.w_resident = wbatch == 1 && w_bytes <= kResidentWBytes;

  // the arg-max epilogue stores nothing through TMA: no staging slabs
  p.slab_set_bytes = am ? 0 : ceil_div(p.block_n, kStoreCols) * kSlabBytes;
  const int opt_kb = option_pw_smem_kb();
  const int limit = opt_kb ? opt_kb * 1024 : kSmemLimit;
  auto fixed_bytes = [&](int sets) {
    return (p.w_resident ? w_bytes : 0) + teams * sets * p.slab_set_bytes + p.bias_floats * 4 +
           (2 * kMaxStages + 2 * kRing + 2 + kResBars) * 8 + 16 * kRing;
  };
  // Under a smaller pw_smem_kb budget resident W may not leave two A stages per consumer next to
  // one slab set: W then streams with A.  At the default budget every W of at most
  // kResidentWBytes leaves that room, so this only changes plans that would otherwise be refused.
  if (p.w_resident && (limit - 1024 - fixed_bytes(1)) / p.a_stage_bytes < 2 * teams)
    p.w_resident = 0;
  // Stages of tiles of tile_m rows in `rings` rings (one per consumer, or one shared ring); returns
  // the most stages each ring can have.  Two slab sets per consumer (the stores of one tile drain
  // while the next epilogue writes) when that still leaves three stages per consumer ring, or
  // kMinTeamStages in a shared one; else one.
  auto plan_rings = [&](int tile_m, int rings) {
    p.tile_m = tile_m;
    p.share_w = rings == 1 && teams > 1;
    p.num_m_blocks = ceil_div(rows, tile_m);
    p.a_stage_bytes = tile_m * p.block_k * 2;
    p.stage_bytes = p.a_stage_bytes + (p.w_resident ? 0 : p.b_stage_bytes);
    const int sets2_stages = rings == 1 ? kMinTeamStages : 3 * rings;
    p.slab_sets = (limit - 1024 - fixed_bytes(2)) / p.stage_bytes >= sets2_stages ? 2 : 1;
    return std::min((limit - 1024 - fixed_bytes(p.slab_sets)) / p.stage_bytes, kMaxStages) / rings;
  };
  int max_team_stages = plan_rings(BLOCK_M, teams);
  EDET_CHECK_ARG(max_team_stages >= 2, "pointwise_tc: block_n %d leaves <2 pipeline stages per consumer",
                 p.block_n);

  // the grid before the work units are known; capped by their number below
  int grid = persistent_grid(INT_MAX, 1);
  if (!grid) return EDET_ERR_CUDA;
  // Shared W: where W streams with A and two consumers run, both take one 128-row tile against
  // one W tile per k-block (half the W traffic from L2), provided the launch still has a 128-row
  // tile for every CTA (with fewer, 64-row tiles spread the work over more SMs), the main loop is
  // long enough to cover the epilogues that now run together (kShareResMinKBlocks) and the budget
  // holds kMinTeamStages shared stages.  Any budget that refuses the 64-row plan refuses this one.
  if (teams == 2 && !am && !p.w_resident && option_pw_share_w() == 0 &&
      batch * ceil_div(rows, 2 * BLOCK_M) * p.num_n_blocks >= grid &&
      (!residual || p.num_k_blocks >= kShareResMinKBlocks)) {
    const int shared_stages = plan_rings(2 * BLOCK_M, 1);
    if (shared_stages >= kMinTeamStages)
      max_team_stages = shared_stages;
    else
      plan_rings(BLOCK_M, teams);
  }
  const int rings = p.share_w ? 1 : teams;
  const int fixed = fixed_bytes(p.slab_sets);
  // Work units.  With W resident and one k-block an M block's A tile serves every N tile (the
  // class head: all anchors of its rows).  A is held only while the M blocks alone still give
  // every CTA a unit: with fewer (the small class-head levels) the N tiles of an M block finish
  // sooner spread over several CTAs.
  p.hold_a = p.w_resident && p.num_n_blocks > 1 && p.num_k_blocks == 1 &&
             batch * p.num_m_blocks >= grid;
  const int unit_n_blocks = p.hold_a ? p.num_n_blocks : 1;
  // bytes of one M block of a unit: its stages (A, and W when streamed) and its output tiles
  const int m_block_bytes =
      p.num_k_blocks * p.stage_bytes + unit_n_blocks * p.tile_m * p.block_n * 2;
  auto units_for = [&](int g) {
    return batch * ceil_div(p.num_m_blocks, g) * (p.hold_a ? 1 : p.num_n_blocks);
  };
  // A unit is the largest of 1, 2, 4, 8 M blocks that still leaves at least kUnitsPerCta units
  // per CTA (the tail of the dynamic schedule stays short), moves at most kMaxUnitBytes, and whose
  // stages fit in one ring (the single producer fills the consumers' rings in unit order, so a
  // unit that does not fit would keep the other consumer waiting).  The per-unit handshake and
  // claim are then spread over several tiles.
  p.unit_m = 8;
  while (p.unit_m > 1 && (units_for(p.unit_m) < kUnitsPerCta * grid ||
                          p.unit_m * m_block_bytes > kMaxUnitBytes ||
                          p.unit_m * p.num_k_blocks > max_team_stages))
    p.unit_m >>= 1;
  p.units_per_image = ceil_div(p.num_m_blocks, p.unit_m);
  p.total_units = units_for(p.unit_m);
  if (p.total_units < grid) grid = p.total_units;
  // a shared ring feeds both consumers: the loads in flight of two
  p.team_stages = std::min(max_team_stages,
                           std::max({kMinTeamStages,
                                     ceil_div(kTeamInFlightBytes * (teams / rings), p.stage_bytes),
                                     p.unit_m * p.num_k_blocks}));
  const int stages = p.team_stages * rings;
  p.num_stages = stages;
  p.desc_layout = desc_layout_for(p.block_k);
  p.desc_sbo = 8 * p.block_k * 2;
  const int smem_bytes = 1024 + stages * p.stage_bytes + fixed;

  CUtensorMap ma, mw, mo, mr;
  int rc;
  if ((rc = make_map(&ma, a, k, rows, batch, lda, static_cast<uint64_t>(rows) * lda, p.tile_m,
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
  // residual boxes: the store box, read into the staging slabs
  mr = mo;
  if (residual && (rc = make_map(&mr, residual, nout, rows, batch, ldr,
                                 static_cast<uint64_t>(rows) * ldr, BLOCK_M, kStoreCols)))
    return rc;

  const bool has_res = residual != nullptr;
  if (am) return launch<EDET_ACT_NONE, false, 2, EPI_ARGMAX>(ma, mw, mo, mr, p, grid, smem_bytes, stream);

#define EDET_PW_CASE(A)                                                                       \
  if (teams == 3)                                                                             \
    return has_res ? launch<A, true, 3>(ma, mw, mo, mr, p, grid, smem_bytes, stream)              \
                   : launch<A, false, 3>(ma, mw, mo, mr, p, grid, smem_bytes, stream);            \
  return has_res ? launch<A, true, 2>(ma, mw, mo, mr, p, grid, smem_bytes, stream)                \
                 : launch<A, false, 2>(ma, mw, mo, mr, p, grid, smem_bytes, stream)
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
