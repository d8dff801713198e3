// Post-processing on the device: pre-NMS (class max/argmax + sigmoid + anchor decode) and a
// bit-faithful NonMaxSuppressionV5 (hard / gaussian soft) followed by the serving-layout gather.
#include <math_constants.h>

#include "common.cuh"

namespace edet {

// ------------------------------------------------------------------------------------------
// pre-NMS
// ------------------------------------------------------------------------------------------
constexpr int kPreMaxLevels = 8;
constexpr int kPrePix = 16;       // pixels per CTA
constexpr int kPreThreads = 256;

struct PreLevel {
  const __half* cls;
  const __half* box;
  int pixels;        // h*w
  int block_begin;   // first CTA (blockIdx.x) of this level
  int anchor_begin;  // first flattened anchor of this level
};
struct PreParams {
  PreLevel lv[kPreMaxLevels];
  int levels, ld_cls, ld_box, num_anchors, num_classes, total_anchors;
};

__global__ void __launch_bounds__(kPreThreads)
pre_nms_kernel(const PreParams p, const float* __restrict__ anchors, float* __restrict__ boxes,
               float* __restrict__ scores, int32_t* __restrict__ classes) {
  pdl_launch_dependents();
  pdl_wait_prior();
  extern __shared__ __align__(16) uint8_t pre_smem[];
  __half* cls_s = reinterpret_cast<__half*>(pre_smem);
  int l = 0;
  while (l + 1 < p.levels && static_cast<int>(blockIdx.x) >= p.lv[l + 1].block_begin) ++l;
  const PreLevel lv = p.lv[l];
  const int n = blockIdx.y;
  const int pix0 = (blockIdx.x - lv.block_begin) * kPrePix;
  const int npix = min(kPrePix, lv.pixels - pix0);
  const bool with_classes = lv.cls != nullptr;   // uniform; false: edet_class_argmax wrote them
  if (with_classes) {
    // coalesced copy of npix * ld_cls halves (contiguous in NHWC)
    const uint4* src = reinterpret_cast<const uint4*>(
        lv.cls + (static_cast<size_t>(n) * lv.pixels + pix0) * p.ld_cls);
    const int nvec = npix * p.ld_cls / 8;
    for (int i = threadIdx.x; i < nvec; i += kPreThreads)
      reinterpret_cast<uint4*>(cls_s)[i] = ldg_nc_v4(src + i);
    __syncthreads();
  }
  const int t = threadIdx.x;
  if (t >= npix * p.num_anchors) return;
  const int pl = t / p.num_anchors, a = t - pl * p.num_anchors;
  const int anchor = lv.anchor_begin + (pix0 + pl) * p.num_anchors + a;
  const size_t o = static_cast<size_t>(n) * p.total_anchors + anchor;
  if (with_classes) {
    const __half* row = cls_s + pl * p.ld_cls + a * p.num_classes;
    float best = __half2float(row[0]);
    int best_c = 0;
    for (int c = 1; c < p.num_classes; ++c) {
      const float v = __half2float(row[c]);
      if (v > best) {  // strict: first maximum wins, like tf.argmax
        best = v;
        best_c = c;
      }
    }
    scores[o] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-best)));
    classes[o] = best_c;
  }
  // box decode (tf2/anchors.py:30-58), float32, no FMA contraction
  const uint2 bv = __ldg(reinterpret_cast<const uint2*>(
      lv.box + (static_cast<size_t>(n) * lv.pixels + pix0 + pl) * p.ld_box + a * 4));
  reinterpret_cast<float4*>(boxes)[o] =
      decode_box(bv, __ldg(reinterpret_cast<const float4*>(anchors) + anchor));
}

// ------------------------------------------------------------------------------------------
// NonMaxSuppressionV5 (TensorFlow core/kernels/image/non_max_suppression_op.cc semantics)
// ------------------------------------------------------------------------------------------
constexpr int kNmsThreads = 1024;
constexpr int kNmsMaxOut = 512;

__device__ __forceinline__ bool better(float sa, int ia, float sb, int ib) {
  return sa > sb || (sa == sb && ia < ib);
}

__device__ __forceinline__ float iou_tf(const float4 a, const float4 b) {
  const float ymin_i = fminf(a.x, a.z), xmin_i = fminf(a.y, a.w);
  const float ymax_i = fmaxf(a.x, a.z), xmax_i = fmaxf(a.y, a.w);
  const float ymin_j = fminf(b.x, b.z), xmin_j = fminf(b.y, b.w);
  const float ymax_j = fmaxf(b.x, b.z), xmax_j = fmaxf(b.y, b.w);
  const float area_i = __fmul_rn(__fsub_rn(ymax_i, ymin_i), __fsub_rn(xmax_i, xmin_i));
  const float area_j = __fmul_rn(__fsub_rn(ymax_j, ymin_j), __fsub_rn(xmax_j, xmin_j));
  if (area_i <= 0.f || area_j <= 0.f) return 0.f;
  const float iymin = fmaxf(ymin_i, ymin_j), ixmin = fmaxf(xmin_i, xmin_j);
  const float iymax = fminf(ymax_i, ymax_j), ixmax = fminf(xmax_i, xmax_j);
  const float inter = __fmul_rn(fmaxf(__fsub_rn(iymax, iymin), 0.f),
                                fmaxf(__fsub_rn(ixmax, ixmin), 0.f));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_i, area_j), inter));
}

__global__ void __launch_bounds__(kNmsThreads)
nms_v5_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
              const int32_t* __restrict__ classes, const float* __restrict__ image_scales,
              int image_id_base, int k, int max_out, float iou_thr, float score_thr, float sigma,
              float clip_h, float clip_w, float* __restrict__ detections,
              int32_t* __restrict__ sel_index, int32_t* __restrict__ valid,
              float* __restrict__ work_scores, int32_t* __restrict__ work_begin,
              const int32_t* __restrict__ need_full) {
  // Full-queue path: only runs for images the shared-memory fast path could not prove exact.
  if (need_full != nullptr && need_full[blockIdx.x] == 0) return;
  __shared__ float4 sel_box[kNmsMaxOut];
  __shared__ int sel_idx[kNmsMaxOut];
  __shared__ float sel_score[kNmsMaxOut];
  __shared__ float sim_s[kNmsMaxOut];
  __shared__ float wgt_s[kNmsMaxOut];
  __shared__ float red_s[32];
  __shared__ int red_i[32];
  __shared__ int best_i;
  __shared__ int nsel_s;

  const int n = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float4* bx = reinterpret_cast<const float4*>(boxes) + static_cast<size_t>(n) * k;
  const float* sc = scores + static_cast<size_t>(n) * k;
  float* ws = work_scores + static_cast<size_t>(n) * k;
  int32_t* wb = work_begin + static_cast<size_t>(n) * k;
  const bool soft = sigma > 0.f;
  const float scale = soft ? __fdiv_rn(-0.5f, sigma) : 0.f;

  // candidate queue = every box with score > threshold; removed entries become -inf
  float my_s = -CUDART_INF_F;
  int my_i = 0x7fffffff;
  for (int i = tid; i < k; i += kNmsThreads) {
    float s = sc[i];
    if (!(s > score_thr)) s = -CUDART_INF_F;
    ws[i] = s;
    wb[i] = 0;
    if (better(s, i, my_s, my_i)) {
      my_s = s;
      my_i = i;
    }
  }
  if (tid == 0) nsel_s = 0;
  __syncthreads();

  while (true) {
    // ---- pop: block-wide arg-max, ties to the lower index ----
    float s = my_s;
    int i = my_i;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float so = __shfl_xor_sync(0xffffffffu, s, o);
      const int io = __shfl_xor_sync(0xffffffffu, i, o);
      if (better(so, io, s, i)) {
        s = so;
        i = io;
      }
    }
    if (lane == 0) {
      red_s[warp] = s;
      red_i[warp] = i;
    }
    __syncthreads();
    if (warp == 0) {
      s = red_s[lane];
      i = red_i[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float so = __shfl_xor_sync(0xffffffffu, s, o);
        const int io = __shfl_xor_sync(0xffffffffu, i, o);
        if (better(so, io, s, i)) {
          s = so;
          i = io;
        }
      }
      const int nsel = nsel_s;
      if (s == -CUDART_INF_F || nsel >= max_out) {
        if (lane == 0) best_i = -1;
      } else {
        // ---- lazily apply the suppression of the boxes selected since the last visit ----
        const int begin = wb[i];
        const float4 cb = bx[i];
        for (int j = begin + lane; j < nsel; j += 32) {
          const float sim = iou_tf(cb, sel_box[j]);
          float wgt = static_cast<float>(exp(static_cast<double>(__fmul_rn(__fmul_rn(scale, sim), sim))));
          if (!(soft || sim <= iou_thr)) wgt = 0.f;
          sim_s[j] = sim;
          wgt_s[j] = wgt;
        }
        __syncwarp();
        if (lane == 0) {
          float cur = s;
          bool hard = false;
          for (int j = nsel - 1; j >= begin; --j) {
            cur = __fmul_rn(cur, wgt_s[j]);
            if (!soft && sim_s[j] > iou_thr) {
              hard = true;
              break;
            }
            if (cur <= score_thr) break;
          }
          float new_s = -CUDART_INF_F;
          if (!hard) {
            if (cur == s) {
              sel_box[nsel] = cb;
              sel_idx[nsel] = i;
              sel_score[nsel] = cur;
              nsel_s = nsel + 1;
            } else if (cur > score_thr) {
              new_s = cur;
              wb[i] = nsel;
            }
          }
          ws[i] = new_s;
          best_i = i;
        }
      }
    }
    __syncthreads();
    const int popped = best_i;
    if (popped < 0) break;
    if ((popped % kNmsThreads) == tid) {
      // owner refreshes its cached local best
      my_s = -CUDART_INF_F;
      my_i = 0x7fffffff;
      for (int j0 = tid; j0 < k; j0 += 8 * kNmsThreads) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {   // issue the loads together: this is latency bound
          const int j = j0 + u * kNmsThreads;
          v[u] = j < k ? ws[j] : -CUDART_INF_F;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int j = j0 + u * kNmsThreads;
          if (j < k && better(v[u], j, my_s, my_i)) {
            my_s = v[u];
            my_i = j;
          }
        }
      }
    }
    // (no barrier needed here: the next iteration's first __syncthreads orders best_i reuse)
  }

  // ---- gather into the serving layout (padded with index 0 / score 0, like TF) ----
  const int nsel = nsel_s;
  const float scale_img = image_scales ? image_scales[n] : 1.f;
  for (int r = tid; r < max_out; r += kNmsThreads) {
    const int idx = r < nsel ? sel_idx[r] : 0;
    const float score = r < nsel ? sel_score[r] : 0.f;
    const float4 b = bx[idx];
    float* d = detections + (static_cast<size_t>(n) * max_out + r) * 7;
    d[0] = static_cast<float>(image_id_base + n);
    d[1] = __fmul_rn(fminf(fmaxf(b.x, 0.f), clip_h), scale_img);
    d[2] = __fmul_rn(fminf(fmaxf(b.y, 0.f), clip_w), scale_img);
    d[3] = __fmul_rn(fminf(fmaxf(b.z, 0.f), clip_h), scale_img);
    d[4] = __fmul_rn(fminf(fmaxf(b.w, 0.f), clip_w), scale_img);
    d[5] = score;
    d[6] = static_cast<float>(classes[static_cast<size_t>(n) * k + idx] + 1);
    sel_index[static_cast<size_t>(n) * max_out + r] = idx;
  }
  if (tid == 0) valid[n] = nsel;
}


// ------------------------------------------------------------------------------------------
// Fast path: the same algorithm, batched, on the top candidates only, in shared memory.
//
// TF's NMS-V5 pops one candidate at a time from a lazily-updated max-heap.  Between two
// selections the selected set S is fixed, so the pops of that "period" can be replayed in
// parallel without changing a single bit:
//   * walk the queue in descending stale-score order; every visited candidate x gets its
//     pending suppression applied (boxes begin_x..|S|-1, newest first, with TF's break rules),
//     giving u_x -- independent of the other candidates, so a whole chunk is done at once
//     (8 lanes per candidate, 64 candidates per chunk);
//   * the period ends at the first position p where either a candidate updated earlier in the
//     period ("fresh", already up to date) now beats x_p -- then that fresh candidate is
//     selected with its decayed score -- or x_p itself came out unchanged -- then x_p is
//     selected.  Everything before p is committed (re-queued with its new score, or dropped).
// The queue is (A) the compacted top candidates, sorted once by (score desc, index asc), consumed
// through a pointer, plus (B) a small sorted array of re-queued candidates; a chunk is the
// rank-merge of the heads of A and B.
//
// Only the top <= kBCapA candidates per image are considered (adaptive two-level histogram
// threshold on the score bits); exactness is PROVEN per image at run time -- every candidate
// touched must score strictly above the best excluded one -- otherwise the image is flagged and
// the full-queue kernel above recomputes it.
// ------------------------------------------------------------------------------------------
constexpr int kBT = 512;            // threads per image
constexpr int kBCapA = 8192;
constexpr int kBCapB = 4096;
constexpr int kBChunk = 64;         // candidates per chunk (8 lanes each)
constexpr int kFastBins = 2048;

// -0 takes +0's key: better() and TF's heap treat the two scores as equal (index order decides)
__device__ __forceinline__ uint32_t score_key(float s) {
  const uint32_t b = s == 0.f ? 0u : __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);  // monotone float -> uint
}
__device__ __forceinline__ float key_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}
// 64-bit queue key: larger == popped earlier (score descending, then index ascending)
__device__ __forceinline__ unsigned long long make_qkey(float s, int idx) {
  return (static_cast<unsigned long long>(score_key(s)) << 32) |
         static_cast<unsigned long long>(~static_cast<uint32_t>(idx));
}
__device__ __forceinline__ float qkey_score(unsigned long long k) {
  return key_score(static_cast<uint32_t>(k >> 32));
}
__device__ __forceinline__ int qkey_idx(unsigned long long k) {
  return static_cast<int>(~static_cast<uint32_t>(k));
}

struct BatchSmem {
  unsigned long long a_key[kBCapA];   // sorted descending; consumed through `ptr`
  unsigned long long b_key[kBCapB];   // sorted descending
  unsigned short b_begin[kBCapB];
  int hist[kFastBins];
  float4 sel_box[kNmsMaxOut];
  int sel_idx[kNmsMaxOut];
  float sel_score[kNmsMaxOut];
  unsigned long long c_key[kBChunk];    // stale key of the chunk position
  unsigned long long c_fresh[kBChunk];  // key after the update (0: dropped / not re-queued)
  float c_u[kBChunk];
  unsigned short c_begin[kBChunk];
  short c_src[kBChunk];                 // >= 0: offset in A from ptr; < 0: -(B index) - 1
  unsigned char c_unchanged[kBChunk];
  unsigned long long n_key[kBChunk];    // re-queued entries of this commit, sorted descending
  float red_s[kBT / 32];
  uint32_t kmin, kmax;
  int count, bstar, sstar, fail;
  int ptr, nb, m, chunk_n;
  int stop_p, sel_pos, sel_is_fresh, pa, pb, n_new;
  float excl_max;
};

// number of elements of the descending array arr[0..n) that are greater than key
__device__ __forceinline__ int count_greater(const unsigned long long* arr, int n,
                                             unsigned long long key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (arr[mid] > key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kBT)
nms_v5_fast_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                   const int32_t* __restrict__ classes, const float* __restrict__ image_scales,
                   int image_id_base, int k, int max_out, float iou_thr, float score_thr,
                   float sigma, float clip_h, float clip_w, float* __restrict__ detections,
                   int32_t* __restrict__ sel_index, int32_t* __restrict__ valid,
                   int32_t* __restrict__ need_full) {
  extern __shared__ __align__(16) uint8_t fast_raw[];
  BatchSmem& sm = *reinterpret_cast<BatchSmem*>(fast_raw);
  const int n = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float4* bx = reinterpret_cast<const float4*>(boxes) + static_cast<size_t>(n) * k;
  const float* sc = scores + static_cast<size_t>(n) * k;
  const bool soft = sigma > 0.f;
  const float scale = soft ? __fdiv_rn(-0.5f, sigma) : 0.f;

  // ---- A. key range of the valid candidates ----
  uint32_t kmin = 0xffffffffu, kmax = 0u;
  for (int i = tid; i < k; i += kBT) {
    const float s = sc[i];
    if (s > score_thr) {
      const uint32_t key = score_key(s);
      kmin = min(kmin, key);
      kmax = max(kmax, key);
    }
  }
  if (tid == 0) {
    sm.kmin = 0xffffffffu; sm.kmax = 0u; sm.count = 0; sm.fail = 0;
    sm.excl_max = -CUDART_INF_F; sm.bstar = 0; sm.sstar = 0;
    sm.ptr = 0; sm.nb = 0; sm.m = 0;
  }
  for (int i = tid; i < kFastBins; i += kBT) sm.hist[i] = 0;
  __syncthreads();
  atomicMin(&sm.kmin, kmin);
  atomicMax(&sm.kmax, kmax);
  __syncthreads();
  kmin = sm.kmin; kmax = sm.kmax;
  const bool any_valid = kmax >= kmin;
  // bin = floor((key - kmin) * inv) in [0, kFastBins); the fraction inside the bin gives a
  // second-level sub-bin.  Both are monotone in the key, which is all the selection needs.
  const double inv = static_cast<double>(kFastBins) /
                     (static_cast<double>(any_valid ? kmax - kmin : 0u) + 1.0);
  auto bin_of = [&](uint32_t key, int& sub) -> int {
    const double x = static_cast<double>(key - kmin) * inv;
    int b = static_cast<int>(x);
    b = b > kFastBins - 1 ? kFastBins - 1 : b;
    int sb = static_cast<int>((x - static_cast<double>(b)) * kFastBins);
    sub = sb > kFastBins - 1 ? kFastBins - 1 : (sb < 0 ? 0 : sb);
    return b;
  };
  // ---- B. coarse histogram -> threshold bin ----
  if (any_valid) {
    for (int i = tid; i < k; i += kBT) {
      const float s = sc[i];
      int sub;
      if (s > score_thr) atomicAdd(&sm.hist[bin_of(score_key(s), sub)], 1);
    }
  }
  __syncthreads();
  if (tid == 0) {
    int acc = 0, b = kFastBins;
    while (b > 0 && acc + sm.hist[b - 1] <= kBCapA) acc += sm.hist[--b];
    sm.bstar = b;       // bins >= bstar are taken whole; bin bstar-1 is refined below
    sm.count = acc;     // (reused as the running total for the refinement)
  }
  __syncthreads();
  const int bstar = sm.bstar;
  const int coarse_total = sm.count;
  __syncthreads();
  // ---- B2. refine the boundary bin with a second-level histogram ----
  for (int i = tid; i < kFastBins; i += kBT) sm.hist[i] = 0;
  __syncthreads();
  if (any_valid && bstar > 0) {
    for (int i = tid; i < k; i += kBT) {
      const float s = sc[i];
      if (s > score_thr) {
        int sub;
        if (bin_of(score_key(s), sub) == bstar - 1) atomicAdd(&sm.hist[sub], 1);
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    int acc = coarse_total, sb = kFastBins;
    if (bstar > 0)
      while (sb > 0 && acc + sm.hist[sb - 1] <= kBCapA) acc += sm.hist[--sb];
    sm.sstar = sb;
    sm.count = 0;
    if (any_valid && acc == 0) sm.fail = 1;  // one score value alone overflows the capacity
  }
  __syncthreads();
  const int sstar = sm.sstar;
  // ---- D. compaction into shared memory; best excluded score ----
  float excl = -CUDART_INF_F;
  if (any_valid && !sm.fail) {
    for (int i = tid; i < k; i += kBT) {
      const float s = sc[i];
      if (s > score_thr) {
        int sub;
        const int b = bin_of(score_key(s), sub);
        if (b >= bstar || (b == bstar - 1 && sub >= sstar)) {
          const int slot = atomicAdd(&sm.count, 1);
          sm.a_key[slot] = make_qkey(s, i);
        } else {
          excl = fmaxf(excl, s);
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) excl = fmaxf(excl, __shfl_xor_sync(0xffffffffu, excl, o));
  if (lane == 0) sm.red_s[warp] = excl;
  __syncthreads();
  if (tid == 0) {
    float e = -CUDART_INF_F;
    for (int w = 0; w < kBT / 32; ++w) e = fmaxf(e, sm.red_s[w]);
    sm.excl_max = e;
  }
  const int count = sm.count;
  int npow2 = 1;
  while (npow2 < count) npow2 <<= 1;
  for (int sl = count + tid; sl < npow2; sl += kBT) sm.a_key[sl] = 0ull;
  __syncthreads();
  const float excl_max = sm.excl_max;
  // ---- sort A descending (bitonic, in shared memory) ----
  for (int size = 2; size <= npow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < (npow2 >> 1); t += kBT) {
        const int lo = 2 * t - (t & (stride - 1));   // index with bit `stride` cleared
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long x = sm.a_key[lo], y = sm.a_key[hi];
        if ((x < y) == desc) { sm.a_key[lo] = y; sm.a_key[hi] = x; }
      }
      __syncthreads();
    }
  }

  // ---- E. periods ----
  const int cand = tid >> 3, sub = tid & 7;          // 8 lanes per chunk candidate
  const unsigned gmask = 0xffu << ((lane >> 3) << 3);  // this candidate's lanes in the warp
  while (!sm.fail) {
    const int m = sm.m, ptr = sm.ptr, nb = sm.nb;     // stable: written only before the last barrier
    if (m >= max_out) break;
    const int ka = min(kBChunk, count - ptr), kb = min(kBChunk, nb);
    if (ka + kb == 0) {                               // queue exhausted
      if (excl_max > -CUDART_INF_F) { if (tid == 0) sm.fail = 2; __syncthreads(); }
      break;
    }
    // -- chunk = rank-merge of the heads of A and B --
    if (tid < ka) {
      const unsigned long long key = sm.a_key[ptr + tid];
      const int r = tid + count_greater(sm.b_key, kb, key);
      if (r < kBChunk) {
        sm.c_key[r] = key; sm.c_begin[r] = 0; sm.c_src[r] = static_cast<short>(tid);
      }
    } else if (tid >= kBChunk && tid < kBChunk + kb) {
      const int j = tid - kBChunk;
      const unsigned long long key = sm.b_key[j];
      const int r = j + count_greater(sm.a_key + ptr, ka, key);
      if (r < kBChunk) {
        sm.c_key[r] = key; sm.c_begin[r] = sm.b_begin[j]; sm.c_src[r] = static_cast<short>(-j - 1);
      }
    }
    const int chunk_n = min(kBChunk, ka + kb);
    __syncthreads();
    // -- pending suppression of every chunk candidate, 8 lanes each --
    if (cand < chunk_n) {
      const unsigned long long key = sm.c_key[cand];
      const float s = qkey_score(key);
      const int idx = qkey_idx(key);
      const int begin = sm.c_begin[cand];
      const float4 cb = bx[idx];
      float cur = s;
      bool hard = false, done = false;
      for (int hi = m; hi > begin && !done; hi -= 8) {
        const int j = hi - 1 - sub;                    // sub-lane 0 = newest of this group of 8
        float simv = 0.f;
        if (j >= begin) simv = iou_tf(cb, sm.sel_box[j]);
        unsigned mask = (__ballot_sync(gmask, simv > 0.f) >> ((lane >> 3) << 3)) & 0xffu;
        float wgt = 1.f;
        if (simv > 0.f) {
          wgt = static_cast<float>(exp(static_cast<double>(__fmul_rn(__fmul_rn(scale, simv), simv))));
          if (!(soft || simv <= iou_thr)) wgt = 0.f;
        }
        while (mask) {                                 // ascending sub-lane = descending j
          const int l = __ffs(mask) - 1;
          mask &= mask - 1;
          const int src = (lane & ~7) + l;
          const float wl = __shfl_sync(gmask, wgt, src);
          const float sl = __shfl_sync(gmask, simv, src);
          cur = __fmul_rn(cur, wl);
          if (!soft && sl > iou_thr) { hard = true; done = true; break; }
          if (cur <= score_thr) { done = true; break; }
        }
      }
      if (sub == 0) {
        const bool unchanged = !hard && (cur == s);
        const bool requeue = !hard && !unchanged && (cur > score_thr);
        sm.c_u[cand] = cur;
        sm.c_unchanged[cand] = unchanged ? 1 : 0;
        sm.c_fresh[cand] = requeue ? make_qkey(cur, idx) : 0ull;
      }
    }
    __syncthreads();
    // -- where does the period end? (warp 0; two chunk positions per lane) --
    if (warp == 0) {
      unsigned long long f0 = lane < chunk_n ? sm.c_fresh[lane] : 0ull;
      unsigned long long f1 = lane + 32 < chunk_n ? sm.c_fresh[lane + 32] : 0ull;
      // inclusive prefix max over 32 lanes, then shift to exclusive
      unsigned long long p0 = f0, p1 = f1;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t0 = __shfl_up_sync(0xffffffffu, p0, o);
        const unsigned long long t1 = __shfl_up_sync(0xffffffffu, p1, o);
        if (lane >= o) { p0 = max(p0, t0); p1 = max(p1, t1); }
      }
      const unsigned long long tot0 = __shfl_sync(0xffffffffu, p0, 31);
      unsigned long long e0 = __shfl_up_sync(0xffffffffu, p0, 1);
      unsigned long long e1 = __shfl_up_sync(0xffffffffu, p1, 1);
      if (lane == 0) { e0 = 0ull; e1 = 0ull; }
      e1 = max(e1, tot0);
      const bool in0 = lane < chunk_n, in1 = lane + 32 < chunk_n;
      const bool stop0 = in0 && ((e0 > sm.c_key[lane]) || sm.c_unchanged[lane]);
      const bool stop1 = in1 && ((e1 > sm.c_key[lane + 32]) || sm.c_unchanged[lane + 32]);
      const unsigned b0 = __ballot_sync(0xffffffffu, stop0), b1 = __ballot_sync(0xffffffffu, stop1);
      int p = chunk_n;
      if (b0) p = __ffs(b0) - 1; else if (b1) p = 32 + __ffs(b1) - 1;
      const bool stopped = p < chunk_n;
      // the exclusive prefix max at p decides between the two endings
      unsigned long long ep = 0ull;
      if (stopped) ep = p < 32 ? __shfl_sync(0xffffffffu, e0, p) : __shfl_sync(0xffffffffu, e1, p - 32);
      const bool fresh_wins = stopped && ep > sm.c_key[stopped ? p : 0];
      // position of the fresh candidate that holds the prefix max
      const unsigned m0 = __ballot_sync(0xffffffffu, fresh_wins && f0 == ep && lane < p);
      const unsigned m1 = __ballot_sync(0xffffffffu, fresh_wins && f1 == ep && lane + 32 < p);
      int sel_pos = -1;
      if (stopped) sel_pos = fresh_wins ? (m0 ? __ffs(m0) - 1 : 32 + __ffs(m1) - 1) : p;
      // elements consumed from the queue: positions < pe (the selected x_p is consumed too)
      const int pe = stopped ? (fresh_wins ? p : p + 1) : chunk_n;
      const bool c0 = lane < pe, c1 = lane + 32 < pe;
      const int a0 = c0 && sm.c_src[lane] >= 0, a1 = c1 && sm.c_src[lane + 32] >= 0;
      const int pa = __popc(__ballot_sync(0xffffffffu, a0)) + __popc(__ballot_sync(0xffffffffu, a1));
      const int pbv = __popc(__ballot_sync(0xffffffffu, c0 && !a0)) + __popc(__ballot_sync(0xffffffffu, c1 && !a1));
      // re-queued entries: consumed, still alive, not the one being selected
      const bool q0 = c0 && f0 != 0ull && lane != sel_pos;
      const bool q1 = c1 && f1 != 0ull && lane + 32 != sel_pos;
      const unsigned qb0 = __ballot_sync(0xffffffffu, q0), qb1 = __ballot_sync(0xffffffffu, q1);
      const int n_new = __popc(qb0) + __popc(qb1);
      // every element looked at must provably precede all excluded candidates
      const int last = stopped ? p : chunk_n - 1;
      if (lane == 0) {
        if (!(qkey_score(sm.c_key[last]) > excl_max)) sm.fail = 3;
        sm.stop_p = p; sm.sel_pos = sel_pos; sm.sel_is_fresh = fresh_wins ? 1 : 0;
        sm.pa = pa; sm.pb = pbv; sm.n_new = n_new; sm.chunk_n = chunk_n;
      }
      // sorted list of the re-queued keys (rank by counting; keys are unique)
      if (q0) {
        int r = 0;
        for (int t = 0; t < pe; ++t) {
          const unsigned long long o = sm.c_fresh[t];
          if (t != sel_pos && o > f0) ++r;
        }
        sm.n_key[r] = f0;
      }
      if (q1) {
        int r = 0;
        for (int t = 0; t < pe; ++t) {
          const unsigned long long o = sm.c_fresh[t];
          if (t != sel_pos && o > f1) ++r;
        }
        sm.n_key[r] = f1;
      }
    }
    __syncthreads();
    if (sm.fail) break;
    // -- commit: B <- merge(B[pb..), re-queued), A pointer, selection --
    {
      const int pb = sm.pb, n_new = sm.n_new, sel_pos = sm.sel_pos;
      const int nb_keep = nb - pb;
      if (nb_keep + n_new > kBCapB) {
        if (tid == 0) sm.fail = 4;
        __syncthreads();
        break;
      }
      // read phase (old B), positions computed by binary search in the other list
      unsigned long long keep_key[kBCapB / kBT];
      unsigned short keep_begin[kBCapB / kBT];
      int keep_pos[kBCapB / kBT];
#pragma unroll
      for (int u = 0; u < kBCapB / kBT; ++u) {
        const int i = pb + tid + u * kBT;
        keep_pos[u] = -1;
        if (i < nb) {
          keep_key[u] = sm.b_key[i];
          keep_begin[u] = sm.b_begin[i];
          keep_pos[u] = (i - pb) + count_greater(sm.n_key, n_new, keep_key[u]);
        }
      }
      int new_pos = -1;
      unsigned long long new_key = 0ull;
      if (tid < n_new) {
        new_key = sm.n_key[tid];
        new_pos = tid + count_greater(sm.b_key + pb, nb_keep, new_key);
      }
      float4 sbox = make_float4(0.f, 0.f, 0.f, 0.f);
      int sidx = 0;
      float sscore = 0.f;
      if (tid == 0 && sel_pos >= 0) {
        const unsigned long long key = sm.c_key[sel_pos];
        sidx = qkey_idx(key);
        sscore = sm.sel_is_fresh ? sm.c_u[sel_pos] : qkey_score(key);
        sbox = bx[sidx];
      }
      __syncthreads();
      // write phase
#pragma unroll
      for (int u = 0; u < kBCapB / kBT; ++u) {
        if (keep_pos[u] >= 0) {
          sm.b_key[keep_pos[u]] = keep_key[u];
          sm.b_begin[keep_pos[u]] = keep_begin[u];
        }
      }
      if (new_pos >= 0) {
        sm.b_key[new_pos] = new_key;
        sm.b_begin[new_pos] = static_cast<unsigned short>(m);   // up to date with all m boxes
      }
      if (tid == 0) {
        sm.nb = nb_keep + n_new;
        sm.ptr = ptr + sm.pa;
        if (sel_pos >= 0) {
          sm.sel_box[m] = sbox;
          sm.sel_idx[m] = sidx;
          sm.sel_score[m] = sscore;
          sm.m = m + 1;
        }
      }
    }
    __syncthreads();
  }
  __syncthreads();
  if (sm.fail) {
    if (tid == 0) need_full[n] = sm.fail;  // reason (1 ties, 2 exhausted, 3 bound, 4 B overflow)
    return;
  }
  if (tid == 0) need_full[n] = 0;
  const int nsel = sm.m;
  const float scale_img = image_scales ? image_scales[n] : 1.f;
  for (int r = tid; r < max_out; r += kBT) {
    const int idx = r < nsel ? sm.sel_idx[r] : 0;
    const float score = r < nsel ? sm.sel_score[r] : 0.f;
    const float4 b = bx[idx];
    float* d = detections + (static_cast<size_t>(n) * max_out + r) * 7;
    d[0] = static_cast<float>(image_id_base + n);
    d[1] = __fmul_rn(fminf(fmaxf(b.x, 0.f), clip_h), scale_img);
    d[2] = __fmul_rn(fminf(fmaxf(b.y, 0.f), clip_w), scale_img);
    d[3] = __fmul_rn(fminf(fmaxf(b.z, 0.f), clip_h), scale_img);
    d[4] = __fmul_rn(fminf(fmaxf(b.w, 0.f), clip_w), scale_img);
    d[5] = score;
    d[6] = static_cast<float>(classes[static_cast<size_t>(n) * k + idx] + 1);
    sel_index[static_cast<size_t>(n) * max_out + r] = idx;
  }
  if (tid == 0) valid[n] = nsel;
}

}  // namespace edet

extern "C" int edet_pre_nms(const edet_half* const* h_cls, const edet_half* const* h_box,
                            const int* h_level_hw, int levels, int ld_cls, int ld_box,
                            int num_anchors, int num_classes, const float* anchors, float* boxes,
                            float* scores, int32_t* classes, int n, edet_stream_t stream) {
  using namespace edet;
  // h_cls == NULL: boxes only (scores / classes come from edet_class_argmax)
  EDET_CHECK_ARG(h_box && h_level_hw && anchors && boxes && (!h_cls || (scores && classes)),
                 "pre_nms: null pointer");
  EDET_CHECK_ARG(levels >= 1 && levels <= kPreMaxLevels, "pre_nms: 1..8 levels");
  EDET_CHECK_ARG(ld_cls % 8 == 0 && ld_cls >= num_anchors * num_classes && ld_box % 4 == 0 &&
                     ld_box >= num_anchors * 4,
                 "pre_nms: bad leading dims (ld_cls=%d ld_box=%d)", ld_cls, ld_box);
  EDET_CHECK_ARG(kPrePix * num_anchors <= kPreThreads, "pre_nms: too many anchors per location");
  PreParams p;
  p.levels = levels; p.ld_cls = ld_cls; p.ld_box = ld_box;
  p.num_anchors = num_anchors; p.num_classes = num_classes;
  int blocks = 0, anchors_total = 0;
  for (int l = 0; l < levels; ++l) {
    PreLevel& lv = p.lv[l];
    lv.cls = h_cls ? reinterpret_cast<const __half*>(h_cls[l]) : nullptr;
    lv.box = reinterpret_cast<const __half*>(h_box[l]);
    EDET_CHECK_ARG((lv.cls || !h_cls) && lv.box, "pre_nms: level %d pointer is null", l);
    lv.pixels = h_level_hw[2 * l] * h_level_hw[2 * l + 1];
    lv.block_begin = blocks;
    lv.anchor_begin = anchors_total;
    blocks += ceil_div(lv.pixels, kPrePix);
    anchors_total += lv.pixels * num_anchors;
  }
  p.total_anchors = anchors_total;
  const size_t smem = h_cls ? static_cast<size_t>(kPrePix) * ld_cls * sizeof(__half) : 0;
  EDET_CHECK_ARG(smem <= 96 * 1024, "pre_nms: ld_cls too large");
  if (smem > 48 * 1024)
    EDET_CHECK_CUDA(cudaFuncSetAttribute(pre_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem)));
  EDET_CHECK_CUDA(launch_pdl(pre_nms_kernel, dim3(blocks, n), dim3(kPreThreads), smem,
                             as_stream(stream), p, anchors, boxes, scores, classes));
  return EDET_OK;
}

extern "C" size_t edet_nms_work_bytes(int n, int k) {
  return static_cast<size_t>(n) * k * (sizeof(float) + sizeof(int32_t)) + static_cast<size_t>(n) * sizeof(int32_t);
}

extern "C" int edet_nms_v5(const float* boxes, const float* scores, const int32_t* classes,
                           const float* image_scales, int image_id_base, int n, int k,
                           int max_output_size, float iou_threshold, float score_threshold,
                           float soft_nms_sigma, float clip_h, float clip_w, float* detections,
                           int32_t* sel_index, int32_t* valid, void* work, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(boxes && scores && classes && detections && sel_index && valid && work,
                 "nms_v5: null pointer");
  EDET_CHECK_ARG(n > 0 && k > 0, "nms_v5: bad shape");
  EDET_CHECK_ARG(max_output_size > 0 && max_output_size <= kNmsMaxOut,
                 "nms_v5: max_output_size must be in 1..%d", kNmsMaxOut);
  float* ws = reinterpret_cast<float*>(work);
  int32_t* wb = reinterpret_cast<int32_t*>(ws + static_cast<size_t>(n) * k);
  int32_t* need_full = wb + static_cast<size_t>(n) * k;
  static int configured[kMaxDevices];
  if (int rc = ensure_dynamic_smem(nms_v5_fast_kernel, static_cast<int>(sizeof(BatchSmem)), configured)) return rc;
  // fast path (top candidates in shared memory, exactness proven per image) ...
  nms_v5_fast_kernel<<<n, kBT, sizeof(BatchSmem), as_stream(stream)>>>(
      boxes, scores, classes, image_scales, image_id_base, k, max_output_size, iou_threshold,
      score_threshold, soft_nms_sigma, clip_h, clip_w, detections, sel_index, valid, need_full);
  EDET_CHECK_LAUNCH();
  // ... and the full-queue kernel, which returns immediately for images the fast path settled.
  nms_v5_kernel<<<n, kNmsThreads, 0, as_stream(stream)>>>(
      boxes, scores, classes, image_scales, image_id_base, k, max_output_size, iou_threshold,
      score_threshold, soft_nms_sigma, clip_h, clip_w, detections, sel_index, valid, ws, wb,
      need_full);
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}
