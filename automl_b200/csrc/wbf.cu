// Weighted box fusion for test-time augmentation: tf2/wbf.py:19-95 (ensemble_detections) over the
// per-class NMS rows of several "models" of one image, the mirrored ones first un-mirrored as
// tf2/postprocess.py:560-573 does it.  float32 in the reference's order of operations, every step
// rounded (no FMA contraction), so the clusters are bit-identical to wbf.py run in float32.
//
// One CTA per image:
//   1. load the image's rows of every model (un-mirrored), key each row of a fused class by
//      (class, input position), and sort the keys: a stable partition of the rows by class;
//   2. one warp per class: rows in input order, each against the current cluster averages
//      (warp-wide IoU + first arg-max), joining the best cluster or starting a new one;
//   3. sort the clusters by (score descending, class, creation order) and write them.
// Both sorts are one bitonic sort of 64-bit keys in shared memory.
#include "common.cuh"

namespace edet {

constexpr int kWbfThreads = 256;
constexpr int kWbfWarps = kWbfThreads / 32;
constexpr unsigned long long kNoKey = ~0ull;

__host__ __device__ inline int wbf_pow2(int r) {
  int p = 1;
  while (p < r) p <<= 1;
  return p;
}

// Dynamic shared memory of one CTA for `r` rows (r <= EDET_WBF_MAX_ROWS).
__host__ __device__ inline size_t wbf_smem_bytes(int r) {
  return 8 * static_cast<size_t>(wbf_pow2(r)) + 4 * static_cast<size_t>(r) * 21 + 4;
}

// np.maximum / np.minimum: a NaN operand gives NaN (fmaxf / fminf would drop it).
__device__ __forceinline__ float np_max(float a, float b) { return (isnan(a) || isnan(b)) ? a + b : fmaxf(a, b); }
__device__ __forceinline__ float np_min(float a, float b) { return (isnan(a) || isnan(b)) ? a + b : fminf(a, b); }

// vectorized_iou (wbf.py:19-36) of cluster average (x11, y11, x12, y12) and row (x21, ..).
__device__ __forceinline__ float wbf_iou(float x11, float y11, float x12, float y12, float x21,
                                         float y21, float x22, float y22) {
  const float xa = np_max(x11, x21), ya = np_max(y11, y21);
  const float xb = np_min(x12, x22), yb = np_min(y12, y22);
  const float inter = __fmul_rn(np_max(__fsub_rn(xb, xa), 0.f), np_max(__fsub_rn(yb, ya), 0.f));
  const float area_a = __fmul_rn(__fsub_rn(x12, x11), __fsub_rn(y12, y11));
  const float area_b = __fmul_rn(__fsub_rn(x22, x21), __fsub_rn(y22, y21));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// np.argmax's order on (value, index): the first NaN wins, else the larger value, ties the lower
// index (+0 == -0).  True if (v, i) comes before (w, j).
__device__ __forceinline__ bool argmax_before(float v, int i, float w, int j) {
  const bool nv = isnan(v), nw = isnan(w);
  if (nv || nw) return nv && (!nw || i < j);
  return v > w || (v == w && i < j);
}

// Descending order of float32 scores as an ascending uint32; -0 and +0 are one key (Python's
// sort sees them equal).
__device__ __forceinline__ unsigned desc_key(float s) {
  const unsigned u = __float_as_uint(__fadd_rn(s, 0.f));
  const unsigned asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}

// Ascending bitonic sort of `p` (a power of two) keys by the whole CTA.
__device__ void bitonic_sort(unsigned long long* keys, int p) {
  for (int k = 2; k <= p; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < p; i += kWbfThreads) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = keys[i], b = keys[l];
          if (((i & k) == 0) == (a > b)) {
            keys[i] = b;
            keys[l] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

// The weight of a cluster's mean score, float32(min(1, count / num_models)) with the division
// in double as Python does it.
__device__ __forceinline__ float count_weight(int count, int num_models) {
  return count >= num_models ? 1.f
                             : static_cast<float>(static_cast<double>(count) / static_cast<double>(num_models));
}

__global__ void __launch_bounds__(kWbfThreads)
wbf_kernel(const float* __restrict__ det, int n, int rows, int num_models, int mirrored_mask,
           const float* __restrict__ image_scales, float width, int num_classes,
           float* __restrict__ out, int* __restrict__ counts) {
  pdl_launch_dependents();
  pdl_wait_prior();         // the rows come from the NMS launch, the scales from a copy
  extern __shared__ __align__(16) unsigned char smem[];
  const int r_all = num_models * rows;
  const int p = wbf_pow2(r_all);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);
  float* row = reinterpret_cast<float*>(keys + p);   // [7][r_all] columns of the image's rows
  int* perm = reinterpret_cast<int*>(row + 7 * r_all);      // sorted position -> row
  int* segs = perm + r_all;                                 // class segment starts (+ end)
  float* avg = reinterpret_cast<float*>(segs + r_all + 1);  // [4][r_all] cluster averages
  float* sum = avg + 4 * r_all;                             // [4][r_all] sum of x * s
  float* ssum = sum + 4 * r_all;                            // sum of s
  float* score = ssum + r_all;
  int* count = reinterpret_cast<int*>(score + r_all);
  int* first = count + r_all;                               // first member (row)
  __shared__ int s_valid, s_nseg, s_clusters;
  const int img = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { s_valid = 0; s_clusters = 0; }
  __syncthreads();

  // 1. rows (un-mirrored) and the class partition keys
  const float ow = mirrored_mask ? __fmul_rn(image_scales[img], width) : 0.f;
  for (int r = tid; r < p; r += kWbfThreads) {
    unsigned long long key = kNoKey;
    if (r < r_all) {
      const int m = r / rows, j = r - m * rows;
      const float* src = det + ((static_cast<long long>(m) * n + img) * rows + j) * 7;
      float v[7];
#pragma unroll
      for (int c = 0; c < 7; ++c) v[c] = src[c];
      if ((mirrored_mask >> m) & 1) {      // postprocess.py:560-573: x1' = ow - x2, x2' = ow - x1
        const float x1 = v[1];
        v[1] = __fsub_rn(ow, v[3]);
        v[3] = __fsub_rn(ow, x1);
      }
#pragma unroll
      for (int c = 0; c < 7; ++c) row[c * r_all + r] = v[c];
      // wbf.py:74-75: detections[:, 6] == cid for cid in range(num_classes)
      const float cls = v[6];
      if (cls >= 0.f && cls < static_cast<float>(num_classes) && cls == truncf(cls)) {
        key = (static_cast<unsigned long long>(static_cast<unsigned>(cls)) << 32) | static_cast<unsigned>(r);
        atomicAdd(&s_valid, 1);
      }
    }
    keys[r] = key;
  }
  __syncthreads();
  bitonic_sort(keys, p);
  const int valid = s_valid;
  for (int q = tid; q < valid; q += kWbfThreads) perm[q] = static_cast<int>(keys[q] & 0xffffffffu);
  if (warp == 0) {          // segment starts in order: ballot compaction
    int base = 0;
    for (int q0 = 0; q0 < valid; q0 += 32) {
      const int q = q0 + lane;
      const bool start = q < valid && (q == 0 || (keys[q] >> 32) != (keys[q - 1] >> 32));
      const unsigned b = __ballot_sync(0xffffffffu, start);
      if (start) segs[base + __popc(b & ((1u << lane) - 1))] = q;
      base += __popc(b);
    }
    if (lane == 0) {
      segs[base] = valid;
      s_nseg = base;
    }
  }
  __syncthreads();            // keys past `valid` stay kNoKey

  // 2. clusters of each class (wbf.py:80-92); cluster k of a segment lives at slot begin + k
  const int nseg = s_nseg;
  for (int sgi = warp; sgi < nseg; sgi += kWbfWarps) {
    const int b = segs[sgi], e = segs[sgi + 1];
    int nc = 0;
    for (int q = b; q < e; ++q) {
      const int r = perm[q];
      const float x1 = row[1 * r_all + r], y1 = row[2 * r_all + r];
      const float x2 = row[3 * r_all + r], y2 = row[4 * r_all + r], s = row[5 * r_all + r];
      float best = 0.f;
      int bi = 0x7fffffff;
      for (int k = lane; k < nc; k += 32) {   // find_matching_cluster (wbf.py:39-48)
        const int sl = b + k;
        const float iou = wbf_iou(avg[sl], avg[r_all + sl], avg[2 * r_all + sl], avg[3 * r_all + sl],
                                  x1, y1, x2, y2);
        if (bi == 0x7fffffff || argmax_before(iou, k, best, bi)) {
          best = iou;
          bi = k;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi != 0x7fffffff && (bi == 0x7fffffff || argmax_before(ob, oi, best, bi))) {
          best = ob;
          bi = oi;
        }
      }
      if (lane == 0) {
        // a new cluster iff no cluster or max(iou) < 0.55 (a NaN maximum joins the first NaN)
        const bool fresh = nc == 0 || best < 0.55f;
        const int sl = b + (fresh ? nc : bi);
        const float xs[4] = {x1, y1, x2, y2};
        int cnt;
        float tot;
        if (fresh) {
          first[sl] = r;
          cnt = 1;
          tot = s;
#pragma unroll
          for (int c = 0; c < 4; ++c) sum[c * r_all + sl] = __fmul_rn(xs[c], s);
        } else {
          cnt = count[sl] + 1;
          tot = __fadd_rn(ssum[sl], s);
#pragma unroll
          for (int c = 0; c < 4; ++c)
            sum[c * r_all + sl] = __fadd_rn(sum[c * r_all + sl], __fmul_rn(xs[c], s));
        }
        count[sl] = cnt;
        ssum[sl] = tot;
        // average_detections (wbf.py:51-67)
#pragma unroll
        for (int c = 0; c < 4; ++c) avg[c * r_all + sl] = __fdiv_rn(sum[c * r_all + sl], tot);
        score[sl] = __fmul_rn(__fdiv_rn(tot, static_cast<float>(cnt)), count_weight(cnt, num_models));
      }
      nc += (nc == 0 || best < 0.55f) ? 1 : 0;
      __syncwarp();
    }
    for (int k = lane; k < e - b; k += 32)
      keys[b + k] = k < nc ? (static_cast<unsigned long long>(desc_key(score[b + k])) << 32) |
                                 static_cast<unsigned>(b + k)
                           : kNoKey;
    if (lane == 0) atomicAdd(&s_clusters, nc);
  }
  __syncthreads();

  // 3. all_clusters.sort(reverse=True, key=score): stable, so ties keep class then creation order
  bitonic_sort(keys, p);
  const int nclus = s_clusters;
  float* o = out + static_cast<long long>(img) * r_all * 7;
  for (int q = tid; q < r_all; q += kWbfThreads) {
    float v[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, -1.f};   // padding row
    if (q < nclus) {
      const int sl = static_cast<int>(keys[q] & 0xffffffffu);
      const int f = first[sl];
      v[0] = row[f];
      v[1] = avg[sl];
      v[2] = avg[r_all + sl];
      v[3] = avg[2 * r_all + sl];
      v[4] = avg[3 * r_all + sl];
      v[5] = score[sl];
      v[6] = row[6 * r_all + f];
    }
#pragma unroll
    for (int c = 0; c < 7; ++c) o[static_cast<long long>(q) * 7 + c] = v[c];
  }
  if (tid == 0) counts[img] = nclus;
}

}  // namespace edet

extern "C" int edet_wbf(const float* detections, int n, int rows, int num_models,
                        int mirrored_mask, const float* image_scales, int width, int num_classes,
                        float* clusters, int32_t* num_clusters, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(detections && clusters && num_clusters, "wbf: null pointer");
  EDET_CHECK_ARG(image_scales || mirrored_mask == 0, "wbf: mirrored models need image_scales");
  EDET_CHECK_ARG(n > 0 && n <= 65535 && rows > 0 && num_models > 0 && num_models <= 30 &&
                     num_classes > 0 && width > 0,
                 "wbf: bad shape (n=%d rows=%d num_models=%d num_classes=%d width=%d)", n, rows,
                 num_models, num_classes, width);
  EDET_CHECK_ARG(static_cast<long long>(num_models) * rows <= EDET_WBF_MAX_ROWS,
                 "wbf: num_models * rows = %lld exceeds %d", static_cast<long long>(num_models) * rows,
                 EDET_WBF_MAX_ROWS);
  EDET_CHECK_ARG((mirrored_mask >> num_models) == 0 && mirrored_mask >= 0,
                 "wbf: mirrored_mask 0x%x names models past num_models=%d", mirrored_mask, num_models);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(detections) % 4 == 0 &&
                     reinterpret_cast<uintptr_t>(image_scales) % 4 == 0 &&
                     reinterpret_cast<uintptr_t>(clusters) % 4 == 0 &&
                     reinterpret_cast<uintptr_t>(num_clusters) % 4 == 0,
                 "wbf: every buffer must be 4-byte aligned");
  const int r_all = num_models * rows;
  const size_t smem = wbf_smem_bytes(r_all);
  static int done[kMaxDevices];
  const int rc = ensure_dynamic_smem(wbf_kernel, static_cast<int>(wbf_smem_bytes(EDET_WBF_MAX_ROWS)), done);
  if (rc != EDET_OK) return rc;
  EDET_CHECK_CUDA(launch_pdl(wbf_kernel, dim3(n), dim3(kWbfThreads), smem, as_stream(stream),
                             detections, n, rows, num_models, mirrored_mask, image_scales,
                             static_cast<float>(width), num_classes, clusters, num_clusters));
  return EDET_OK;
}
