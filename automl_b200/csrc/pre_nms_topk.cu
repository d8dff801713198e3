// Pre-NMS with `max_nms_inputs > 0`: the top-k (anchor, class) logits of every image, then
// sigmoid + anchor box decode of the selected pairs.
// Replaces tf2/postprocess.py:88-102 (topk_class_boxes: reshape to [N, anchors*classes],
// tf.math.top_k, index // num_classes, index % num_classes, gather_nd) inside pre_nms (:119-156)
// and tf2/anchors.py:30-58 (decode_box_outputs).  tf.math.top_k(sorted=False) defines the SET
// (on ties the lower flat index is kept), not the order; the output here is sorted by
// (logit descending, flat index ascending), which is what the oracle restatement returns.
//
// One CTA per image (the work is one streaming pass per radix digit over A*C fp16 logits,
// 8.8 MB for D0; all images run concurrently):
//   1-2. two-pass radix select on the order-preserving 16-bit key of the fp16 logit -> threshold
//        key T, G = #(key > T), r = k - G ties to keep
//   3.   ordered compaction: key > T always; key == T only the first r in flat-index order
//        (block prefix sum over the tie counts of each 8192-element chunk)
//   4.   bitonic sort of the k 64-bit (key, ~flat) entries in shared memory
//   5.   score = sigmoid(logit), box = decode(box logits of the anchor, anchor box)
// Algorithmic HBM bytes per launch: 3 passes * 2*N*total_anchors*ld_cls + 32*N*k.
#include "common.cuh"

namespace edet {
namespace topk {

constexpr int kThreads = 1024;
constexpr int kMaxLevels = 8;
constexpr int kMaxK = 8192;

struct Level {
  const __half* cls;
  const __half* box;
  int pixels;        // h * w
  int anchor_begin;  // first flattened anchor of this level
};
struct Params {
  Level lv[kMaxLevels];
  int levels, ld_cls, ld_box, num_anchors, num_classes, total_anchors, k;
};

struct Smem {
  unsigned long long keys[kMaxK];
  unsigned hist[256];
  int warp_sums[kThreads / 32];
  int count;          // entries appended so far
  int tie_base;       // ties seen in the chunks already processed
  unsigned sel_hi, sel_key;
  int sel_rank;
};

// -0 takes +0's key: tf.math.top_k compares the logits as floats, where the two are equal (a tie
// that keeps the lower flat index)
__device__ __forceinline__ unsigned key16(unsigned short h) {
  h = h == 0x8000u ? static_cast<unsigned short>(0) : h;
  return (h & 0x8000u) ? (~static_cast<unsigned>(h) & 0xffffu) : (static_cast<unsigned>(h) | 0x8000u);
}
__device__ __forceinline__ unsigned short unkey16(unsigned k) {
  return static_cast<unsigned short>((k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu));
}

// Calls fn(key16, flat_index) for the 8 elements of 16-byte vector `v` of image n (flat order
// is level-major, then pixel, then column < A*C); returns false when v is past the end.
template <typename F>
__device__ __forceinline__ void for_vec(const Params& p, int n, long long v, F fn) {
  const int vpr = p.ld_cls >> 3;     // vectors per pixel row
  const int ac = p.num_anchors * p.num_classes;
  long long base = 0;
  for (int l = 0; l < p.levels; ++l) {
    const long long nv = static_cast<long long>(p.lv[l].pixels) * vpr;
    if (v < base + nv) {
      const long long lvv = v - base;
      const int pix = static_cast<int>(lvv / vpr), vc = static_cast<int>(lvv - static_cast<long long>(pix) * vpr) * 8;
      if (vc >= ac) return;   // all-padding vector
      const uint4 raw = ldg_nc_v4(reinterpret_cast<const uint4*>(
          p.lv[l].cls + (static_cast<size_t>(n) * p.lv[l].pixels + pix) * p.ld_cls + vc));
      const unsigned short* h = reinterpret_cast<const unsigned short*>(&raw);
      const unsigned flat0 = static_cast<unsigned>(
          (static_cast<long long>(p.lv[l].anchor_begin) + static_cast<long long>(pix) * p.num_anchors) *
              p.num_classes + vc);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (vc + e < ac) fn(key16(h[e]), flat0 + e);
      return;
    }
    base += nv;
  }
}

__global__ void __launch_bounds__(kThreads)
pre_nms_topk_kernel(const Params p, const float* __restrict__ anchors, float* __restrict__ boxes,
                    float* __restrict__ scores, int32_t* __restrict__ classes,
                    int32_t* __restrict__ indices) {
  extern __shared__ __align__(16) uint8_t topk_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(topk_raw);
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long total_vec = 0;
  for (int l = 0; l < p.levels; ++l) total_vec += static_cast<long long>(p.lv[l].pixels) * (p.ld_cls >> 3);

  // ---- 1-2. radix select: high byte, then low byte of the 16-bit key ----
  if (tid == 0) { sm.sel_hi = 0; sm.sel_rank = p.k; }
  for (int pass = 0; pass < 2; ++pass) {
    for (int i = tid; i < 256; i += kThreads) sm.hist[i] = 0u;
    __syncthreads();
    const unsigned hi = sm.sel_hi;
    for (long long v = tid; v < total_vec; v += kThreads) {
      for_vec(p, n, v, [&](unsigned key, unsigned) {
        // the logits of a detector sit in a handful of bins: aggregate equal bins across the
        // warp so that a hot bin costs one shared-memory atomic per warp, not 32
        if (pass == 0 || (key >> 8) == hi) {
          const unsigned bin = pass == 0 ? (key >> 8) : (key & 0xffu);
          const unsigned peers = __match_any_sync(__activemask(), bin);
          if ((peers & (0u - peers)) == (1u << lane)) atomicAdd(&sm.hist[bin], __popc(peers));
        }
      });
    }
    __syncthreads();
    if (tid == 0) {
      int rank = sm.sel_rank, d = 255;
      for (; d > 0; --d) {
        const int cnt = static_cast<int>(sm.hist[d]);
        if (rank <= cnt) break;
        rank -= cnt;
      }
      sm.sel_rank = rank;          // after pass 1: ties (key == T) to keep
      if (pass == 0) sm.sel_hi = static_cast<unsigned>(d);
      else sm.sel_key = (sm.sel_hi << 8) | static_cast<unsigned>(d);
    }
    __syncthreads();
  }
  const unsigned T = sm.sel_key;
  const int keep_ties = sm.sel_rank;
  // ---- 3. ordered compaction ----
  if (tid == 0) { sm.count = 0; sm.tie_base = 0; }
  for (int i = tid; i < kMaxK; i += kThreads) sm.keys[i] = 0ull;
  __syncthreads();
  for (long long v0 = 0; v0 < total_vec; v0 += kThreads) {
    const long long v = v0 + tid;
    int my_ties = 0;
    unsigned tie_flat[8];
    if (v < total_vec) {
      for_vec(p, n, v, [&](unsigned key, unsigned flat) {
        if (key > T) {
          const int pos = atomicAdd(&sm.count, 1);
          if (pos < kMaxK) sm.keys[pos] = (static_cast<unsigned long long>(key) << 32) | (0xffffffffu - flat);
        } else if (key == T) {
          tie_flat[my_ties++] = flat;
        }
      });
    }
    const int base = sm.tie_base;
    if (base < keep_ties && __syncthreads_or(my_ties > 0)) {
      // exclusive prefix of my_ties over the block (flat order == thread order inside a chunk)
      int incl = my_ties;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      if (lane == 31) sm.warp_sums[warp] = incl;
      __syncthreads();
      int woff = 0;
      for (int w = 0; w < warp; ++w) woff += sm.warp_sums[w];
      int rank = base + woff + incl - my_ties;
      for (int e = 0; e < my_ties; ++e, ++rank) {
        if (rank < keep_ties) {
          const int pos = atomicAdd(&sm.count, 1);
          if (pos < kMaxK) sm.keys[pos] = (static_cast<unsigned long long>(T) << 32) | (0xffffffffu - tie_flat[e]);
        }
      }
      __syncthreads();
      if (tid == kThreads - 1) sm.tie_base = base + woff + incl;
      __syncthreads();
    } else {
      __syncthreads();   // keeps sm.tie_base reads and writes of consecutive chunks ordered
    }
  }
  __syncthreads();
  // ---- 4. sort descending: larger logit first, then smaller flat index ----
  for (int size = 2; size <= kMaxK; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < kMaxK / 2; i += kThreads) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long a = sm.keys[lo], b = sm.keys[hi];
        if ((a < b) == desc) { sm.keys[lo] = b; sm.keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  // ---- 5. outputs ----
  for (int j = tid; j < p.k; j += kThreads) {
    const unsigned long long e = sm.keys[j];
    const unsigned flat = 0xffffffffu - static_cast<unsigned>(e & 0xffffffffu);
    const int anchor = static_cast<int>(flat / p.num_classes);
    const int cls = static_cast<int>(flat - static_cast<unsigned>(anchor) * p.num_classes);
    int l = 0;
    while (l + 1 < p.levels && anchor >= p.lv[l + 1].anchor_begin) ++l;
    const int rel = anchor - p.lv[l].anchor_begin;
    const int pix = rel / p.num_anchors, a = rel - pix * p.num_anchors;
    const unsigned short hb = unkey16(static_cast<unsigned>(e >> 32));
    const float logit = __half2float(*reinterpret_cast<const __half*>(&hb));
    const size_t o = static_cast<size_t>(n) * p.k + j;
    scores[o] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-logit)));
    classes[o] = cls;
    indices[o] = anchor;
    const uint2 bv = __ldg(reinterpret_cast<const uint2*>(
        p.lv[l].box + (static_cast<size_t>(n) * p.lv[l].pixels + pix) * p.ld_box + a * 4));
    reinterpret_cast<float4*>(boxes)[o] =
        decode_box(bv, __ldg(reinterpret_cast<const float4*>(anchors) + anchor));
  }
}

}  // namespace topk
}  // namespace edet

extern "C" int edet_pre_nms_topk(const edet_half* const* h_cls, const edet_half* const* h_box,
                                 const int* h_level_hw, int levels, int ld_cls, int ld_box,
                                 int num_anchors, int num_classes, const float* anchors,
                                 int max_nms_inputs, float* boxes, float* scores,
                                 int32_t* classes, int32_t* indices, int n, edet_stream_t stream) {
  using namespace edet;
  using namespace edet::topk;
  EDET_CHECK_ARG(h_cls && h_box && h_level_hw && anchors && boxes && scores && classes && indices,
                 "pre_nms_topk: null pointer");
  EDET_CHECK_ARG(levels >= 1 && levels <= kMaxLevels, "pre_nms_topk: 1..8 levels");
  EDET_CHECK_ARG(ld_cls % 8 == 0 && ld_cls >= num_anchors * num_classes && ld_box % 4 == 0 &&
                     ld_box >= num_anchors * 4,
                 "pre_nms_topk: bad leading dims (ld_cls=%d ld_box=%d)", ld_cls, ld_box);
  Params p;
  p.levels = levels; p.ld_cls = ld_cls; p.ld_box = ld_box;
  p.num_anchors = num_anchors; p.num_classes = num_classes; p.k = max_nms_inputs;
  long long total = 0;
  int anchors_total = 0;
  for (int l = 0; l < levels; ++l) {
    Level& lv = p.lv[l];
    lv.cls = reinterpret_cast<const __half*>(h_cls[l]);
    lv.box = reinterpret_cast<const __half*>(h_box[l]);
    EDET_CHECK_ARG(lv.cls && lv.box, "pre_nms_topk: level %d pointer is null", l);
    lv.pixels = h_level_hw[2 * l] * h_level_hw[2 * l + 1];
    lv.anchor_begin = anchors_total;
    anchors_total += lv.pixels * num_anchors;
    total += static_cast<long long>(lv.pixels) * num_anchors * num_classes;
  }
  p.total_anchors = anchors_total;
  EDET_CHECK_ARG(max_nms_inputs > 0 && max_nms_inputs <= kMaxK && max_nms_inputs <= total,
                 "pre_nms_topk: max_nms_inputs must be in 1..min(%d, anchors*classes) (got %d)", kMaxK,
                 max_nms_inputs);
  EDET_CHECK_ARG(total < 0xffffffffLL, "pre_nms_topk: too many (anchor, class) pairs");
  static int configured[kMaxDevices];
  if (int rc = ensure_dynamic_smem(pre_nms_topk_kernel, static_cast<int>(sizeof(Smem)), configured)) return rc;
  pre_nms_topk_kernel<<<n, kThreads, sizeof(Smem), as_stream(stream)>>>(p, anchors, boxes, scores,
                                                                       classes, indices);
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}
