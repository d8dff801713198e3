// Softmax + top-k of classifier logits: what a classification user reads (infer.py's top-1, the
// TF-Hub notebook's top-5 with probabilities: tf.nn.softmax then tf.math.top_k) without copying
// the [N, num_classes] logits back.  One CTA per image; the selection runs on the logits, so the
// rounding of the probabilities cannot reorder classes.
#include "common.cuh"

namespace edet {

constexpr int kTopkThreads = 256;
constexpr int kTopkWarps = kTopkThreads / 32;
constexpr int kMaxTopK = 32;

// Total order of (logit descending, class ascending) as one 64-bit key, larger = earlier; 0 is
// below every key of a real logit (-NaN aside).  -0 and +0 compare equal, as top_k compares them,
// so both map to the key of +0 and tie on the class index.
__device__ __forceinline__ unsigned long long topk_key(float v, int idx) {
  unsigned u = v == 0.f ? 0u : __float_as_uint(v);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return (static_cast<unsigned long long>(u) << 32) | (0xffffffffu - static_cast<unsigned>(idx));
}

// Thread t owns the classes t, t + 256, t + 512, ...
__device__ __forceinline__ unsigned long long best_below(const float* row, int c,
                                                        unsigned long long bound) {
  unsigned long long best = 0;
  for (int i = threadIdx.x; i < c; i += kTopkThreads) {
    const unsigned long long key = topk_key(__ldg(row + i), i);
    if (key < bound && key > best) best = key;
  }
  return best;
}

__global__ void __launch_bounds__(kTopkThreads)
softmax_topk_kernel(const float* __restrict__ logits, int c, int k, float* __restrict__ probs,
                    int32_t* __restrict__ classes) {
  __shared__ float red[kTopkWarps];
  __shared__ unsigned long long kred[2][kTopkWarps];
  __shared__ unsigned long long sel[kMaxTopK];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* row = logits + static_cast<size_t>(blockIdx.x) * c;

  float m = -INFINITY;
  for (int i = threadIdx.x; i < c; i += kTopkThreads) m = fmaxf(m, __ldg(row + i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < kTopkWarps; ++w) m = fmaxf(m, red[w]);
  __syncthreads();                                  // red is reused for the sum

  // sum of exp(l - max): a thread's classes in ascending order, an xor-shuffle tree over the warp,
  // then the 8 warps pairwise -- an order fixed by c alone
  float s = 0.f;
  for (int i = threadIdx.x; i < c; i += kTopkThreads) s = __fadd_rn(s, expf(__fsub_rn(__ldg(row + i), m)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  if (lane == 0) red[warp] = s;

  // top-k: each thread holds its best key below the last one it gave up; per round the block
  // maximum is selected and only its owner looks for its next candidate
  unsigned long long cand = best_below(row, c, ~0ull);
  for (int r = 0; r < k; ++r) {
    unsigned long long b = cand;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long v = __shfl_xor_sync(0xffffffffu, b, o);
      b = v > b ? v : b;
    }
    if (lane == 0) kred[r & 1][warp] = b;
    __syncthreads();
    b = kred[r & 1][0];
#pragma unroll
    for (int w = 1; w < kTopkWarps; ++w) b = kred[r & 1][w] > b ? kred[r & 1][w] : b;
    if (threadIdx.x == 0) sel[r] = b;
    if (cand == b) cand = best_below(row, c, b);
  }
  __syncthreads();
  if (threadIdx.x < k) {
    const float sum = __fadd_rn(__fadd_rn(__fadd_rn(red[0], red[1]), __fadd_rn(red[2], red[3])),
                                __fadd_rn(__fadd_rn(red[4], red[5]), __fadd_rn(red[6], red[7])));
    const int idx = static_cast<int>(0xffffffffu - static_cast<unsigned>(sel[threadIdx.x]));
    const size_t o = static_cast<size_t>(blockIdx.x) * k + threadIdx.x;
    probs[o] = __fdiv_rn(expf(__fsub_rn(__ldg(row + idx), m)), sum);
    classes[o] = idx;
  }
}
static_assert(kTopkWarps == 8, "the final sum is written for 8 warps");

}  // namespace edet

extern "C" int edet_softmax_topk(const float* logits, int n, int num_classes, int k, float* probs,
                                 int32_t* classes, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(n > 0 && num_classes > 0, "softmax_topk: bad shape (n=%d num_classes=%d)", n,
                 num_classes);
  EDET_CHECK_ARG(k >= 1 && k <= num_classes && k <= kMaxTopK,
                 "softmax_topk: k=%d must be in [1, min(num_classes=%d, %d)]", k, num_classes,
                 kMaxTopK);
  EDET_CHECK_ARG(logits && probs && classes, "softmax_topk: null pointer");
  EDET_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(probs) |
                  reinterpret_cast<uintptr_t>(classes)) % 4 == 0,
                 "softmax_topk: pointers must be 4-byte aligned");
  softmax_topk_kernel<<<n, kTopkThreads, 0, as_stream(stream)>>>(logits, num_classes, k, probs,
                                                                 classes);
  EDET_CHECK_LAUNCH();
  return EDET_OK;
}
