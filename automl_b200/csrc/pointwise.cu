// edet_pointwise_conv: argument checks + dispatch (wgmma path / SIMT cross-check kernel).
#include "tc_common.cuh"

namespace edet {

// Plain CUDA-core GEMM used only to cross-check the tensor-core kernel on the device.
// 64x64 output tile per 256-thread block, 4x4 outputs per thread, K in slabs of 16.
__global__ void __launch_bounds__(256)
pointwise_simt_kernel(const __half* __restrict__ a, int lda, const __half* __restrict__ wt,
                      int wbatch, const float* __restrict__ bias,
                      const __half* __restrict__ residual, int ldr, __half* __restrict__ out,
                      int ldo, int rows, int k, int nout, int act) {
  __shared__ float sa[16][64 + 1];
  __shared__ float sw[16][64 + 1];
  const int b = blockIdx.z;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const __half* ab = a + static_cast<size_t>(b) * rows * lda;
  const __half* wb = wt + (wbatch > 1 ? static_cast<size_t>(b) * nout * k : 0);
  float acc[4][4] = {};
  for (int k0 = 0; k0 < k; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, kk = i & 15;
      const int m = m0 + r, n = n0 + r, kx = k0 + kk;
      sa[kk][r] = (m < rows && kx < k) ? __half2float(ab[static_cast<size_t>(m) * lda + kx]) : 0.f;
      sw[kk][r] = (n < nout && kx < k) ? __half2float(wb[static_cast<size_t>(n) * k + kx]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float av[4], wv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = sa[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) wv[j] = sw[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= nout) continue;
      float x = apply_act(acc[i][j] + bias[n], act);
      if (residual)
        x += __half2float(residual[(static_cast<size_t>(b) * rows + m) * ldr + n]);
      out[(static_cast<size_t>(b) * rows + m) * ldo + n] = __float2half_rn(x);
    }
  }
}

}  // namespace edet

extern "C" int edet_pointwise_conv(const edet_half* a, int lda, const edet_half* wt, int wbatch,
                                   const float* bias, const edet_half* residual, int ldr,
                                   edet_half* out, int ldo, int batch, int rows, int k, int nout,
                                   int act, int impl, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(a && wt && bias && out, "pointwise: null pointer");
  EDET_CHECK_ARG(batch > 0 && rows > 0 && k > 0 && nout > 0, "pointwise: bad shape");
  EDET_CHECK_ARG(k % 8 == 0 && lda % 8 == 0 && ldo % 8 == 0 && lda >= k && ldo >= nout,
                 "pointwise: k=%d lda=%d ldo=%d must be multiples of 8 (lda>=k, ldo>=nout=%d)", k,
                 lda, ldo, nout);
  EDET_CHECK_ARG(wbatch == 1 || wbatch == batch, "pointwise: wbatch must be 1 or batch");
  EDET_CHECK_ARG(!residual || (ldr % 8 == 0 && ldr >= nout && nout % 8 == 0),
                 "pointwise: residual needs ldr%%8==0 and nout%%8==0");
  EDET_CHECK_ARG((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(wt) |
                  reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(residual)) % 16 == 0,
                 "pointwise: pointers must be 16-byte aligned");
  cudaStream_t s = as_stream(stream);
  const __half* ha = reinterpret_cast<const __half*>(a);
  const __half* hw = reinterpret_cast<const __half*>(wt);
  const __half* hr = reinterpret_cast<const __half*>(residual);
  __half* ho = reinterpret_cast<__half*>(out);
  if (impl == EDET_PW_TCGEN05) {
    return pwtc::run(ha, lda, hw, wbatch, bias, hr, ldr, ho, ldo, batch, rows, k, nout, act, s);
  }
  if (impl == EDET_PW_SIMT) {
    dim3 grid(ceil_div(rows, 64), ceil_div(nout, 64), batch);
    pointwise_simt_kernel<<<grid, 256, 0, s>>>(ha, lda, hw, wbatch, bias, hr, ldr, ho, ldo, rows,
                                               k, nout, act);
    EDET_CHECK_LAUNCH();
    return EDET_OK;
  }
  set_error("pointwise: unknown impl %d", impl);
  return EDET_ERR_INVALID;
}

extern "C" int edet_class_argmax(const edet_half* a, int lda, const edet_half* wt_padded,
                                 const float* bias_padded, float* scores, int32_t* classes,
                                 int anchor_begin, int total_anchors, int num_anchors, int batch,
                                 int rows, int k, edet_stream_t stream) {
  using namespace edet;
  EDET_CHECK_ARG(a && wt_padded && bias_padded && scores && classes, "class_argmax: null pointer");
  EDET_CHECK_ARG(batch > 0 && rows > 0 && k > 0 && k % 8 == 0 && lda % 8 == 0 && lda >= k,
                 "class_argmax: bad shape (k=%d lda=%d)", k, lda);
  EDET_CHECK_ARG(num_anchors > 0 && anchor_begin >= 0 &&
                     anchor_begin + static_cast<long long>(rows) * num_anchors <= total_anchors,
                 "class_argmax: anchors [%d, +%d*%d) exceed %d", anchor_begin, rows, num_anchors,
                 total_anchors);
  pwtc::ArgmaxArgs am{scores, classes, anchor_begin, total_anchors, num_anchors};
  return pwtc::run(reinterpret_cast<const __half*>(a), lda, reinterpret_cast<const __half*>(wt_padded),
                   1, bias_padded, nullptr, 0, nullptr, 0, batch, rows, k,
                   num_anchors * 96, EDET_ACT_NONE, as_stream(stream), &am);
}
