// Shared device/host helpers for the automl_b200 kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/automl_b200.h"

namespace edet {

void set_error(const char* fmt, ...);

#define EDET_CHECK_ARG(cond, ...)            \
  do {                                       \
    if (!(cond)) {                           \
      ::edet::set_error(__VA_ARGS__);        \
      return EDET_ERR_INVALID;               \
    }                                        \
  } while (0)

#define EDET_CHECK_CUDA(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::edet::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                        __FILE__, __LINE__);                                         \
      return EDET_ERR_CUDA;                                                          \
    }                                                                                \
  } while (0)

#define EDET_CHECK_LAUNCH() EDET_CHECK_CUDA(cudaGetLastError())

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// TensorFlow 'SAME' padding before the first element (extra padding goes after the last).
__host__ __device__ inline int same_pad_before(int in, int k, int s) {
  int out = (in + s - 1) / s;
  int total = (out - 1) * s + k - in;
  if (total < 0) total = 0;
  return total / 2;
}

// Activations (utils.py:36-53 of the reference). Computed in fp32.
// swish: x * sigmoid(x) with ex2.approx / rcp.approx (2 MUFU ops, ~1e-7 relative).
__device__ __forceinline__ float act_swish(float x) {
  return __fdividef(x, 1.0f + __expf(-x));
}
__device__ __forceinline__ float act_sigmoid(float x) {
  return __fdividef(1.0f, 1.0f + __expf(-x));
}
template <int ACT>
__device__ __forceinline__ float apply_act_t(float x) {
  if (ACT == EDET_ACT_SWISH) return act_swish(x);
  if (ACT == EDET_ACT_RELU) return fmaxf(x, 0.f);
  if (ACT == EDET_ACT_RELU6) return fminf(fmaxf(x, 0.f), 6.f);
  if (ACT == EDET_ACT_HSWISH) return x * fminf(fmaxf(x + 3.f, 0.f), 6.f) * (1.f / 6.f);
  if (ACT == EDET_ACT_SIGMOID) return act_sigmoid(x);
  return x;
}
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case EDET_ACT_SWISH: return act_swish(x);
    case EDET_ACT_RELU: return fmaxf(x, 0.f);
    case EDET_ACT_RELU6: return fminf(fmaxf(x, 0.f), 6.f);
    case EDET_ACT_HSWISH: return x * fminf(fmaxf(x + 3.f, 0.f), 6.f) * (1.f / 6.f);
    case EDET_ACT_SIGMOID: return act_sigmoid(x);
    default: return x;
  }
}

// Component-wise fp32 pair arithmetic, round to nearest.  sm_90 has no packed fp32 pipe, so each
// is two scalar instructions; the results are those of the scalar ops.
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// Activation on a pair of values; the two MUFU ops per element dominate the swish epilogues.
template <int ACT>
__device__ __forceinline__ float2 apply_act2(float2 x) {
  if (ACT == EDET_ACT_SWISH) {
    const float2 t = fmul2_rn(x, make_float2(-1.4426950408889634f, -1.4426950408889634f));
    float2 e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(t.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(t.y));
    const float2 d = fadd2_rn(e, make_float2(1.f, 1.f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r.x) : "f"(d.x));   // rcp(inf) = 0: x -> -0 for x << 0
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r.y) : "f"(d.y));
    return fmul2_rn(x, r);
  }
  return make_float2(apply_act_t<ACT>(x.x), apply_act_t<ACT>(x.y));
}

// Activation on two pairs (4 values).  For swish the four reciprocals of 1 + e^-x share ONE
// MUFU.RCP (Montgomery's batch inversion: 1/d0 = d2 * (d1*d3) / (d0*d1*d2*d3) ...), so a swish
// costs 1.25 MUFU ops per element instead of 2 -- the MUFU pipe (16 lanes/clk/SM) is what bounds
// the swish epilogues of this network.  x is clamped at -20.79 (e^-x <= 2^30, so the product of
// four denominators stays finite); below that swish(x) > -2e-8, which is 0 in fp16 either way.
// Relative error ~6 fp32 ulp.
template <int ACT>
__device__ __forceinline__ void apply_act4(float2& a, float2& b) {
  if (ACT == EDET_ACT_SWISH) {
    const float kLo = -20.794415f;   // -30 * ln 2
    a.x = fmaxf(a.x, kLo); a.y = fmaxf(a.y, kLo);
    b.x = fmaxf(b.x, kLo); b.y = fmaxf(b.y, kLo);
    const float2 k = make_float2(-1.4426950408889634f, -1.4426950408889634f);
    const float2 ta = fmul2_rn(a, k), tb = fmul2_rn(b, k);
    float2 ea, eb;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ea.x) : "f"(ta.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ea.y) : "f"(ta.y));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(eb.x) : "f"(tb.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(eb.y) : "f"(tb.y));
    const float2 one = make_float2(1.f, 1.f);
    const float2 da = fadd2_rn(ea, one), db = fadd2_rn(eb, one);
    const float2 p = fmul2_rn(da, db);          // (d0*d2, d1*d3)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(p.x * p.y));
    const float2 q = make_float2(p.y * r, p.x * r);   // (1/(d0*d2), 1/(d1*d3))
    a = fmul2_rn(a, fmul2_rn(db, q));             // x * 1/d0, x * 1/d1
    b = fmul2_rn(b, fmul2_rn(da, q));
    return;
  }
  a = apply_act2<ACT>(a);
  b = apply_act2<ACT>(b);
}

// Anchor box decode (tf2/anchors.py:30-58), float32, no FMA contraction: `bv` = the four fp16 box
// logits (ty, tx, th, tw) of one anchor, `an` = its anchor box (ymin, xmin, ymax, xmax).
__device__ __forceinline__ float4 decode_box(const uint2& bv, const float4& an) {
  const float2 t01 = __half22float2(*reinterpret_cast<const __half2*>(&bv.x));
  const float2 t23 = __half22float2(*reinterpret_cast<const __half2*>(&bv.y));
  const float ty = t01.x, tx = t01.y, th = t23.x, tw = t23.y;
  const float ycenter_a = __fmul_rn(__fadd_rn(an.x, an.z), 0.5f);
  const float xcenter_a = __fmul_rn(__fadd_rn(an.y, an.w), 0.5f);
  const float ha = __fsub_rn(an.z, an.x), wa = __fsub_rn(an.w, an.y);
  const float w = __fmul_rn(expf(tw), wa), h = __fmul_rn(expf(th), ha);
  const float yc = __fadd_rn(__fmul_rn(ty, ha), ycenter_a);
  const float xc = __fadd_rn(__fmul_rn(tx, wa), xcenter_a);
  const float hh = __fmul_rn(h, 0.5f), hw = __fmul_rn(w, 0.5f);
  return make_float4(__fsub_rn(yc, hh), __fsub_rn(xc, hw), __fadd_rn(yc, hh), __fadd_rn(xc, hw));
}

// 8 halves <-> 8 floats through one 128-bit register quad.
struct alignas(16) Half8 {
  __half2 h[4];
};
__device__ __forceinline__ void half8_to_float(const uint4& v, float* f) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 float_to_half8(const float* f) {
  uint4 v;
  __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

inline cudaStream_t as_stream(edet_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- per-device state (capi.cu) -------------------------------------------------------------
// Everything the launch wrappers cache about "the device" is keyed by the CURRENT device ordinal:
// one process may drive several engines on several GPUs (Engine(device=...)), so a process-wide
// static would hand cuda:1 the SM count, scheduler-counter address and shared-memory opt-in
// state of cuda:0.
// Library options (edet_set_option): implementation switches for A/B measurements.
int option_dw_impl();   // 0 auto (tiled kernel where eligible), 1 register kernel only, 2 = 0
int option_stem_impl(); // 0 auto (tensor-core stem), 1 CUDA-core stem kernel
int option_sepconv_impl();  // 0 auto (TMA-staged input for c <= 64, one buffer), 1 loads straight from global, 2 TMA double buffer
int option_pw_teams();  // 0 auto, 2 / 3 = force that many epilogue teams in pointwise_tc
int option_pw_smem_kb();     // 0 auto, else the shared-memory budget (KiB) of a pointwise_tc CTA
int option_persist_slack();  // CTAs a persistent kernel leaves out of its grid (default 0)
int option_max_ctas();       // 0 (default): no cap, else the exact grid of a persistent kernel
int option_pw_share_w();     // 0 auto, 1 = pointwise_tc keeps 64-row tiles where W streams
constexpr int kMaxDevices = 64;
int current_device();                 // ordinal of the current device, -1 (+ error text) on failure
int device_sm_count();                // multiprocessor count of the current device, 0 on failure
// Grid of every persistent kernel: max(1, min(total_work, ctas_per_sm * sm_count - persist_slack,
// max_ctas or unbounded)).  Never more CTAs than work items: a CTA whose first item does not exist
// would never claim one, and the dynamic tile scheduler counts on every CTA retiring after a
// claim.  0 (+ error text) when the SM count cannot be read.
int persistent_grid(int total_work, int ctas_per_sm);
// Opt a kernel into `bytes` of dynamic shared memory once per (kernel instantiation, device).
// `done` is the caller's zero-initialised static int[kMaxDevices] (one per instantiation), so no
// CUDA API call is made on the steady-state / graph-capture path.
template <typename F>
inline int ensure_dynamic_smem(F kernel, int bytes, int* done) {
  const int dev = current_device();
  if (dev < 0) return EDET_ERR_CUDA;
  if (done[dev] >= bytes) return EDET_OK;
  EDET_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done[dev] = bytes;
  return EDET_OK;
}

// Programmatic dependent launch (PDL): every kernel of the path is launched with the
// programmatic-stream-serialization attribute and signals `launch_dependents` as its first
// instruction, so the NEXT kernel's CTAs may be scheduled and run their prologue while the tail of
// the previous kernel drains -- the step is ~220 short launches.  Before its own `pdl_wait_prior()`
// a kernel may only
//  - set up shared memory and mbarriers and prefetch tensor-map descriptors;
//  - read CONSTANTS: buffers the host wrote before the first launch and no kernel ever writes
//    (weights, biases, depthwise taps, fusion weights), into registers or shared memory.
// It must not read anything a kernel writes (activations, SE sums, SE-scaled or per-image weights:
// the previous kernel may still be writing them) and must not write global memory at all (the
// previous kernel may still be reading it).  The wait returns only when every prior grid has
// completed and flushed, so after it both are safe.  DESIGN.md section 4 lists each family's
// pre-wait reads; a caller must never pass a device-computed buffer as one of them.
// tests/test_gpu_pdl_chains.py and tests/test_pdl_sass.py check this rule.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait_prior() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace edet
