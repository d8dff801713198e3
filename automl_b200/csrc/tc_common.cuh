// Shared pieces of the wgmma / TMA kernels (sm_90a): PTX wrappers, wgmma smem descriptors and
// the host-side tensor-map encoder.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace edet {
namespace pwtc {

constexpr int MMA_K = 16;

// pointwise_tc.cu: the GEMM entry point shared by edet_pointwise_conv and edet_class_argmax
struct ArgmaxArgs {
  float* scores;         // [batch][total_anchors]
  int32_t* classes;      // [batch][total_anchors]
  int anchor_begin, total_anchors, num_anchors;
};
int run(const __half* a, int lda, const __half* wt, int wbatch, const float* bias,
        const __half* residual, int ldr, __half* out, int ldo, int batch, int rows, int k, int nout,
        int act, cudaStream_t stream, const ArgmaxArgs* am = nullptr);

// ---- PTX wrappers ------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1,
                                             int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(map)),
      "r"(src), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1,
                                             int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(map)),
      "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// ---- warpgroup MMA (wgmma) ------------------------------------------------------------------
// D[64 x 16] (+)= A[64 x 16] * B[16 x 16]^T, fp16 in, fp32 accumulators in registers, both
// operands K-major in shared memory (smem descriptors below).  Issued by all 128 threads of a
// warpgroup.  Fragment of thread t (warp w = (t >> 5) & 3, lane l):
//   d[0], d[1] = row 16w + l/4,     columns 2(l%4), 2(l%4)+1
//   d[2], d[3] = row 16w + l/4 + 8, same columns
//   d[4..7]    = the same two rows, columns + 8
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void wg_mma_m64n16(float* d, uint64_t desc_a, uint64_t desc_b,
                                              uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// Makes the accumulators opaque to the compiler: after wg_wait, so that no read of them is
// scheduled before the MMAs that write them have completed.
template <int NT>
__device__ __forceinline__ void wg_fence_acc(float (&acc)[NT][8]) {
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int e = 0; e < 8; ++e) asm volatile("" : "+f"(acc[j][e])::"memory");
}
// One K-major k-block: acc[j] (+)= A[64 rows][16 * ksteps] * B[16j .. 16j+15][...]^T for j < nt.
// desc_a / desc_b address row 0 of the 64-row A block / the B tile; b_chunk = descriptor units
// (16 bytes) between 16-row B chunks = the smem row pitch in bytes.  Not waited for.
template <int NT>
__device__ __forceinline__ void wg_mma_kblock(float (&acc)[NT][8], uint64_t desc_a,
                                              uint64_t desc_b, int b_chunk, int nt, int ksteps,
                                              bool first) {
  for (int ks = 0; ks < ksteps; ++ks) {
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      // advance 16 halves = 32 bytes inside the swizzle atom: +2 in the >>4 address field
      if (j < nt)
        wg_mma_m64n16(acc[j], desc_a + static_cast<uint64_t>(ks * 2),
                      desc_b + static_cast<uint64_t>(j * b_chunk + ks * 2),
                      (first && ks == 0) ? 0u : 1u);
    }
  }
}
// Wide variants: D[64 x N] (+)= A[64 x 16] * B[N x 16]^T in ONE instruction, N = 32 / 64 / 96 / 128.  The
// fragment of d[8j .. 8j+7] is the m64n16 fragment of columns 16j .. 16j+15 (above), so a
// float[N / 16][8] accumulator means the same thing whichever width wrote it, and every output
// still sums its k16 products in the same order.  B rows follow each other at the descriptor's SBO.
__device__ __forceinline__ void wg_mma_m64n32(float* d, uint64_t desc_a, uint64_t desc_b,
                                              uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wg_mma_m64n64(float* d, uint64_t desc_a, uint64_t desc_b,
                                              uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wg_mma_m64n96(float* d, uint64_t desc_a, uint64_t desc_b,
                                              uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
      "%48, %49, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wg_mma_m64n128(float* d, uint64_t desc_a, uint64_t desc_b,
                                              uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// One K-major k-block over the whole tile: acc (+)= A[64 rows][16 * ksteps] * B[16 NT rows]^T, one
// wgmma per k-step.  The width is a template parameter: choosing it at run time around the wgmma
// puts it on a divergent path, and ptxas then serialises every wgmma of the kernel.  Not waited for.
template <int NT>
__device__ __forceinline__ void wg_mma_kblock_wide(float (&acc)[NT][8], uint64_t desc_a,
                                                   uint64_t desc_b, int ksteps, bool first) {
  static_assert(NT == 2 || NT == 4 || NT == 6 || NT == 8, "wide wgmma: N = 32, 64, 96 or 128");
  float* d = &acc[0][0];
  for (int ks = 0; ks < ksteps; ++ks) {
    const uint64_t a = desc_a + static_cast<uint64_t>(ks * 2);
    const uint64_t b = desc_b + static_cast<uint64_t>(ks * 2);
    const uint32_t accumulate = (first && ks == 0) ? 0u : 1u;
    if constexpr (NT == 2) wg_mma_m64n32(d, a, b, accumulate);
    if constexpr (NT == 4) wg_mma_m64n64(d, a, b, accumulate);
    if constexpr (NT == 6) wg_mma_m64n96(d, a, b, accumulate);
    if constexpr (NT == 8) wg_mma_m64n128(d, a, b, accumulate);
  }
}
// Named barrier over the `threads` threads of barrier `id` (1..15; 0 is __syncthreads).
__device__ __forceinline__ void named_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// K-major swizzled smem matrix descriptor (wgmma layout): start>>4 [0,14) | LBO>>4 [16,30) = 1 |
// SBO>>4 [32,46) = 8 rows * row pitch | layout [62,64): 1 = SWIZZLE_128B, 2 = 64B, 3 = 32B.
// The 64B / 32B variants (row pitch 64 / 32 bytes) are used for the thin-K layers (K <= 32 / 16)
// so that a pipeline stage only holds the bytes that exist.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, int sbo, int layout) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(sbo >> 4) << 32;
  d |= static_cast<uint64_t>(layout) << 62;
  return d;
}
// wgmma layout code of a K-major tile whose rows are `block_k` halves
inline int desc_layout_for(int block_k) { return block_k == 64 ? 1 : (block_k == 32 ? 2 : 3); }


__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- dynamic tile scheduler for single-role persistent kernels --------------------------------
// A persistent kernel that walks its tiles with a static stride assumes all its CTAs start
// together; when another stream (the NMS of the previous batch) holds some SMs, the CTAs that
// start late still own their full share of tiles and the kernel runs two waves.  Here CTA i owns
// tile i and every further tile comes from a global counter, so late CTAs simply find less (or
// no) work.  sched[0] = tiles handed out beyond the first gridDim.x, sched[1] = CTAs that are
// done; the last CTA resets both, so a slot is reusable by the next launch without a memset.
// A CTA stops claiming after its first claim >= total_tiles and then calls sched_retire once.
// sched_claim does not look at its result, so a caller can issue it ahead of other work and only
// wait for the atomic where it uses the tile.
__device__ __forceinline__ int sched_claim(unsigned* sched) {
  return static_cast<int>(gridDim.x + atomicAdd(&sched[0], 1u));
}
__device__ __forceinline__ void sched_retire(unsigned* sched) {
  __threadfence();
  if (atomicAdd(&sched[1], 1u) == gridDim.x - 1) {
    sched[0] = 0u;
    sched[1] = 0u;
    __threadfence();
  }
}
__device__ __forceinline__ int sched_next_tile(unsigned* sched, int total_tiles) {
  const int t = sched_claim(sched);
  if (t >= total_tiles) sched_retire(sched);   // this CTA's last fetch
  return t;
}
// Global pool of self-resetting scheduler counters for unbound launches, one pool per device
// (defined in capi.cu; see next_sched_slot).
constexpr int kSchedSlots = 4096;
// ---- host side ------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) !=
          cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || sym == nullptr) {
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(sym);
  return fn;
}

// The scheduler slot ({next tile, finished CTAs} counter pair) of one launch, stored to *slot.
// Two launches that run at the same time must never share a slot: both would claim from one
// counter and skip tiles, and the slot could be left dirty for every later launch.  A captured
// graph keeps the address for as long as it lives.
//   - bound (edet_sched_bind on the calling thread): the next of the caller's consecutive slots;
//     EDET_ERR_INVALID once they are used up.  The caller owns them and guarantees that two
//     launches holding the same slot are never in flight together (the launch lists of
//     lowering.py give each op its own slot);
//   - unbound: the CURRENT device's global pool of kSchedSlots, round robin, so a slot comes back
//     kSchedSlots launches later -- fine for standalone launches, not for graphs that live on.
// Records the slot for edet_last_sched_slot.  EDET_OK or an error code (+ text).  Defined in
// capi.cu.
int next_sched_slot(unsigned** slot);

// 3-D half tensor [d2][d1][d0] (d0 contiguous), box [1][box1][64], 128B swizzle.
inline int make_map(CUtensorMap* map, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2,
                    uint64_t stride1_elems, uint64_t stride2_elems, uint32_t box1,
                    uint32_t box0 = 64) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return EDET_ERR_CUDA;
  }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_elems * 2, stride2_elems * 2};
  cuuint32_t box[3] = {box0, box1, 1};
  const CUtensorMapSwizzle swz = box0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : box0 == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                              : CU_TENSOR_MAP_SWIZZLE_32B;
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) dims=[%llu,%llu,%llu] strides=[%llu,%llu] box1=%u",
              static_cast<int>(r), (unsigned long long)d0, (unsigned long long)d1,
              (unsigned long long)d2, (unsigned long long)strides[0],
              (unsigned long long)strides[1], box1);
    return EDET_ERR_CUDA;
  }
  return EDET_OK;
}


// 4-D half tensor [d3][d2][d1][d0] (NHWC activations: d0 = C, d1 = W, d2 = H, d3 = N), box
// [1][box2][box1][box0]; swizzle follows box0 (64 / 32 / 16 halves -> 128B / 64B / 32B).
inline int make_map4(CUtensorMap* map, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2,
                     uint64_t d3, uint32_t box0, uint32_t box1, uint32_t box2, bool swizzle = true) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return EDET_ERR_CUDA;
  }
  cuuint64_t dims[4] = {d0, d1, d2, d3};
  cuuint64_t strides[3] = {d0 * 2, d0 * d1 * 2, d0 * d1 * d2 * 2};
  cuuint32_t box[4] = {box0, box1, box2, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  // swizzle == false: dense [box2][box1][box0] tile (pixel rows of box0 halves, no XOR pattern)
  const CUtensorMapSwizzle swz = !swizzle      ? CU_TENSOR_MAP_SWIZZLE_NONE
                                 : box0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : box0 == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                              : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed (%d) dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u]",
              static_cast<int>(r), (unsigned long long)d0, (unsigned long long)d1,
              (unsigned long long)d2, (unsigned long long)d3, box0, box1, box2);
    return EDET_ERR_CUDA;
  }
  return EDET_OK;
}

// 4-D half tensor with explicit (element) strides for d1, d2, d3 (d0 contiguous): strided views
// such as the (row parity, column parity) sub-images a stride-2 convolution reads.
inline int make_map4_strided(CUtensorMap* map, const void* ptr, uint64_t d0, uint64_t d1,
                             uint64_t d2, uint64_t d3, uint64_t s1, uint64_t s2, uint64_t s3,
                             uint32_t box0, uint32_t box1, uint32_t box2) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return EDET_ERR_CUDA;
  }
  cuuint64_t dims[4] = {d0, d1, d2, d3};
  cuuint64_t strides[3] = {s1 * 2, s2 * 2, s3 * 2};
  cuuint32_t box[4] = {box0, box1, box2, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapSwizzle swz = box0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : box0 == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                              : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d strided) failed (%d) dims=[%llu,%llu,%llu,%llu] "
              "strides=[%llu,%llu,%llu] box=[%u,%u,%u]", static_cast<int>(r),
              (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
              (unsigned long long)d3, (unsigned long long)strides[0],
              (unsigned long long)strides[1], (unsigned long long)strides[2], box0, box1, box2);
    return EDET_ERR_CUDA;
  }
  return EDET_OK;
}

}  // namespace pwtc
}  // namespace edet
