// Shared by bifpn.cu (fuse + depthwise) and sepconv_tc.cu (fuse + depthwise + pointwise on the
// tensor cores): the description of a BiFPN node input and its host-side validation.
#pragma once
#include <math_constants.h>

#include "common.cuh"

namespace edet {

constexpr int kFuseMaxIn = 3;

struct FuseIn {
  const __half* ptr;
  int h, w, mode;
  int pool_h, pool_w, stride_h, stride_w, pad_t, pad_l;
  float scale_h, scale_w;  // in/out, float32 as TF computes it
  float weight;
};
struct FuseParams {
  FuseIn in[kFuseMaxIn];
  int n_inputs;
};

__device__ __forceinline__ void load8(const __half* base, int hh, int ww, int c, int y, int x,
                                      int ch, float* f) {
  half8_to_float(__ldg(reinterpret_cast<const uint4*>(
                     base + (static_cast<size_t>(y) * ww + x) * c + ch)), f);
}


// One 8-channel group of one input resampled at node pixel (y, x): identity / TF1 nearest
// upsample / 'SAME' max-pool (padded cells never win).
__device__ __forceinline__ void resample8(const FuseIn& fi, const __half* base, int c, int y, int x,
                                          int ch, float* v) {
  if (fi.mode == EDET_RS_SAME) {
    load8(base, fi.h, fi.w, c, y, x, ch, v);
  } else if (fi.mode == EDET_RS_UP) {
    const int sy = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(y), fi.scale_h))), fi.h - 1);
    const int sx = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(x), fi.scale_w))), fi.w - 1);
    load8(base, fi.h, fi.w, c, sy, sx, ch, v);
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = -CUDART_INF_F;
    const int sy0 = y * fi.stride_h - fi.pad_t, sx0 = x * fi.stride_w - fi.pad_l;
    for (int py = 0; py < fi.pool_h; ++py) {
      const int sy = sy0 + py;
      if (sy < 0 || sy >= fi.h) continue;
      for (int px = 0; px < fi.pool_w; ++px) {
        const int sx = sx0 + px;
        if (sx < 0 || sx >= fi.w) continue;
        float t[8];
        load8(base, fi.h, fi.w, c, sy, sx, ch, t);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], t[e]);
      }
    }
  }
}

// ---- compile-time input signatures -----------------------------------------------------------
// A BiFPN cell (tf2/fpn_configs.py:24-72) only has three node shapes: top-down nodes read
// [same level, upsampled coarser level]; bottom-up nodes read [same level input, same level
// top-down output, pooled finer level]; the topmost bottom-up node reads [same level, pooled].
// A QuFPN cell (:75-163) adds two: the quad-add nodes read [same, same], the nodes of its
// second top-down path read [same level input, same level path-3 output, upsampled coarser level].
constexpr int kSigGeneric = 0, kSigSameUp = 1, kSigSameSameDown = 2, kSigSameDown = 3,
              kSigSameSame = 4, kSigSameSameUp = 5;
__host__ __device__ constexpr int sig_inputs(int sig) {
  return (sig == kSigSameSameDown || sig == kSigSameSameUp) ? 3 : 2;
}
__host__ __device__ constexpr int sig_mode(int sig, int i) {
  return sig == kSigSameUp         ? (i == 0 ? EDET_RS_SAME : EDET_RS_UP)
         : sig == kSigSameSameDown ? (i < 2 ? EDET_RS_SAME : EDET_RS_DOWN)
         : sig == kSigSameSame     ? EDET_RS_SAME
         : sig == kSigSameSameUp   ? (i < 2 ? EDET_RS_SAME : EDET_RS_UP)
                                   : (i == 0 ? EDET_RS_SAME : EDET_RS_DOWN);
}
inline int fuse_signature(const FuseParams& p) {
  auto is = [&](int i, int mode) { return p.in[i].mode == mode; };
  // the unrolled DOWN path holds a 3 x 3 window in registers
  auto pool33 = [&](int i) { return p.in[i].pool_h == 3 && p.in[i].pool_w == 3; };
  if (p.n_inputs == 2 && is(0, EDET_RS_SAME) && is(1, EDET_RS_UP)) return kSigSameUp;
  if (p.n_inputs == 3 && is(0, EDET_RS_SAME) && is(1, EDET_RS_SAME) && is(2, EDET_RS_DOWN) && pool33(2))
    return kSigSameSameDown;
  if (p.n_inputs == 2 && is(0, EDET_RS_SAME) && is(1, EDET_RS_DOWN) && pool33(1)) return kSigSameDown;
  if (p.n_inputs == 2 && is(0, EDET_RS_SAME) && is(1, EDET_RS_SAME)) return kSigSameSame;
  if (p.n_inputs == 3 && is(0, EDET_RS_SAME) && is(1, EDET_RS_SAME) && is(2, EDET_RS_UP))
    return kSigSameSameUp;
  return kSigGeneric;
}

// Raw 16-byte loads of one 8-channel group of one input at node pixel (y, x), mode known at
// compile time: returns the number of taps loaded (1 for SAME / UP; up to 9 for a 3 x 3 'SAME'
// max-pool, padded cells skipped).  resample_reduce turns them into the resampled fp32 values
// exactly as resample8 does (max of the in-image taps).
template <int MODE>
__device__ __forceinline__ int resample_raw(const FuseIn& fi, const __half* base, int c, int y, int x,
                                            int ch, uint4* raw) {
  if (MODE == EDET_RS_SAME) {
    raw[0] = __ldg(reinterpret_cast<const uint4*>(base + (static_cast<size_t>(y) * fi.w + x) * c + ch));
    return 1;
  }
  if (MODE == EDET_RS_UP) {
    const int sy = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(y), fi.scale_h))), fi.h - 1);
    const int sx = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(x), fi.scale_w))), fi.w - 1);
    raw[0] = __ldg(reinterpret_cast<const uint4*>(base + (static_cast<size_t>(sy) * fi.w + sx) * c + ch));
    return 1;
  }
  const int sy0 = y * fi.stride_h - fi.pad_t, sx0 = x * fi.stride_w - fi.pad_l;
  int n = 0;
#pragma unroll
  for (int py = 0; py < 3; ++py) {
#pragma unroll
    for (int px = 0; px < 3; ++px) {
      const int sy = sy0 + py, sx = sx0 + px;
      const bool ok = sy >= 0 && sy < fi.h && sx >= 0 && sx < fi.w;
      // padded cells repeat an in-image tap: max() is idempotent, so the result is unchanged.
      // The window of an in-image node pixel always contains (clamped) in-image cells.
      const int cy = min(max(sy, 0), fi.h - 1), cx = min(max(sx, 0), fi.w - 1);
      (void)ok;
      raw[n++] = __ldg(reinterpret_cast<const uint4*>(base + (static_cast<size_t>(cy) * fi.w + cx) * c + ch));
    }
  }
  return n;
}
template <int MODE>
__device__ __forceinline__ void resample_reduce(const uint4* raw, int taps, float* v) {
  half8_to_float(raw[0], v);
  if (MODE == EDET_RS_DOWN) {
#pragma unroll
    for (int t = 1; t < 9; ++t) {
      if (t < taps) {
        float f[8];
        half8_to_float(raw[t], f);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], f[e]);
      }
    }
  }
}

// Validates the caller's edet_fuse_input list against the node shape and fills FuseParams.
inline int fill_fuse_params(const edet_fuse_input* h_inputs, int n_inputs, int h, int wd,
                            const char* who, FuseParams* out) {
  EDET_CHECK_ARG(h_inputs != nullptr, "%s: null input list", who);
  EDET_CHECK_ARG(n_inputs >= 1 && n_inputs <= kFuseMaxIn, "%s: 1..3 inputs (got %d)", who, n_inputs);
  FuseParams& p = *out;
  p.n_inputs = n_inputs;
  for (int i = 0; i < n_inputs; ++i) {
    const edet_fuse_input& s = h_inputs[i];
    FuseIn& d = p.in[i];
    EDET_CHECK_ARG(s.ptr != nullptr, "%s: input %d is null", who, i);
    d.ptr = reinterpret_cast<const __half*>(s.ptr);
    d.h = s.h; d.w = s.w; d.mode = s.mode; d.weight = s.weight;
    d.pool_h = d.pool_w = d.stride_h = d.stride_w = 1; d.pad_t = d.pad_l = 0;
    d.scale_h = d.scale_w = 1.f;
    if (s.mode == EDET_RS_SAME) {
      EDET_CHECK_ARG(s.h == h && s.w == wd, "%s: input %d is %dx%d, node is %dx%d", who, i, s.h, s.w, h, wd);
    } else if (s.mode == EDET_RS_UP) {
      EDET_CHECK_ARG(s.h <= h && s.w <= wd, "%s: input %d cannot be upsampled", who, i);
      d.scale_h = static_cast<float>(s.h) / static_cast<float>(h);
      d.scale_w = static_cast<float>(s.w) / static_cast<float>(wd);
    } else if (s.mode == EDET_RS_DOWN) {
      EDET_CHECK_ARG(ceil_div(s.h, s.stride_h) == h && ceil_div(s.w, s.stride_w) == wd,
                     "%s: input %d pooled size mismatch", who, i);
      d.pool_h = s.pool_h; d.pool_w = s.pool_w; d.stride_h = s.stride_h; d.stride_w = s.stride_w;
      d.pad_t = same_pad_before(s.h, s.pool_h, s.stride_h);
      d.pad_l = same_pad_before(s.w, s.pool_w, s.stride_w);
    } else {
      set_error("%s: bad mode %d", who, s.mode);
      return EDET_ERR_INVALID;
    }
  }
  return EDET_OK;
}

}  // namespace edet
