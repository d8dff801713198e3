/*
 * automl_b200 C ABI: the sm_90a kernels behind the EfficientDet forward path.
 *
 * The reference (google/automl, /root/reference/efficientdet) has no plugin / FFI layer: its
 * hot path bottoms out in TensorFlow ops.  Each entry point below replaces the TF op(s) a
 * reference function dispatches, cited as file:line under /root/reference/efficientdet.  A
 * reference maintainer binds them with ctypes (see INTEGRATION.md) from the same Python call
 * sites.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter name starts with `h_`;
 *   - activations are NHWC IEEE half (`uint16_t` storage), channel counts multiples of 8,
 *     pixel stride (`ld*`) in elements, multiple of 8 (16-byte rows for TMA / 128-bit access);
 *   - folded inference BatchNorm: weights already carry gamma/sqrt(var+eps), `bias` is
 *     beta - mean*scale (+ conv bias) in float32;
 *   - the caller owns all memory (no allocation, no ownership transfer in the library);
 *   - every call only ENQUEUES work on `stream` (a cudaStream_t) and is CUDA-graph capturable;
 *   - return value 0 = ok, otherwise an EDET_ERR_* code; edet_last_error() gives the text.
 *     No exceptions cross the boundary.
 */
#ifndef AUTOML_B200_H_
#define AUTOML_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* edet_stream_t; /* cudaStream_t */
typedef uint16_t edet_half;  /* IEEE binary16 bits */

enum {
  EDET_OK = 0,
  EDET_ERR_INVALID = 1,   /* bad argument (shape / alignment / enum) */
  EDET_ERR_CUDA = 2,      /* a CUDA runtime / driver call failed */
  EDET_ERR_UNSUPPORTED = 3
};

/* utils.py:36-53 activation_fn; codes shared with automl_b200/utils.py */
enum {
  EDET_ACT_NONE = 0,
  EDET_ACT_SWISH = 1,
  EDET_ACT_RELU = 2,
  EDET_ACT_RELU6 = 3,
  EDET_ACT_HSWISH = 4,
  EDET_ACT_SIGMOID = 5
};

/* Pointwise implementation selector. */
enum {
  EDET_PW_TCGEN05 = 0, /* TMA -> smem -> wgmma -> registers -> epilogue -> TMA store */
  EDET_PW_SIMT = 1     /* plain CUDA-core kernel, kept only as an on-device cross-check */
};

int edet_version(void);
const char* edet_last_error(void);
/* Process-wide implementation switches, for A/B measurements and tests only (results are the same
 * for every setting).  Options: "dw_impl" = 0 (default: TMA-tiled depthwise kernel where eligible,
 * register-tiled kernel otherwise) | 1 (register-tiled kernel only); "pw_teams" = 0 (default:
 * two consumer warpgroups) | 2 | 3; "stem_impl" = 0 (default: tensor-core stem) | 1 (CUDA-core stem);
 * "sepconv_impl" = 0 (default: TMA-staged input tile for c <= 64, one buffer, four CTAs per SM) |
 * 1 (loads from global) | 2 (TMA, two buffers, three CTAs per SM);
 * "pw_smem_kb" = 0 (default: 227 KiB, one pointwise CTA per SM) | 64..227;
 * "persist_slack" = CTAs a persistent kernel leaves out of its grid (default 0). */
int edet_set_option(const char* name, int value);
int edet_get_option(const char* name, int* value);
/* Number of SMs / compute capability of the current device (major*10+minor). */
int edet_device_info(int* sm_count, int* cc);

/*
 * Serving pre-process: uint8 HWC images (all the same size) -> normalise -> aspect-preserving
 * bilinear resize (TF2 half-pixel centres) -> zero pad to [out_h, out_w].
 * Replaces inference.image_preprocess inference.py:37-56 and
 * dataloader.DetectionInputProcessor dataloader.py:59-65, 115-142.
 *   in  uint8 [n, h, w, 3]     out float32 [n, out_h, out_w, 3]
 *   h_mean_rgb / h_stddev_rgb: HOST float32[3];  h_image_scale: HOST out, scale back to the
 *   original image (image_scale_to_original), may be NULL
 */
int edet_preprocess(const uint8_t* in, float* out, int n, int h, int w, int out_h, int out_w,
                    const float* h_mean_rgb, const float* h_stddev_rgb, float* h_image_scale,
                    edet_stream_t stream);

/*
 * Stem: Conv2D 3x3 stride 2 'same' (3 -> cout, no bias) + BN + act.
 * Replaces backbone/efficientnet_model.py:511-527 (Stem.call).
 *   in   float32 [n, h, w, 3] NHWC            out  half [n, ceil(h/2), ceil(w/2), cout]
 *   w    half [27][cout]  (ky, kx, cin major; BN scale folded)      bias float32 [cout]
 */
int edet_stem_conv(const float* in, edet_half* out, const edet_half* w, const float* bias,
                   int n, int h, int wd, int cout, int act, edet_stream_t stream);

/* k x k convolution 'SAME' (ksize in {1,3,5}, stride in {1,2}) + bias (BN folded) + act
 * (+ residual) as an implicit GEMM on the tensor cores (wgmma): the Fused-MBConv convolutions of EfficientNetV2.
 * Replaces Conv2D k x k + BN (+ act) (+ skip)  efficientnetv2/effnetv2_model.py:331-341, 355-364,
 * 387-404 (FusedMBConvBlock), residual :270-277.
 *   in  half [n, h, w, cin]                 wt  half [ksize*ksize][cout][cin] (tap-major, cin
 *   contiguous, BN scale folded)            bias float32 [cout]
 *   residual half [n, ho, wo, cout] or NULL out half [n, ho, wo, cout], ho = ceil(h / stride)
 *   cin % 8 == 0, cout % 8 == 0; act in {NONE, SWISH, RELU6}. */
int edet_conv2d(const edet_half* in, const edet_half* wt, const float* bias,
                const edet_half* residual, edet_half* out, int n, int h, int w, int cin, int cout,
                int ksize, int stride, int act, edet_stream_t stream);

/* Fused front half of an MBConv block: expand 1x1 + BN + act  ->  depthwise kxk 'SAME' + BN +
 * act (+ SE squeeze), the expanded [N,H,W,cmid] tensor never leaves the SM (wgmma accumulators
 * in registers -> fp16 tile in shared memory -> depthwise).  Same results as edet_pointwise_conv
 * followed by edet_depthwise_conv (the expanded value is rounded to fp16 in both).
 * Replaces: backbone/efficientnet_model.py:303-333 (the two convs + BNs), :387-391 (their use in
 * MBConvBlock._call) and the reduce_mean of :192.
 *   x [n,h,w,cin] fp16 (cin % 8 == 0), we [cmid][cin] fp16, bias_e [cmid] f32,
 *   wd [k*k][cmid] float32, bias_d [cmid] f32, out [n,ceil(h/stride),ceil(w/stride),cmid] fp16,
 *   se_sum int64 [n][cmid] (2^-20 fixed point, ADDED to) or NULL; k in {3,5}, stride in {1,2},
 *   act in {EDET_ACT_SWISH, EDET_ACT_RELU6} applied after both convs (as the reference does). */
int edet_mbconv_expand_dw(const edet_half* x, const edet_half* we, const float* bias_e,
                          const float* wd, const float* bias_d, edet_half* out,
                          int64_t* se_sum, int n, int h, int w, int cin, int cmid, int k,
                          int stride, int act, edet_stream_t stream);

/*
 * Pointwise (1x1) convolution as a GEMM with fused epilogue:
 *   out[b, r, :] = act( A[b, r, :] @ Wt[b or 0]^T + bias ) (+ residual[b, r, :])
 * Replaces Conv2D 1x1 + BN (+ swish) (+ residual add):
 *   expand  backbone/efficientnet_model.py:303-317, 388
 *   project backbone/efficientnet_model.py:345-358, 399-412 (SE excitation enters through the
 *           per-image pre-scaled weights written by edet_se_fc, so A is read once, unscaled)
 *   resample 1x1  efficientdet_arch.py:78-95
 *   separable-conv pointwise halves  efficientdet_arch.py:512-533, 149-191, 206-249
 *   a     half [batch, rows, k]   (pixel stride lda)
 *   wt    half [wbatch, nout, k]  (k contiguous; wbatch is 1 or batch)
 *   out   half [batch, rows, nout] (pixel stride ldo >= nout)
 *   residual  nullable, same shape/stride convention as out (ldr)
 * k, lda, ldo, ldr multiples of 8.  impl: EDET_PW_*.
 */
int edet_pointwise_conv(const edet_half* a, int lda, const edet_half* wt, int wbatch,
                        const float* bias, const edet_half* residual, int ldr, edet_half* out,
                        int ldo, int batch, int rows, int k, int nout, int act, int impl,
                        edet_stream_t stream);

/*
 * Depthwise k x k convolution 'same' (k in {3,5}, stride in {1,2}) + bias + act, optionally
 * accumulating the per-(image, channel) sum of the activated output for the SE squeeze.
 * Replaces DepthwiseConv2D + BN + swish  backbone/efficientnet_model.py:320-333, 391 and the
 * depthwise half of SeparableConv2D  efficientdet_arch.py:149-191, 206-249 (bias NULL, act NONE).
 *   in   half [n, h, w, c]     out  half [n, ceil(h/s), ceil(w/s), c]
 *   w    float32 [k*k][c] (BN scale folded; the taps stay fp32: a depthwise tap error is not
 *        averaged over a K dimension like a GEMM weight's)      bias float32 [c] or NULL
 *   se_sum  int64 [n, c] or NULL: ADDED to (caller zeroes it), 2^-20 fixed point, so the
 *           reduction is order independent and bit-reproducible
 */
int edet_depthwise_conv(const edet_half* in, edet_half* out, const float* w,
                        const float* bias, int64_t* se_sum, int n, int h, int wd, int c, int k,
                        int stride, int act, edet_stream_t stream);

/*
 * Squeeze-and-excitation gate, and the excitation folded into the project weights:
 *   mean = se_sum * 2^-20 * inv_hw ; s = sigmoid(W2 @ act(W1 @ mean + b1) + b2)
 *   wt_scaled[img, o, c] = wt[o, c] * s[img, c]
 * Replaces backbone/efficientnet_model.py:183-195 (SE.call) and the multiply at :195.
 *   se_sum   int64 [n, c]               w1 float32 [se][c], b1 [se], w2 float32 [se][c] (the
 *            second FC stored TRANSPOSED so both FCs read coalesced), b2 [c]
 *   hidden   float32 [n, se] (output / scratch: the squeezed activations)
 *   gate     float32 [n, c] (output, always written)
 *   wt       half [nout][c] project weights (nullable -> only the gate is produced)
 *   wt_scaled half [n][nout][c]
 *   zero_buf int64 [n, zero_count] or NULL: cleared by this call (the accumulator of the next
 *            block, so no separate memset launch is needed)
 */
int edet_se_fc(const int64_t* se_sum, float inv_hw, const float* w1, const float* b1,
               const float* w2, const float* b2, float* hidden, float* gate, const edet_half* wt,
               edet_half* wt_scaled, int64_t* zero_buf, int zero_count, int n, int c, int se,
               int nout, int act, edet_stream_t stream);

/*
 * One BiFPN node in a single pass: per input {identity | TF1 nearest-neighbour upsample |
 * max-pool (pool, stride, 'SAME') downsample} -> weighted fusion -> act -> depthwise 3x3 'same'.
 * Replaces resample_feature_map efficientdet_arch.py:100-130, fuse_features :418-475 (the
 * normalised weights are computed on the host from WSM; 'sum' passes 1.0), activation :509-510
 * and the depthwise half of the SeparableConv2D :512-525.
 */
enum { EDET_RS_SAME = 0, EDET_RS_UP = 1, EDET_RS_DOWN = 2 };
typedef struct {
  const edet_half* ptr; /* half [n, h, w, c] */
  int h, w;
  int mode;             /* EDET_RS_* */
  int pool_h, pool_w, stride_h, stride_w; /* EDET_RS_DOWN only */
  float weight;         /* normalised fusion weight of this input */
} edet_fuse_input;
int edet_fuse_dw(const edet_fuse_input* h_inputs, int n_inputs, const float* dw_w,
                 edet_half* out, int n, int h, int wd, int c, int act, edet_stream_t stream);

/* Fused separable convolution of a head tower layer (wgmma):
 *   out = post_act( pointwise( depthwise3x3( input ) ) + bias )
 * i.e. a depthwise conv followed by edet_pointwise_conv without the [n,h,w,c] intermediate in HBM
 * (the depthwise result is rounded to fp16 in shared memory, exactly as the pair rounds it in
 * global memory).  Replaces a head tower layer (efficientdet_arch.py:149-191 / :206-249: the
 * activation comes after the per-level BN folded into pw_wt / bias).  h_inputs: ONE input with
 * mode EDET_RS_SAME and weight 1, pre_act = EDET_ACT_NONE; anything else returns
 * EDET_ERR_UNSUPPORTED (the whole-BiFPN-node form was removed in round 2: slower than
 * edet_fuse_dw + edet_pointwise_conv).
 *   dw_w float32 [9][c], pw_wt half [nout][c], bias float32 [nout], out half [n,h,wd,ldo]
 *   c % 8 == 0, c <= 128; nout % 8 == 0, nout <= 128; ldo >= nout, ldo % 8 == 0. */
int edet_sepconv(const edet_fuse_input* h_inputs, int n_inputs, int pre_act, const float* dw_w,
                 const edet_half* pw_wt, const float* bias, edet_half* out, int ldo, int n, int h,
                 int wd, int c, int nout, int post_act, edet_stream_t stream);

/* Max-pool 'SAME' (padded cells never win). Replaces efficientdet_arch.py:103-112 for the
 * P6/P7/P8 extra levels (efficientdet_arch.py:369-387). */
int edet_max_pool(const edet_half* in, edet_half* out, int n, int h, int wd, int c, int pool_h,
                  int pool_w, int stride_h, int stride_w, edet_stream_t stream);

/*
 * Class-predict 1x1 convolution of ONE pyramid level fused with the class half of pre-NMS: the
 * [n, h, w, num_anchors * num_classes] logits are never written; per pixel and anchor the kernel
 * rounds each logit to fp16 (what edet_pointwise_conv would have stored), takes max / first
 * arg-max over the classes and the sigmoid of the max, exactly as edet_pre_nms does -- bit-identical
 * scores and classes.  Replaces the pointwise half of class-predict (efficientdet_arch.py:166-174)
 * + tf2/postprocess.py:88-156 (topk_class_boxes with max_nms_inputs == 0, sigmoid in pre_nms).
 *   a            half [batch, rows, lda]: the predict layer's depthwise output (rows = h_l * w_l)
 *   wt_padded    half [num_anchors * 96][k]: row a*96 + c = class c of anchor a (zero pad rows;
 *                num_classes <= 96)
 *   bias_padded  float32 [num_anchors * 96], -inf on the pad rows (they can never be the maximum)
 *   scores float32 / classes int32 [batch, total_anchors], written at
 *                anchor_begin + row * num_anchors + a
 * Follow with edet_pre_nms(h_cls = NULL, ...) for the boxes.
 */
int edet_class_argmax(const edet_half* a, int lda, const edet_half* wt_padded,
                      const float* bias_padded, float* scores, int32_t* classes, int anchor_begin,
                      int total_anchors, int num_anchors, int batch, int rows, int k,
                      edet_stream_t stream);

/*
 * Pre-NMS: per image and anchor, max / argmax over classes, sigmoid, anchor box decode.
 * h_cls == NULL: box decode only (scores / classes may be NULL; see edet_class_argmax).
 * Replaces tf2/postprocess.py:67-156 (merge_class_box_level_outputs, topk_class_boxes with
 * max_nms_inputs == 0, pre_nms) and tf2/anchors.py:30-58 (decode_box_outputs).
 *   h_cls[l] half [n, h_l, w_l, ld_cls] (anchor-major, class-minor: a*num_classes + c)
 *   h_box[l] half [n, h_l, w_l, ld_box] (a*4 + {ty,tx,th,tw})
 *   anchors  float32 [total_anchors, 4]
 *   boxes float32 [n, total, 4]  scores float32 [n, total]  classes int32 [n, total]
 */
int edet_pre_nms(const edet_half* const* h_cls, const edet_half* const* h_box,
                 const int* h_level_hw /* [levels][2] */, int levels, int ld_cls, int ld_box,
                 int num_anchors, int num_classes, const float* anchors, float* boxes,
                 float* scores, int32_t* classes, int n, edet_stream_t stream);

/*
 * Global NMS with tf.raw_ops.NonMaxSuppressionV5 semantics (hard, or gaussian soft when
 * soft_nms_sigma > 0), padded to max_output_size, then gather + class offset + clip + scale
 * into the serving layout.  Replaces tf2/postprocess.py:159-205 (nms), :375-406
 * (postprocess_global), :61-64 (clip_boxes) and inference.py:233-271 (det_post_process).
 *   detections float32 [n, max_output_size, 7] rows [image_id, ymin, xmin, ymax, xmax, score, class]
 *              (image_id = image_id_base + index in this call: the rank's offset in a sharded batch)
 *   sel_index int32 [n, max_output_size] (selected anchor index, 0 padded), valid int32 [n]
 *   work  scratch, edet_nms_work_bytes(n, k) bytes
 */
size_t edet_nms_work_bytes(int n, int k);
int edet_nms_v5(const float* boxes, const float* scores, const int32_t* classes,
                const float* image_scales /* [n] or NULL */, int image_id_base, int n, int k,
                int max_output_size,
                float iou_threshold, float score_threshold, float soft_nms_sigma,
                float clip_h, float clip_w, float* detections, int32_t* sel_index,
                int32_t* valid, void* work, edet_stream_t stream);

/*
 * Pre-NMS with nms_configs.max_nms_inputs > 0: per image the top max_nms_inputs (anchor, class)
 * logits (ties: lower flat index anchor*num_classes + class), then sigmoid and box decode of the
 * selected pairs.  Replaces tf2/postprocess.py:88-102 (topk_class_boxes, top-k branch) inside
 * pre_nms (:119-156) and tf2/anchors.py:30-58.  Inputs as edet_pre_nms; outputs sorted by
 * (logit descending, flat index ascending):
 *   boxes float32 [n, k, 4], scores float32 [n, k], classes int32 [n, k], indices int32 [n, k]
 *   (anchor index of each row), k = max_nms_inputs <= 8192.
 */
int edet_pre_nms_topk(const edet_half* const* h_cls, const edet_half* const* h_box,
                      const int* h_level_hw /* [levels][2] */, int levels, int ld_cls, int ld_box,
                      int num_anchors, int num_classes, const float* anchors, int max_nms_inputs,
                      float* boxes, float* scores, int32_t* classes, int32_t* indices, int n,
                      edet_stream_t stream);

/*
 * CUDA replacement for nms_np.per_class_nms (nms_np.py:220-264) with the `hard` (nms_np.py:89-126)
 * and `diou` (:28-86) methods: per class greedy NMS in descending score order, float32 "+1 pixel"
 * IoU in nms_np's order of operations (keep decisions bit-identical to NumPy's), survivors of all
 * classes merged, top max_boxes_to_draw by score.  Replaces the tf.numpy_function call of
 * tf2/postprocess.py:541-556 (generate_detections with nms_configs.pyfunc).
 *   boxes float32 [n, k, 4] (ymin, xmin, ymax, xmax), scores float32 [n, k], classes int32 [n, k]
 *   (0-based; values outside [0, num_classes) are ignored), image_ids / image_scales float32 [n]
 *   or NULL (row index / 1.0)
 *   detections float32 [n, max_boxes_to_draw, 7]: [image_id, xmin, ymin, xmax, ymax, score,
 *   class + 1], boxes x image_scale; rows beyond the survivors are [image_id, 0,0,0,0, -1e5, 0]
 *   keep_index int32 [n, max_boxes_to_draw]: anchor index of each row (-1 for dummy rows)
 *   num_valid int32 [n]
 * hard / diou: equal scores -> the higher anchor index first (NumPy's unstable argsort leaves this
 * undefined).
 * EDET_NMS_GAUSSIAN / EDET_NMS_LINEAR: soft NMS (nms_np.py:129-191) with `sigma` (gaussian),
 * `iou_thresh` (linear) and `score_thresh` (nms_np's defaults 0.5 / 0.3 / 0.001 are applied by the
 * caller); `work` is a float32 [n][k] workspace (may be NULL for hard / diou).  linear is
 * bit-identical to NumPy; gaussian evaluates exp in double and rounds to float32, NumPy's SIMD
 * float32 exp is within 2 ulp of that, so scores may differ in the last bits.  Equal scores ->
 * the lower anchor index first.
 */
#define EDET_NMS_HARD 0
#define EDET_NMS_DIOU 1
#define EDET_NMS_GAUSSIAN 2
#define EDET_NMS_LINEAR 3
int edet_per_class_nms(const float* boxes, const float* scores, const int32_t* classes,
                       const float* image_ids, const float* image_scales, int n, int k,
                       int num_classes, int max_boxes_to_draw, int method, float iou_thresh,
                       float sigma, float score_thresh, float* work, float* detections,
                       int32_t* keep_index, int32_t* num_valid, edet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* AUTOML_B200_H_ */
