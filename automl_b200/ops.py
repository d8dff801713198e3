"""Tensor-level wrappers over the C-ABI (torch tensors are only device-memory containers).

Every function enqueues on the CURRENT torch CUDA stream, allocates nothing except where
stated, and raises if the tensors are not CUDA / not contiguous / misaligned.  There is no CPU
implementation behind any of them.
"""
import ctypes

import numpy as np
import torch

from automl_b200 import _lib
from automl_b200._lib import FuseInput, PW_SIMT, PW_TCGEN05, RS_DOWN, RS_SAME, RS_UP  # noqa: F401


def _stream():
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t, dtype=None):
  if t is None:
    return None
  if not t.is_cuda:
    raise ValueError('automl_b200 ops need CUDA tensors (no CPU fallback)')
  if dtype is not None and t.dtype != dtype:
    raise ValueError('expected %s, got %s' % (dtype, t.dtype))
  if not t.is_contiguous():
    raise ValueError('tensor must be contiguous')
  return ctypes.c_void_p(t.data_ptr())


def _round8(x):
  return (x + 7) // 8 * 8


def set_option(name, value):
  """Process-wide implementation switch (A/B measurements, tests): see edet_set_option."""
  _lib.call('edet_set_option', name.encode(), int(value))


def get_option(name):
  v = ctypes.c_int(0)
  _lib.call('edet_get_option', name.encode(), ctypes.byref(v))
  return v.value


def sched_bind(slots, count=0):
  """Binds the calling thread's slot-using launches to `count` consecutive scheduler slots at
  device address `slots` (2 * count zeroed uint32); None unbinds (see edet_sched_bind)."""
  _lib.call('edet_sched_bind', ctypes.c_void_p(slots) if slots else None, int(count))


def last_sched_slot():
  """Device address of the scheduler slot of this thread's latest slot-using launch (0 before
  the first)."""
  v = ctypes.c_void_p()
  _lib.call('edet_last_sched_slot', ctypes.byref(v))
  return v.value or 0


def preprocess(raw, out, mean_rgb, stddev_rgb):
  """raw uint8 [N,h,w,3] -> out fp32 [N,H,W,3]; returns image_scale_to_original (float)."""
  n, h, w, _ = raw.shape
  _, oh, ow, _ = out.shape
  mean = (ctypes.c_float * 3)(*[float(v) for v in mean_rgb])
  std = (ctypes.c_float * 3)(*[float(v) for v in stddev_rgb])
  scale = ctypes.c_float(0.0)
  _lib.call('edet_preprocess', _ptr(raw, torch.uint8), _ptr(out, torch.float32), n, h, w, oh, ow,
            mean, std, ctypes.byref(scale), _stream())
  return scale.value


def preprocess_float(images, out, mean_rgb, stddev_rgb):
  """images float32 [N,h,w,3] -> out float32 [N,H,W,3], as `preprocess` computes it for uint8
  images (an image of integral values 0..255 gives the same bits); returns
  image_scale_to_original (float).  Refuses other dtypes, shapes and strides before launching."""
  if images.dim() != 4 or images.shape[-1] != 3 or out.dim() != 4 or out.shape[-1] != 3:
    raise ValueError('preprocess_float: images %s and out %s must be [N, h, w, 3] and [N, H, W, 3]'
                     % (tuple(images.shape), tuple(out.shape)))
  n, h, w, _ = images.shape
  _, oh, ow, _ = out.shape
  if out.shape[0] != n:
    raise ValueError('preprocess_float: %d images, out holds %d' % (n, out.shape[0]))
  mean = (ctypes.c_float * 3)(*[float(v) for v in mean_rgb])
  std = (ctypes.c_float * 3)(*[float(v) for v in stddev_rgb])
  scale = ctypes.c_float(0.0)
  _lib.call('edet_preprocess_float', _ptr(images, torch.float32), _ptr(out, torch.float32), n, h, w,
            oh, ow, mean, std, ctypes.byref(scale), _stream())
  return scale.value


PRE_DESC_WORDS = 6      # int32 words of one edet_preprocess_image row: offset (2 words), h, w, scaled_h, scaled_w


def preprocess_ragged(packed, desc, out, mean_rgb, stddev_rgb):
  """A ragged request in one launch: packed uint8 (the images back to back, HWC), desc int32
  [N, 6] edet_preprocess_image rows (byte offset into `packed`, h, w, scaled_h, scaled_w; the
  caller keeps every image inside `packed`) -> out fp32 [N,H,W,3], each image as `preprocess`
  computes it alone."""
  n, oh, ow = out.shape[0], out.shape[1], out.shape[2]
  if tuple(out.shape) != (n, oh, ow, 3) or tuple(desc.shape) != (n, PRE_DESC_WORDS):
    raise ValueError('preprocess_ragged: out %s must be [N, H, W, 3] and desc %s [N, %d]'
                     % (tuple(out.shape), tuple(desc.shape), PRE_DESC_WORDS))
  mean = (ctypes.c_float * 3)(*[float(v) for v in mean_rgb])
  std = (ctypes.c_float * 3)(*[float(v) for v in stddev_rgb])
  _lib.call('edet_preprocess_ragged', _ptr(packed, torch.uint8), _ptr(desc, torch.int32),
            _ptr(out, torch.float32), n, oh, ow, mean, std, _stream())


def preprocess_mirrored(packed, desc, out, mean_rgb, stddev_rgb):
  """A request and its mirror in one launch (flip test-time augmentation): packed / desc as
  preprocess_ragged for N images -> out fp32 [2N,H,W,3], out[:N] as preprocess_ragged writes it and
  out[N + i] = out[i] flipped on width."""
  n2, oh, ow = out.shape[0], out.shape[1], out.shape[2]
  n = n2 // 2
  if tuple(out.shape) != (2 * n, oh, ow, 3) or n < 1 or tuple(desc.shape) != (n, PRE_DESC_WORDS):
    raise ValueError('preprocess_mirrored: out %s must be [2N, H, W, 3] and desc %s [N, %d]'
                     % (tuple(out.shape), tuple(desc.shape), PRE_DESC_WORDS))
  mean = (ctypes.c_float * 3)(*[float(v) for v in mean_rgb])
  std = (ctypes.c_float * 3)(*[float(v) for v in stddev_rgb])
  _lib.call('edet_preprocess_mirrored', _ptr(packed, torch.uint8), _ptr(desc, torch.int32),
            _ptr(out, torch.float32), n, oh, ow, mean, std, _stream())


def stem_conv(images, out, w, bias, act):
  """images fp32 [N,H,W,3] -> out fp16 [N,ceil(H/2),ceil(W/2),C]."""
  n, h, wd, c3 = images.shape
  assert c3 == 3
  _lib.call('edet_stem_conv', _ptr(images, torch.float32), _ptr(out, torch.float16),
            _ptr(w, torch.float16), _ptr(bias, torch.float32), n, h, wd, out.shape[-1], act,
            _stream())


def pointwise_conv(a, wt, bias, out, act, residual=None, rows=None, batch=None, nout=None,
                   impl=PW_TCGEN05):
  """a fp16 [batch, rows, lda] (k = wt.shape[-1] <= lda), wt fp16 [wbatch, nout, k] or [nout, k],
  out fp16 [batch, rows, ldo]."""
  k = wt.shape[-1]
  wbatch = wt.shape[0] if wt.dim() == 3 else 1
  n_out = nout if nout is not None else wt.shape[-2]
  lda, ldo = a.shape[-1], out.shape[-1]
  if batch is None:
    batch = 1
  if rows is None:
    rows = a.numel() // (lda * batch)
  ldr = residual.shape[-1] if residual is not None else 0
  _lib.call('edet_pointwise_conv', _ptr(a, torch.float16), lda, _ptr(wt, torch.float16), wbatch,
            _ptr(bias, torch.float32), _ptr(residual, torch.float16), ldr,
            _ptr(out, torch.float16), ldo, batch, rows, k, n_out, act, impl, _stream())


def depthwise_conv(x, out, w, bias, act, k, stride, se_sum=None):
  """se_sum: int64 [N, C] accumulator (added to; 2^-20 fixed point) or None."""
  n, h, wd, c = x.shape
  _lib.call('edet_depthwise_conv', _ptr(x, torch.float16), _ptr(out, torch.float16),
            _ptr(w, torch.float32), _ptr(bias, torch.float32), _ptr(se_sum, torch.int64),
            n, h, wd, c, k, stride, act, _stream())


def conv2d(x, wt, bias, out, act, ksize, stride, residual=None):
  """k x k 'SAME' convolution on the tensor cores (wgmma): x fp16 [N,H,W,cin], wt fp16 [k*k, cout, cin], bias fp32
  [cout], out fp16 [N,ceil(H/s),ceil(W/s),cout], residual like out or None."""
  n, h, w, cin = x.shape
  cout = wt.shape[1]
  _lib.call('edet_conv2d', _ptr(x, torch.float16), _ptr(wt, torch.float16),
            _ptr(bias, torch.float32), _ptr(residual, torch.float16), _ptr(out, torch.float16),
            n, h, w, cin, cout, ksize, stride, act, _stream())


def conv_transpose_weights(kernel, c0, scale=None):
  """Packs a Keras Conv2DTranspose kernel [3, 3, cout, cin] (float, cin = c0 + c1) into the
  float64 [4 taps][4 * round8(cout)][round8(c0) + round8(c1)] sub-pixel layout of
  edet_conv2d_transpose: row (py*2+px)*C8 + co of tap ty*2+tx is kernel[ky, kx, co] for output
  phase (py, px), ky = 1 if py else (2 if ty == 0 else 0) (kx alike), zero for ty < py or tx < px.
  Input channels [0, c0) go to columns [0, c0), the rest to columns round8(c0)...  `scale`
  [cout] (the folded BN scale) multiplies each output channel."""
  kernel = np.asarray(kernel, np.float64)
  kh, kw, cout, cin = kernel.shape
  assert (kh, kw) == (3, 3) and 0 < c0 <= cin
  if scale is not None:
    kernel = kernel * np.asarray(scale, np.float64)[:, None]
  c8, c1 = _round8(cout), cin - c0
  off1 = _round8(c0)
  out = np.zeros((4, 4 * c8, off1 + _round8(c1)), np.float64)
  for py in range(2):
    for px in range(2):
      rows = slice((py * 2 + px) * c8, (py * 2 + px) * c8 + cout)
      for ty in range(py, 2):
        for tx in range(px, 2):
          ky = 1 if py else (2 if ty == 0 else 0)
          kx = 1 if px else (2 if tx == 0 else 0)
          out[ty * 2 + tx, rows, :c0] = kernel[ky, kx, :, :c0]
          out[ty * 2 + tx, rows, off1:off1 + c1] = kernel[ky, kx, :, c0:]
  return out


def conv2d_transpose(a0, wt, bias, out, act, cout, a1=None, c0=None, c1=None):
  """Conv2DTranspose 3x3 stride 2 'SAME' + bias + act on the tensor cores: a0 fp16 [N,H,W,lda0]
  (channels [0, c0), c0 defaults to lda0), a1 None or fp16 [N,H,W,lda1] (channels [0, c1)) read as
  the K channels after a0's, wt fp16 from conv_transpose_weights, bias fp32 [cout], out fp16
  [N,2H,2W,ldo] with ldo >= round8(cout)."""
  n, h, w, lda0 = a0.shape
  c0 = lda0 if c0 is None else c0
  lda1 = 0
  if a1 is not None:
    assert tuple(a1.shape[:3]) == (n, h, w)
    lda1 = a1.shape[-1]
    c1 = lda1 if c1 is None else c1
  else:
    c1 = 0
  if tuple(out.shape[:3]) != (n, 2 * h, 2 * w):
    raise ValueError('conv2d_transpose: out must be [%d, %d, %d, ldo], got %s'
                     % (n, 2 * h, 2 * w, tuple(out.shape)))
  if tuple(wt.shape) != (4, 4 * _round8(cout), _round8(c0) + _round8(c1)):
    raise ValueError('conv2d_transpose: wt shape %s does not match cout %d, c0 %d, c1 %d'
                     % (tuple(wt.shape), cout, c0, c1))
  _lib.call('edet_conv2d_transpose', _ptr(a0, torch.float16), c0, lda0, _ptr(a1, torch.float16),
            c1, lda1, _ptr(wt, torch.float16), _ptr(bias, torch.float32), act,
            _ptr(out, torch.float16), out.shape[-1], n, h, w, cout, _stream())


def mbconv_expand_dw(x, we, bias_e, wd, bias_d, out, act, k, stride, se_sum=None):
  """Fused expand 1x1 + depthwise kxk: x fp16 [N,H,W,cin], we fp16 [cmid,cin], wd fp32
  [k*k,cmid], out fp16 [N,Ho,Wo,cmid]; se_sum int64 [N,cmid] (added to) or None."""
  n, h, wd_, cin = x.shape
  cmid = we.shape[0]
  _lib.call('edet_mbconv_expand_dw', _ptr(x, torch.float16), _ptr(we, torch.float16),
            _ptr(bias_e, torch.float32), _ptr(wd, torch.float32), _ptr(bias_d, torch.float32),
            _ptr(out, torch.float16), _ptr(se_sum, torch.int64), n, h, wd_, cin, cmid, k, stride,
            act, _stream())


def se_fc(se_sum, inv_hw, w1, b1, w2, b2, gate, act, wt=None, wt_scaled=None, zero_buf=None,
          hidden=None):
  """se_sum int64 [N, C]; zero_buf: int64 [N, Cz] buffer cleared by the same launch; hidden:
  float32 [N, se] scratch for the squeezed activations (allocated here when not given)."""
  n, c = gate.shape
  se = w1.shape[0]
  if hidden is None:
    hidden = torch.empty(n, se, dtype=torch.float32, device=gate.device)
  nout = wt.shape[0] if wt is not None else 0
  zc = zero_buf.shape[1] if zero_buf is not None else 0
  _lib.call('edet_se_fc', _ptr(se_sum, torch.int64), ctypes.c_float(inv_hw),
            _ptr(w1, torch.float32), _ptr(b1, torch.float32), _ptr(w2, torch.float32),
            _ptr(b2, torch.float32), _ptr(hidden, torch.float32), _ptr(gate, torch.float32),
            _ptr(wt, torch.float16),
            _ptr(wt_scaled, torch.float16), _ptr(zero_buf, torch.int64), zc, n, c, se, nout, act,
            _stream())


def make_fuse_inputs(specs):
  """specs: list of (tensor [N,h,w,C], mode, pool(4-tuple or None), weight)."""
  arr = (FuseInput * len(specs))()
  for i, (t, mode, pool, weight) in enumerate(specs):
    arr[i].ptr = t.data_ptr()
    arr[i].h, arr[i].w = t.shape[1], t.shape[2]
    arr[i].mode = mode
    ph, pw, sh, sw = pool if pool else (1, 1, 1, 1)
    arr[i].pool_h, arr[i].pool_w, arr[i].stride_h, arr[i].stride_w = ph, pw, sh, sw
    arr[i].weight = float(weight)
  return arr


def fuse_dw(specs, dw_w, out, act, channel_weights=None):
  """channel_weights: None (each spec's scalar weight) or fp32 [len(specs), C], the normalised
  per-channel fusion weights of the channel_* methods (the specs' weights are then ignored)."""
  n, h, wd, c = out.shape
  for t, _, _, _ in specs:
    _ptr(t, torch.float16)
  arr = make_fuse_inputs(specs)
  if channel_weights is None:
    _lib.call('edet_fuse_dw', arr, len(specs), _ptr(dw_w, torch.float32),
              _ptr(out, torch.float16), n, h, wd, c, act, _stream())
    return
  if tuple(channel_weights.shape) != (len(specs), c):
    raise ValueError('fuse_dw: channel_weights must be [%d, %d], got %s'
                     % (len(specs), c, tuple(channel_weights.shape)))
  _lib.call('edet_fuse_dw_channel', arr, len(specs), _ptr(channel_weights, torch.float32),
            _ptr(dw_w, torch.float32), _ptr(out, torch.float16), n, h, wd, c, act, _stream())


SEPCONV_MAX_C = 128   # edet_sepconv limits (c and nout)


def sepconv(specs, pre_act, dw_w, pw_wt, bias, out, post_act, nout=None):
  """Head tower layer in one kernel (depthwise 3x3 + pointwise 1x1): specs = ONE (tensor,
  RS_SAME, None, 1.0) input, pre_act ACT_NONE; pw_wt fp16 [nout, c], out fp16 [N,h,w,ldo]
  (ldo >= nout)."""
  n, h, wd, ldo = out.shape
  c = pw_wt.shape[-1]
  n_out = nout if nout is not None else pw_wt.shape[0]
  for t, _, _, _ in specs:
    _ptr(t, torch.float16)
  arr = make_fuse_inputs(specs)
  _lib.call('edet_sepconv', arr, len(specs), pre_act, _ptr(dw_w, torch.float32),
            _ptr(pw_wt, torch.float16), _ptr(bias, torch.float32), _ptr(out, torch.float16), ldo,
            n, h, wd, c, n_out, post_act, _stream())


def max_pool(x, out, pool, stride):
  n, h, wd, c = x.shape
  _lib.call('edet_max_pool', _ptr(x, torch.float16), _ptr(out, torch.float16), n, h, wd, c,
            pool[0], pool[1], stride[0], stride[1], _stream())


def global_avg_pool(x, out):
  """x fp16 [N, ..., C] (NHWC map) -> out float32 [N, C], the mean over the pixels."""
  n, c = x.shape[0], x.shape[-1]
  if tuple(out.shape) != (n, c):
    raise ValueError('global_avg_pool: out must be [%d, %d], got %s' % (n, c, tuple(out.shape)))
  _lib.call('edet_global_avg_pool', _ptr(x, torch.float16), _ptr(out, torch.float32), n,
            x.numel() // max(n * c, 1), c, _stream())


def dense(x, wt, bias, out):
  """x float32 [N, K], wt fp16 [num_classes, K], bias float32 [num_classes] -> out float32
  [N, num_classes] = x @ wt^T + bias."""
  n, k = x.shape
  m = wt.shape[0]
  if wt.shape[1] != k or tuple(bias.shape) != (m,) or tuple(out.shape) != (n, m):
    raise ValueError('dense: x %s, wt %s, bias %s, out %s do not agree'
                     % (tuple(x.shape), tuple(wt.shape), tuple(bias.shape), tuple(out.shape)))
  _lib.call('edet_dense', _ptr(x, torch.float32), _ptr(wt, torch.float16),
            _ptr(bias, torch.float32), _ptr(out, torch.float32), n, k, m, _stream())


CLS_BILINEAR, CLS_BICUBIC = _lib.CLS_BILINEAR, _lib.CLS_BICUBIC
CLS_DESC_WORDS = 8      # int32 words of one edet_cls_image row: offset (2 words), h, w, y0, x0, crop_h, crop_w
SOFTMAX_TOPK_MAX_K = 32


def cls_preprocess(images, desc, out, mode, bicubic_table=None):
  """Classification eval pre-process of a (ragged) request in one launch: images uint8 (every image
  packed back to back, HWC), desc int32 [N, 8] edet_cls_image rows (byte offset into `images`, h,
  w, crop window; the caller keeps every window inside `images`), out float32 [N, S, S, 3]; mode
  CLS_BILINEAR, or CLS_BICUBIC with bicubic_table float32 [2050] (see edet_cls_preprocess)."""
  n, s = out.shape[0], out.shape[1]
  if tuple(out.shape) != (n, s, s, 3) or tuple(desc.shape) != (n, CLS_DESC_WORDS):
    raise ValueError('cls_preprocess: out %s must be [N, S, S, 3] and desc %s [N, %d]'
                     % (tuple(out.shape), tuple(desc.shape), CLS_DESC_WORDS))
  if mode == CLS_BICUBIC and (bicubic_table is None or bicubic_table.numel() != 2050):
    raise ValueError('cls_preprocess: the bicubic mode needs the float32 [2050] coefficient table')
  _lib.call('edet_cls_preprocess', _ptr(images, torch.uint8), _ptr(desc, torch.int32), n, s, mode,
            _ptr(bicubic_table, torch.float32), _ptr(out, torch.float32), _stream())


def softmax_topk(logits, probs, classes):
  """logits float32 [N, C] -> probs float32 [N, k], classes int32 [N, k]: the k largest logits by
  (logit descending, class ascending) and their softmax probabilities, 1 <= k <= min(C, 32)."""
  n, c = logits.shape
  k = probs.shape[1] if probs.dim() == 2 else -1
  if tuple(probs.shape) != (n, k) or tuple(classes.shape) != (n, k):
    raise ValueError('softmax_topk: probs %s and classes %s must be [%d, k]'
                     % (tuple(probs.shape), tuple(classes.shape), n))
  _lib.call('edet_softmax_topk', _ptr(logits, torch.float32), n, c, k, _ptr(probs, torch.float32),
            _ptr(classes, torch.int32), _stream())


SEG_MASK_WORDS = 6      # int32 words of one edet_seg_mask_image row: offset (2 words), h, w, scaled_h, scaled_w
SEG_MAX_CLASSES = 256   # the masks are uint8


def seg_masks(logits, num_classes, grid_factor, table, max_hw, out):
  """Masks at each image's own size in one launch: logits fp16 [N, Hs, Ws, ld] (the segmentation
  head's output, ld % 8 == 0), table int32 [N, 6] edet_seg_mask_image rows (byte offset of the mask
  in `out`, h, w, scaled_h, scaled_w; the caller keeps every mask inside `out`), max_hw the largest
  (h, w) of the table, out uint8 -> out[offset:offset + h*w] = the h x w arg-max mask of each image,
  sampled at the nearest cell of the letterboxed input (see edet_seg_masks)."""
  if not 1 <= num_classes <= SEG_MAX_CLASSES:
    raise ValueError('seg_masks: %d classes do not fit a uint8 mask (1..%d)'
                     % (num_classes, SEG_MAX_CLASSES))
  if logits.dim() != 4 or logits.shape[-1] % 8 or logits.shape[-1] < num_classes:
    raise ValueError('seg_masks: logits %s must be [N, Hs, Ws, ld], ld a multiple of 8 >= %d'
                     % (tuple(logits.shape), num_classes))
  n, hs, ws, ld = logits.shape
  if tuple(table.shape) != (n, SEG_MASK_WORDS):
    raise ValueError('seg_masks: table %s must be [%d, %d]' % (tuple(table.shape), n, SEG_MASK_WORDS))
  _lib.call('edet_seg_masks', _ptr(logits, torch.float16), n, hs, ws, ld, num_classes,
            int(grid_factor), _ptr(table, torch.int32), int(max_hw[0]), int(max_hw[1]),
            _ptr(out, torch.uint8), _stream())


CLASS_ARGMAX_COLS = 96  # columns per anchor of the padded class-head weights (edet_class_argmax)


def class_argmax(a, wt_padded, bias_padded, scores, classes, anchor_begin, num_anchors):
  """Class-predict 1x1 conv fused with the class half of pre-NMS for one level: a fp16
  [N,H,W,lda] (the depthwise output of the predict layer, F = wt_padded.shape[-1] <= lda
  channels), wt_padded fp16 [num_anchors*96, F] (row a*96 + c = class c of anchor a, zero rows
  for c >= num_classes), bias_padded fp32 [num_anchors*96] (-inf on the pad rows) -> scores fp32 /
  classes i32 [N, total_anchors] at anchors anchor_begin + pixel*num_anchors + a."""
  n, h, w, lda = a.shape
  f = wt_padded.shape[-1]
  assert wt_padded.shape == (num_anchors * CLASS_ARGMAX_COLS, f) and f <= lda
  _lib.call('edet_class_argmax', _ptr(a, torch.float16), lda, _ptr(wt_padded, torch.float16),
            _ptr(bias_padded, torch.float32), _ptr(scores, torch.float32),
            _ptr(classes, torch.int32), anchor_begin, scores.shape[1], num_anchors, n, h * w, f,
            _stream())


def pre_nms(cls_levels, box_levels, level_hw, num_anchors, num_classes, anchors, boxes, scores,
            classes):
  """cls_levels[l] fp16 [N,H_l,W_l,ld_cls]; boxes fp32 [N,A,4], scores fp32 [N,A], classes i32.
  cls_levels=None: boxes only (scores / classes were written by class_argmax)."""
  levels = len(box_levels)
  n = box_levels[0].shape[0]
  ld_box = box_levels[0].shape[-1]
  if cls_levels is None:
    ld_cls = _round8(num_anchors * num_classes)
    cls_p = None
    scores = classes = None
  else:
    ld_cls = cls_levels[0].shape[-1]
    cls_p = (ctypes.c_void_p * levels)(*[_ptr(t, torch.float16).value for t in cls_levels])
  box_p = (ctypes.c_void_p * levels)(*[_ptr(t, torch.float16).value for t in box_levels])
  hw = (ctypes.c_int * (2 * levels))(*[v for pair in level_hw for v in pair])
  _lib.call('edet_pre_nms', cls_p, box_p, hw, levels, ld_cls, ld_box, num_anchors, num_classes,
            _ptr(anchors, torch.float32), _ptr(boxes, torch.float32),
            _ptr(scores, torch.float32), _ptr(classes, torch.int32), n, _stream())


def pre_nms_topk(cls_levels, box_levels, level_hw, num_anchors, num_classes, anchors, boxes, scores,
                 classes, indices):
  """Top-k pre-NMS (max_nms_inputs = scores.shape[1]): boxes fp32 [N,k,4], scores fp32 [N,k],
  classes / indices i32 [N,k]."""
  levels = len(cls_levels)
  n, k = scores.shape
  ld_cls, ld_box = cls_levels[0].shape[-1], box_levels[0].shape[-1]
  cls_p = (ctypes.c_void_p * levels)(*[_ptr(t, torch.float16).value for t in cls_levels])
  box_p = (ctypes.c_void_p * levels)(*[_ptr(t, torch.float16).value for t in box_levels])
  hw = (ctypes.c_int * (2 * levels))(*[v for pair in level_hw for v in pair])
  _lib.call('edet_pre_nms_topk', cls_p, box_p, hw, levels, ld_cls, ld_box, num_anchors, num_classes,
            _ptr(anchors, torch.float32), k, _ptr(boxes, torch.float32), _ptr(scores, torch.float32),
            _ptr(classes, torch.int32), _ptr(indices, torch.int32), n, _stream())


def nms_work_bytes(n, k):
  return _lib.load().edet_nms_work_bytes(n, k)


def nms_v5(boxes, scores, classes, image_scales, image_id_base, max_output_size, iou_threshold,
           score_threshold, soft_nms_sigma, clip_hw, detections, sel_index, valid, work):
  n, k = scores.shape
  _lib.call('edet_nms_v5', _ptr(boxes, torch.float32), _ptr(scores, torch.float32),
            _ptr(classes, torch.int32), _ptr(image_scales, torch.float32), image_id_base, n, k,
            max_output_size, ctypes.c_float(iou_threshold), ctypes.c_float(score_threshold),
            ctypes.c_float(soft_nms_sigma), ctypes.c_float(clip_hw[0]),
            ctypes.c_float(clip_hw[1]), _ptr(detections, torch.float32),
            _ptr(sel_index, torch.int32), _ptr(valid, torch.int32), _ptr(work), _stream())


NMS_METHODS = {'hard': _lib.NMS_HARD, '': _lib.NMS_HARD, None: _lib.NMS_HARD, 'diou': _lib.NMS_DIOU,
               'gaussian': _lib.NMS_GAUSSIAN, 'linear': _lib.NMS_LINEAR}


def per_class_nms(boxes, scores, classes, image_ids, image_scales, num_classes, max_boxes_to_draw,
                  method, iou_thresh, detections, keep_index, num_valid, sigma=None,
                  score_thresh=None, work=None):
  """nms_np.per_class_nms on the device: boxes fp32 [N,K,4] (ymin,xmin,ymax,xmax), scores fp32
  [N,K], classes i32 [N,K], image_ids / image_scales fp32 [N] or None -> detections fp32
  [N,max_boxes,7], keep_index i32 [N,max_boxes], num_valid i32 [N].  None / 0 thresholds take
  nms_np's defaults (`x or default`, nms_np.py:43, 100, 148-150); the soft methods need `work`,
  a float32 [N,K] workspace (allocated here when not given)."""
  n, k = scores.shape
  if method not in NMS_METHODS:
    raise ValueError('Unknown NMS method: {}'.format(method))
  code = NMS_METHODS[method]
  soft = code in (_lib.NMS_GAUSSIAN, _lib.NMS_LINEAR)
  thr = float(iou_thresh) if iou_thresh else (0.3 if soft else 0.5)
  sig = float(sigma) if sigma else 0.5
  sth = float(score_thresh) if score_thresh else 0.001
  if soft and work is None:
    work = torch.empty(n, k, dtype=torch.float32, device=scores.device)
  _lib.call('edet_per_class_nms', _ptr(boxes, torch.float32), _ptr(scores, torch.float32),
            _ptr(classes, torch.int32), _ptr(image_ids, torch.float32),
            _ptr(image_scales, torch.float32), n, k, num_classes, max_boxes_to_draw, code,
            ctypes.c_float(thr), ctypes.c_float(sig), ctypes.c_float(sth),
            _ptr(work, torch.float32), _ptr(detections, torch.float32),
            _ptr(keep_index, torch.int32), _ptr(num_valid, torch.int32), _stream())


WBF_MAX_ROWS = 1024     # EDET_WBF_MAX_ROWS: num_models * rows of one image


def wbf(detections, num_models, num_classes, clusters, num_clusters, mirrored_mask=0,
        image_scales=None, width=1):
  """Weighted box fusion (tf2/wbf.py ensemble_detections) of every image in one launch:
  detections fp32 [num_models * N, rows, 7] (model m of image i at block m * N + i, per-class NMS
  rows [image_id, x1, y1, x2, y2, score, class]) -> clusters fp32 [N, num_models * rows, 7]
  (sorted by score, then padding rows [0, 0, 0, 0, 0, 0, -1]) and num_clusters i32 [N].  Models
  whose bit is set in `mirrored_mask` are un-mirrored first about image_scales fp32 [N] * width
  (see edet_wbf)."""
  if detections.dim() != 3 or detections.shape[2] != 7 or detections.shape[0] % num_models:
    raise ValueError('wbf: detections %s must be [num_models * N, rows, 7], num_models = %d'
                     % (tuple(detections.shape), num_models))
  n, rows = detections.shape[0] // num_models, detections.shape[1]
  if tuple(clusters.shape) != (n, num_models * rows, 7) or tuple(num_clusters.shape) != (n,):
    raise ValueError('wbf: clusters %s must be [%d, %d, 7] and num_clusters %s [%d]'
                     % (tuple(clusters.shape), n, num_models * rows, tuple(num_clusters.shape), n))
  if image_scales is not None and tuple(image_scales.shape) != (n,):
    raise ValueError('wbf: image_scales %s must be [%d]' % (tuple(image_scales.shape), n))
  _lib.call('edet_wbf', _ptr(detections, torch.float32), n, rows, num_models, int(mirrored_mask),
            _ptr(image_scales, torch.float32), int(width), int(num_classes),
            _ptr(clusters, torch.float32), _ptr(num_clusters, torch.int32), _stream())
