"""Tensor-level wrappers over the C-ABI (torch tensors are only device-memory containers).

Every function enqueues on the CURRENT torch CUDA stream, allocates nothing except where
stated, and raises if the tensors are not CUDA / not contiguous / misaligned.  There is no CPU
implementation behind any of them.
"""
import ctypes

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


def fuse_dw(specs, dw_w, out, act):
  n, h, wd, c = out.shape
  for t, _, _, _ in specs:
    _ptr(t, torch.float16)
  arr = make_fuse_inputs(specs)
  _lib.call('edet_fuse_dw', arr, len(specs), _ptr(dw_w, torch.float32),
            _ptr(out, torch.float16), n, h, wd, c, act, _stream())


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


CLASS_ARGMAX_COLS = 96   # columns per anchor of the padded class-head weights (edet_class_argmax)


def class_argmax(a, wt_padded, bias_padded, scores, classes, anchor_begin, num_anchors):
  """Class-predict 1x1 conv fused with the class half of pre-NMS for one level: a fp16
  [N,H,W,F] (the depthwise output of the predict layer), wt_padded fp16 [num_anchors*96, F] (row
  a*96 + c = class c of anchor a, zero rows for c >= num_classes), bias_padded fp32
  [num_anchors*96] (-inf on the pad rows) -> scores fp32 / classes i32 [N, total_anchors] at
  anchors anchor_begin + pixel*num_anchors + a."""
  n, h, w, f = a.shape
  assert wt_padded.shape == (num_anchors * CLASS_ARGMAX_COLS, f)
  _lib.call('edet_class_argmax', _ptr(a, torch.float16), f, _ptr(wt_padded, torch.float16),
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
