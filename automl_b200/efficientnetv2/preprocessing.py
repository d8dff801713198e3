"""Eval pre-process of the EfficientNet V1 / V2 classifiers on the device, for decoded uint8 images:
the reference's efficientnetv2/preprocessing.py::preprocess_image (:120-157) with
is_training=False.

  image = preprocessing.preprocess_image(uint8_hw3, 384, augname='randaug')   # float32 [S, S, 3]

Two recipes, chosen by `augname` as the reference does (:133):
  * 'effnetv1_*' (every V1 model and efficientnetv2-b0..b3): the legacy recipe of
    preprocess_legacy.py:110-127, 184-244 -- a center crop of S / (S + 32) of the shorter side,
    offsets rounded up, TF1 resize_bicubic (no half-pixel centres) and (x - mean) / stddev with the
    ImageNet statistics;
  * anything else (efficientnetv2-s/m/l/xl use 'randaug'): preprocess_for_eval :58-70 -- the same
    crop with offsets rounded down, only when S < 320, tf.image.resize bilinear (half-pixel
    centres), then (x - 128) / 128 (:153).
The host computes the crop windows (`crop_window`); the resize and the normalisation run in one
edet_cls_preprocess launch per request.  Decoding (JPEG / PNG) and the training recipes are out
of scope.
"""
import numpy as np
import torch

from automl_b200 import ops

BICUBIC_TABLE_SIZE = 1024
_TABLES = {}


def is_legacy(augname):
  """preprocessing.py:133: an 'effnetv1_' augname selects the legacy recipe."""
  return bool(augname) and augname.startswith('effnetv1_')


def crop_window(h, w, image_size, legacy):
  """(y0, x0, crop_h, crop_w) of the eval crop of an h x w image.  The crop side is
  int32(float32(S / (S + 32)) * float32(min(h, w))) (the Python ratio meets a float32 tensor and
  the product is truncated, preprocessing.py:62-65, preprocess_legacy.py:116-120); the offsets
  are (h - crop) // 2 (bilinear recipe, :66) or (h - crop + 1) // 2 (legacy, :122-123).  The
  bilinear recipe crops only when S < 320 (:60) and otherwise resizes the whole image."""
  h, w, image_size = int(h), int(w), int(image_size)
  if not legacy and image_size >= 320:
    return 0, 0, h, w
  ratio = np.float32(image_size / (image_size + 32))
  crop = int(ratio * np.float32(min(h, w)))
  if crop < 1:
    raise ValueError('a %dx%d image has an empty %d-pixel eval crop' % (h, w, image_size))
  r = 1 if legacy else 0
  return (h - crop + r) // 2, (w - crop + r) // 2, crop, crop


def bicubic_table():
  """TF's resize_bicubic coefficient table (a = -0.75, kTableSize = 1024): float32 [2 * 1025],
  entry i at x = i / 1024: t[2i] = ((a+2)x - (a+3))x^2 + 1, t[2i+1] = ((a(x+1) - 5a)(x+1) + 8a)(x+1)
  - 4a, evaluated in double and stored as float."""
  a = -0.75
  x = np.arange(BICUBIC_TABLE_SIZE + 1, dtype=np.float64) / BICUBIC_TABLE_SIZE
  t = np.empty(2 * (BICUBIC_TABLE_SIZE + 1), np.float32)
  t[0::2] = ((a + 2) * x - (a + 3)) * x * x + 1
  x1 = x + 1.0
  t[1::2] = ((a * x1 - 5 * a) * x1 + 8 * a) * x1 - 4 * a
  return t


def device_table(device):
  """The bicubic table on `device`, uploaded once per device."""
  key = str(torch.device(device))
  if key not in _TABLES:
    _TABLES[key] = torch.from_numpy(bicubic_table()).to(device)
  return _TABLES[key]


def image_table(shapes, image_size, legacy):
  """Descriptor rows of a request whose images (h, w) are packed back to back in this order:
  int32 [N, 8] edet_cls_image rows and the packed byte count."""
  desc = np.zeros((len(shapes), ops.CLS_DESC_WORDS), np.int32)
  offset = 0
  for i, (h, w) in enumerate(shapes):
    if h < 1 or w < 1:
      raise ValueError('empty image (%d x %d)' % (h, w))
    desc[i, 2:] = (h, w) + crop_window(h, w, image_size, legacy)
    desc[i:i + 1, :2].view(np.int64)[0, 0] = offset
    offset += 3 * h * w
  return desc, offset


def check_image(image):
  """A decoded image: uint8 [h, w, 3] (numpy array or torch tensor)."""
  dtype = image.dtype
  if not (dtype == np.uint8 or dtype == torch.uint8) or len(image.shape) != 3 or image.shape[2] != 3:
    raise ValueError('expected a uint8 [h, w, 3] image, got %s %s' % (dtype, tuple(image.shape)))


def _check_dtype(image_dtype):
  """None or a float32 dtype (numpy, torch, or anything with a numpy `as_numpy_dtype`)."""
  if image_dtype is None:
    return
  if isinstance(image_dtype, torch.dtype):
    ok = image_dtype == torch.float32
  else:
    try:
      ok = np.dtype(getattr(image_dtype, 'as_numpy_dtype', image_dtype)) == np.float32
    except TypeError:
      ok = False
  if not ok:
    raise ValueError('only float32 output is supported, got %s' % (image_dtype,))


def preprocess_image(image, image_size, is_training=False, image_dtype=None, augname=None,
                     device='cuda:0'):
  """preprocessing.preprocess_image for eval: a decoded uint8 [h, w, 3] image (numpy or torch) ->
  float32 [S, S, 3] device tensor on `device`, computed on the current stream."""
  if is_training:
    raise NotImplementedError('the training pre-process (random crop, flip, AutoAugment / '
                              'RandAugment) is out of scope')
  _check_dtype(image_dtype)
  if not isinstance(image, torch.Tensor):
    image = np.asarray(image)
  check_image(image)
  size = int(image_size)
  legacy = is_legacy(augname)
  h, w = int(image.shape[0]), int(image.shape[1])
  desc, _ = image_table([(h, w)], size, legacy)
  raw = torch.as_tensor(image).to(device).contiguous()
  out = torch.empty((1, size, size, 3), dtype=torch.float32, device=device)
  with torch.cuda.device(out.device):
    ops.cls_preprocess(raw, torch.from_numpy(desc).to(device), out,
                       ops.CLS_BICUBIC if legacy else ops.CLS_BILINEAR,
                       device_table(device) if legacy else None)
  return out[0]
