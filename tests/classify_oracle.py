"""CPU oracle of the EfficientNet V1 / V2 classification serving path (TEST INFRASTRUCTURE ONLY):
the eval pre-process of both recipes and the softmax top-k output, restated in numpy float32 in
the reference's order of operations (every op one float32 rounding, as the device computes).

Restated from /root/reference/efficientnetv2:
  preprocessing.py:58-70     preprocess_for_eval: crop only when image_size < 320; crop side
                             int32(ratio * float32(min(h, w))), ratio = S / (S + 32) as a float32
                             constant; offsets (h - crop) // 2; tf.image.resize (bilinear,
                             half-pixel centres, no antialias)
  preprocessing.py:131-157   'effnetv1_' augname -> legacy recipe; else (x - 128) / 128
  preprocess_legacy.py:110-127   _decode_and_center_crop: same crop side, offsets
                             (h - crop + 1) // 2; _resize_image :77-82 -> tf.image.resize_bicubic
                             (TF1: align_corners = half_pixel_centers = False)
  preprocess_legacy.py:239-243   (x - mean_rgb) / stddev_rgb, ImageNet statistics * 255 as float32
TensorFlow's own kernels (what tf.image.resize / resize_bicubic compute on the CPU):
  bilinear: in = (out + 0.5) * (in_size / out_size) - 0.5, lower = max(floor(in), 0),
            upper = min(ceil(in), in_size - 1), lerp = in - floor(in); top / bottom along x, then y
  bicubic:  coefficient table of 1025 steps, a = -0.75, evaluated in double, stored as float;
            in = out * (in_size / out_size), i = floor(in), offset = lrintf((in - i) * 1024);
            weights t[2o+1], t[2o], t[2(1024-o)], t[2(1024-o)+1] on taps i-1..i+2 clamped to the
            image; each of the 4 columns interpolated vertically, then the row; products summed
            left to right.
Parity status: "parity unpinned" against TensorFlow's kernels (TensorFlow cannot be installed
here); tests/test_classify_preprocess_pins.py holds these restatements to hand-derived fixtures and
to plain float64 loops.

Softmax top-k (tf.nn.softmax, tf.math.top_k): float64 softmax of the float32 logits; classes by a
stable sort of (-logit, index), top_k's documented tie rule (equal values: lower index first).
"""
import numpy as np

f32 = np.float32
MEAN_RGB = np.array([0.485 * 255, 0.456 * 255, 0.406 * 255], np.float32)
STDDEV_RGB = np.array([0.229 * 255, 0.224 * 255, 0.225 * 255], np.float32)
TABLE_SIZE = 1024


def crop_window(h, w, image_size, legacy):
  """(y0, x0, crop_h, crop_w); raises ValueError when the crop is empty."""
  if not legacy and image_size >= 320:
    return 0, 0, h, w
  crop = int(f32(image_size / (image_size + 32)) * f32(min(h, w)))
  if crop < 1:
    raise ValueError('empty crop')
  if legacy:
    return (h - crop + 1) // 2, (w - crop + 1) // 2, crop, crop
  return (h - crop) // 2, (w - crop) // 2, crop, crop


def bicubic_table():
  """float32 [2 * 1025]: TF's GetCoeffsTable(use_keys_cubic=false)."""
  t = np.zeros(2 * (TABLE_SIZE + 1), np.float32)
  a = -0.75
  for i in range(TABLE_SIZE + 1):
    x = i * 1.0 / TABLE_SIZE
    t[2 * i] = ((a + 2) * x - (a + 3)) * x * x + 1
    x += 1.0
    t[2 * i + 1] = ((a * x - 5 * a) * x + 8 * a) * x - 4 * a
  return t


TABLE = bicubic_table()


def bilinear_taps(out_size, in_size):
  scale = f32(in_size) / f32(out_size)
  src = (np.arange(out_size, dtype=np.float32) + f32(0.5)) * scale - f32(0.5)
  fl = np.floor(src)
  lo = np.maximum(fl, 0).astype(np.int64)
  hi = np.minimum(np.ceil(src), in_size - 1).astype(np.int64)
  return lo, hi, (src - fl).astype(np.float32)


def resize_bilinear(img, out_h, out_w):
  """float32 [h, w, 3] -> float32 [out_h, out_w, 3] (tf.image.resize, bilinear)."""
  img = np.asarray(img, np.float32)
  y0, y1, ly = bilinear_taps(out_h, img.shape[0])
  x0, x1, lx = bilinear_taps(out_w, img.shape[1])
  lx, ly = lx[None, :, None], ly[:, None, None]
  top = img[y0][:, x0] + (img[y0][:, x1] - img[y0][:, x0]) * lx
  bot = img[y1][:, x0] + (img[y1][:, x1] - img[y1][:, x0]) * lx
  return top + (bot - top) * ly


def bicubic_offsets(out_size, in_size):
  """(floor of the source coordinate, table offset) per output index, legacy scaler."""
  scale = f32(in_size) / f32(out_size)
  src = np.arange(out_size, dtype=np.float32) * scale
  fi = np.floor(src)
  return fi, np.rint((src - fi) * f32(TABLE_SIZE)).astype(np.int64)     # lrintf: half to even


def bicubic_taps(out_size, in_size):
  """indices int64 [out, 4] and weights float32 [out, 4] of TF1 resize_bicubic (legacy scaler)."""
  fi, off = bicubic_offsets(out_size, in_size)
  w = np.stack([TABLE[2 * off + 1], TABLE[2 * off], TABLE[2 * (TABLE_SIZE - off)],
                TABLE[2 * (TABLE_SIZE - off) + 1]], 1)
  idx = np.clip(fi.astype(np.int64)[:, None] + np.arange(-1, 3)[None, :], 0, in_size - 1)
  return idx, w.astype(np.float32)


def resize_bicubic(img, out_h, out_w):
  """float32 [h, w, 3] -> float32 [out_h, out_w, 3] (TF1 resize_bicubic, TF's CPU kernel)."""
  img = np.asarray(img, np.float32)
  yi, wy = bicubic_taps(out_h, img.shape[0])
  xi, wx = bicubic_taps(out_w, img.shape[1])
  cols = []
  for j in range(4):                     # vertical interpolation at each x tap
    p = img[:, xi[:, j]]                 # [h, out_w, 3]
    s = p[yi[:, 0]] * wy[:, 0, None, None]
    for r in range(1, 4):
      s = s + p[yi[:, r]] * wy[:, r, None, None]
    cols.append(s)
  v = wx[None, :, 0, None] * cols[0]
  for j in range(1, 4):
    v = v + wx[None, :, j, None] * cols[j]
  return v.astype(np.float32)


def preprocess_window(image, image_size, legacy, window):
  """uint8 [h, w, 3], an explicit crop window (y0, x0, crop_h, crop_w) -> float32 [S, S, 3]."""
  y0, x0, ch, cw = window
  crop = np.asarray(image)[y0:y0 + ch, x0:x0 + cw].astype(np.float32)
  if legacy:
    return (resize_bicubic(crop, image_size, image_size) - MEAN_RGB) / STDDEV_RGB
  return (resize_bilinear(crop, image_size, image_size) - f32(128.0)) / f32(128.0)


def preprocess_image(image, image_size, legacy):
  """preprocessing.preprocess_image(image, image_size, is_training=False, augname) for a decoded
  uint8 image; legacy = augname.startswith('effnetv1_')."""
  h, w = np.shape(image)[:2]
  return preprocess_window(image, image_size, legacy, crop_window(h, w, image_size, legacy))


def softmax_topk(logits, k):
  """float32 [N, C] -> (float64 probs [N, k], int64 classes [N, k])."""
  x = np.asarray(logits, np.float32)
  order = np.stack([np.lexsort((np.arange(x.shape[1]), -x[i].astype(np.float64)))[:k]
                    for i in range(x.shape[0])])
  x64 = x.astype(np.float64)
  e = np.exp(x64 - x64.max(1, keepdims=True))
  p = e / e.sum(1, keepdims=True)
  return np.take_along_axis(p, order, 1), order
