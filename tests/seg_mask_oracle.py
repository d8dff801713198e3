"""Numpy restatement of the segmentation masks (TEST INFRASTRUCTURE ONLY; imports nothing of the
product).  The reference stops at the logits; its demo takes tf.argmax(pred, -1) at the network
resolution (tf2/segmentation.py:25-27).  Each image's mask is at its own size h x w: pixel (y, x)
takes the arg-max over the classes at the nearest logits cell of its region of the letterboxed
input, the image's scaled sh x sw top-left corner, with the logits grid f times coarser than the
input:
  cell_y = min(((2y + 1) * sh) // (2 * h * f), Hs - 1)      (x alike; integers only)
  mask[y, x] = np.argmax(logits[i, cell_y, cell_x, :C])    (first index on ties, first NaN wins)
"""
import numpy as np


def cells(n, scaled, f, limit):
  """Cell index of each of the n output pixels along one axis (int64 [n])."""
  p = np.arange(n, dtype=np.int64)
  return np.minimum((2 * p + 1) * scaled // (2 * n * f), limit - 1)


def cells_float64(n, scaled, f, limit):
  """The same in float64: floor((p + 0.5) * scaled / n / f)."""
  p = np.arange(n, dtype=np.float64)
  return np.minimum(np.floor((p + 0.5) * scaled / n / f).astype(np.int64), limit - 1)


def class_map(logits, num_classes):
  """uint8 [N, Hs, Ws]: np.argmax over the first num_classes channels."""
  return np.argmax(np.asarray(logits)[..., :num_classes], axis=-1).astype(np.uint8)


def masks(logits, num_classes, f, images):
  """logits [N, Hs, Ws, >= C] (fp16 or any numpy float), images [(h, w, sh, sw)] per image ->
  list of uint8 [h, w] masks."""
  cmap = class_map(logits, num_classes)
  hs, ws = cmap.shape[1:3]
  out = []
  for i, (h, w, sh, sw) in enumerate(images):
    cy, cx = cells(h, sh, f, hs), cells(w, sw, f, ws)
    out.append(cmap[i][cy[:, None], cx[None, :]])
  return out


def pixels(logits, num_classes, f, image, index, ys, xs):
  """Mask values of image `index` = (h, w, sh, sw) at pixels (ys[k], xs[k]) only (for masks too
  large to build on the host)."""
  h, w, sh, sw = image
  hs, ws = logits.shape[1:3]
  ys, xs = np.asarray(ys, np.int64), np.asarray(xs, np.int64)
  cy = np.minimum((2 * ys + 1) * sh // (2 * h * f), hs - 1)
  cx = np.minimum((2 * xs + 1) * sw // (2 * w * f), ws - 1)
  return np.argmax(np.asarray(logits)[index, cy, cx, :num_classes], axis=-1).astype(np.uint8)
