"""Weighted box fusion for flip test-time augmentation, restated in plain numpy (float32 scalars,
every operation rounded on its own) from the reference:

  /root/reference/efficientdet/tf2/wbf.py:19-95       vectorized_iou, find_matching_cluster,
                                                       average_detections, ensemble_detections
  /root/reference/efficientdet/tf2/postprocess.py:560-573   un-mirroring a flipped input's rows

tests/test_wbf_pins.py holds this file to the goldens that tests/golden/make_wbf_golden.py records
by running the unmodified wbf.py; the GPU tests hold edet_wbf to this file.  Test infrastructure."""
import numpy as np

F32 = np.float32
THRESH = F32(0.55)          # wbf.py:45; a float32 compared with 0.55 decides alike in float32 and float64


def unmirror(rows, image_scale, width):
  """postprocess.py:560-573 on [R, 7] rows of a mirrored input: ow = image_scale * width (float32),
  x1' = ow - x2, x2' = ow - x1."""
  rows = np.asarray(rows, F32)
  ow = F32(image_scale) * F32(width)
  out = rows.copy()
  out[:, 1] = ow - rows[:, 3]
  out[:, 3] = ow - rows[:, 1]
  return out


def stack_models(blocks, mirrored_mask, image_scale, width):
  """concat(model 0 rows, model 1 rows, ...) of one image, mirrored models un-mirrored."""
  return np.concatenate([unmirror(b, image_scale, width) if (mirrored_mask >> m) & 1 else np.asarray(b, F32)
                         for m, b in enumerate(blocks)], axis=0)


def iou(avg, d):
  """vectorized_iou (wbf.py:19-36) of one cluster average and one row, float32, numpy's NaN rules
  (np.maximum / np.minimum propagate NaN)."""
  x11, y11, x12, y12 = avg[1], avg[2], avg[3], avg[4]
  x21, y21, x22, y22 = d[1], d[2], d[3], d[4]
  xa, ya = np.maximum(x11, x21), np.maximum(y11, y21)
  xb, yb = np.minimum(x12, x22), np.minimum(y12, y22)
  inter = np.maximum(xb - xa, F32(0)) * np.maximum(yb - ya, F32(0))
  area_a = (x12 - x11) * (y12 - y11)
  area_b = (x22 - x21) * (y22 - y21)
  return inter / (area_a + area_b - inter)


def _average(members, num_models):
  """average_detections (wbf.py:51-67); sums sequential in join order, starting from the first
  term (tf.math.reduce_sum of one element is that element)."""
  s = members[0][5]
  xs = [members[0][c] * s for c in range(1, 5)]
  for d in members[1:]:
    s = s + d[5]
    xs = [xs[c - 1] + d[c] * d[5] for c in range(1, 5)]
  n = len(members)
  weight = F32(min(1, n / num_models))       # Python float, rounded to float32 by the multiply
  return np.array([members[0][0], xs[0] / s, xs[1] / s, xs[2] / s, xs[3] / s,
                   (s / F32(n)) * weight, members[0][6]], F32)


def ensemble(rows, num_classes, num_models):
  """ensemble_detections (wbf.py:70-95) of one image's [R, 7] rows -> float32 [k, 7] clusters.
  Only classes cid in range(num_classes) are fused (class num_classes of nms_np's 1-based rows is
  dropped, class 0 holds its dummy rows); rows of a class in input order; clusters class by class
  in creation order, then a stable sort by score, descending."""
  rows = np.asarray(rows, F32)
  out = []
  with np.errstate(all='ignore'):
    for cid in range(num_classes):
      members, avgs = [], []
      for d in rows[rows[:, 6] == cid]:
        k = -1
        if avgs:
          ious = np.array([iou(a, d) for a in avgs], F32)
          if not ious.max() < THRESH:          # np.max propagates NaN: a NaN maximum joins
            k = int(np.argmax(ious))           # first index of the maximum, first NaN wins
        if k == -1:
          members.append([d])
          avgs.append(_average([d], num_models))
        else:
          members[k].append(d)
          avgs[k] = _average(members[k], num_models)
      out.extend(avgs)
  out.sort(reverse=True, key=lambda a: a[5])
  return np.array(out, F32).reshape(-1, 7)


def same_bits(a, b):
  """Bit-for-bit equality of float32 arrays, any NaN equal to any NaN."""
  a, b = np.asarray(a, F32), np.asarray(b, F32)
  if a.shape != b.shape:
    return False
  na, nb = np.isnan(a), np.isnan(b)
  return bool((na == nb).all() and (a.view(np.uint32)[~na] == b.view(np.uint32)[~nb]).all())
