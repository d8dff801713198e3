"""Generates tests/golden/wbf.npz: weighted box fusion for flip test-time augmentation, computed by
the UNMODIFIED reference /root/reference/efficientdet/tf2/wbf.py (ensemble_detections) under a
small numpy-backed `tensorflow` stand-in, on inputs from the real
/root/reference/efficientdet/nms_np.py (per_class_nms) and on hand-built cases.

The stand-in computes in float32 throughout.  Its tf.math.reduce_sum is sequential, starting from
the first element (TensorFlow does not pin its summation order; DESIGN.md section 2), and
reduce_mean is that sum over the float32 count.  numpy >= 2 keeps `float32 * Python float` and
`float32 < 0.55` in float32 (NEP 50); main() checks that no value left float32.

Each case stores the raw per-model blocks (`<case>/det` [num_models, rows, 7]), `<case>/meta`
[num_models, mirrored_mask, num_classes, width], `<case>/scale` (the image_scale) and
`<case>/out`, the reference's [k, 7] clusters of concat(model rows), mirrored models un-mirrored
first as tf2/postprocess.py:560-573 does it.  Run from the repo root:
  python tests/golden/make_wbf_golden.py
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/efficientdet'
F32 = np.float32


def _reduce_sum(x):
  x = np.asarray(x).ravel()
  acc = x[0]
  for v in x[1:]:
    acc = acc + v
  return acc


def tf_standin():
  tf = types.ModuleType('tensorflow')
  tf.split = lambda x, n, axis=0: np.split(np.asarray(x), n, axis=axis)
  tf.maximum, tf.minimum = np.maximum, np.minimum
  tf.reshape = lambda x, s: np.reshape(x, s)
  tf.stack = lambda xs: np.stack([np.asarray(x) for x in xs])
  tf.where = lambda c: np.argwhere(np.asarray(c))
  tf.equal = lambda a, b: np.asarray(a) == b
  tf.gather_nd = lambda p, idx: np.asarray(p)[tuple(np.asarray(idx).T)]
  tf.argmax = lambda x: np.argmax(x)
  tf.math = types.SimpleNamespace(
      reduce_max=lambda x: np.max(x), reduce_sum=_reduce_sum,
      reduce_mean=lambda x: _reduce_sum(x) / F32(np.asarray(x).size))
  return tf


def import_reference():
  sys.modules['tensorflow'] = tf_standin()
  spec = importlib.util.spec_from_file_location('ref_wbf', os.path.join(REF, 'tf2', 'wbf.py'))
  wbf = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(wbf)
  sys.path.insert(0, REF)
  import nms_np  # pylint: disable=g-import-not-at-top
  return wbf, nms_np


def unmirror(rows, image_scale, width):
  """tf2/postprocess.py:560-573 in float32."""
  ow = F32(image_scale) * F32(width)
  return np.stack([rows[:, 0], ow - rows[:, 3], rows[:, 2], ow - rows[:, 1], rows[:, 4], rows[:, 5],
                   rows[:, 6]], axis=-1).astype(F32)


def run_reference(wbf, blocks, mirrored_mask, num_classes, width, scale):
  rows = np.concatenate([unmirror(b, scale, width) if (mirrored_mask >> m) & 1 else b
                         for m, b in enumerate(blocks)], axis=0).astype(F32)
  with np.errstate(all='ignore'):
    try:
      out = wbf.ensemble_detections({'num_classes': num_classes}, rows, len(blocks))
    except ValueError:          # np.stack([]): no row of a fused class
      out = np.zeros((0, 7), F32)
  out = np.asarray(out)
  assert out.dtype == F32, out.dtype
  return out.reshape(-1, 7)


def nms_pair_cases(nms_np, rng):
  """Per-class NMS rows of an image and of its jittered mirror (and a third jittered view)."""
  cases = {}
  width, num_classes, k, max_out = 256, 6, 90, 100
  configs = {'hard': dict(method='hard', iou_thresh=0.5, score_thresh=None, sigma=None),
             'gaussian': dict(method='gaussian', iou_thresh=None, score_thresh=0.001, sigma=0.5),
             'linear': dict(method='linear', iou_thresh=0.3, score_thresh=0.001, sigma=None)}
  for ci, (name, cfg) in enumerate(configs.items()):
    cfg = dict(cfg, max_output_size=max_out)
    for num_models in (1, 2, 3):
      y1, x1 = rng.uniform(0, 200, k), rng.uniform(0, 200, k)
      hw = rng.uniform(8, 64, (k, 2))
      boxes = np.stack([y1, x1, np.minimum(y1 + hw[:, 0], 256), np.minimum(x1 + hw[:, 1], 256)], 1)
      scores = rng.uniform(0, 1, k)
      classes = rng.integers(0, num_classes, k)
      scale = F32(rng.uniform(0.5, 3.0))
      image_id = 7 + ci
      blocks = []
      for m in range(num_models):
        b = boxes + rng.normal(0, 1.5, boxes.shape) * (m > 0)
        if m == 1:                       # the mirrored view: x -> width - x in the network frame
          b = np.stack([b[:, 0], width - b[:, 3], b[:, 2], width - b[:, 1]], 1)
        s = np.clip(scores + rng.normal(0, 0.02, k) * (m > 0), 0.0, 1.0)
        det = nms_np.per_class_nms(b.astype(F32), s.astype(F32), classes, np.array([image_id], F32),
                                   np.array([scale], F32), num_classes, max_out, cfg)
        blocks.append(np.asarray(det, F32))
      cases['nms_%s_m%d' % (name, num_models)] = (blocks, 0b10 if num_models > 1 else 0,
                                                   num_classes, width, scale)
  return cases


def _row(cls, box, score, image_id=3.0):
  return [image_id] + list(box) + [score, cls]


def _iou_f32(a, b):
  with np.errstate(all='ignore'):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    xa, ya, xb, yb = np.maximum(a[0], b[0]), np.maximum(a[1], b[1]), np.minimum(a[2], b[2]), np.minimum(a[3], b[3])
    inter = np.maximum(xb - xa, F32(0)) * np.maximum(yb - ya, F32(0))
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)


def _crossing_box(base):
  """(box just below, box just above) IoU 0.55f with `base`, one float32 ulp apart in x2."""
  base = np.asarray(base, F32)
  lo, hi = F32(base[0] + 1), F32(base[2] + 200)
  for _ in range(200):                 # bisect x2 of a box sharing base's y extent
    mid = F32((lo + hi) / 2)
    if _iou_f32(base, [base[0], base[1], mid, base[3]]) >= F32(0.55):
      lo = mid
    else:
      hi = mid
  x2 = lo
  while _iou_f32(base, [base[0], base[1], x2, base[3]]) >= F32(0.55):
    x2 = np.nextafter(x2, F32(np.inf))
  below = [base[0], base[1], x2, base[3]]
  above = [base[0], base[1], np.nextafter(x2, F32(-np.inf)), base[3]]
  assert _iou_f32(base, below) < F32(0.55) <= _iou_f32(base, above)
  return below, above


def hand_cases(rng):
  cases = {}
  dummy = _row(0, (0, 0, 0, 0), -1e5)
  # score ties across classes and within a class (separate boxes): class order, then creation order
  rows = [_row(2, (0, 0, 10, 10), 0.5), _row(1, (50, 50, 60, 60), 0.5), _row(1, (0, 0, 10, 10), 0.5),
          _row(3, (100, 0, 110, 10), 0.25), _row(2, (100, 100, 120, 120), 0.5), dummy, dummy]
  cases['ties'] = ([np.array(rows, F32)], 0, 4, 256, F32(1))
  # a row equidistant to two clusters joins the first
  rows = [_row(1, (0, 0, 10, 10), 0.9), _row(1, (4, 0, 14, 10), 0.8), _row(1, (2, 0, 12, 10), 0.7)]
  cases['equidistant'] = ([np.array(rows, F32)], 0, 2, 256, F32(1))
  # IoU one ulp below / above 0.55f
  base = (10.0, 20.0, 50.0, 70.0)
  below, above = _crossing_box(base)
  cases['iou_below'] = ([np.array([_row(1, base, 0.9), _row(1, below, 0.8)], F32)], 0, 2, 256, F32(1))
  cases['iou_above'] = ([np.array([_row(1, base, 0.9), _row(1, above, 0.8)], F32)], 0, 2, 256, F32(1))
  # a cluster of 12 members, and a second one in another class
  big = [_row(1, np.array([30, 30, 80, 90]) + rng.normal(0, 1.0, 4), rng.uniform(0.3, 0.9)) for _ in range(12)]
  big += [_row(2, np.array([30, 30, 80, 90]) + rng.normal(0, 1.0, 4), rng.uniform(0.3, 0.9)) for _ in range(9)]
  cases['big_cluster_m1'] = ([np.array(big, F32)], 0, 3, 256, F32(1))
  cases['big_cluster_m3'] = ([np.array(big[:7], F32), np.array(big[7:14], F32), np.array(big[14:], F32)],
                             0, 3, 256, F32(1))
  # empty classes (rows only in 1 and 7 of 10), and a class-num_classes row that is dropped
  rows = [_row(7, (5, 5, 25, 25), 0.6), _row(1, (5, 5, 25, 25), 0.7), _row(10, (5, 5, 25, 25), 0.99),
          _row(7, (6, 5, 25, 26), 0.4), _row(1, (90, 90, 95, 99), 0.2)]
  cases['empty_and_dropped'] = ([np.array(rows, F32)], 0, 10, 256, F32(1))
  # all-dummy images: one class-0 cluster at -1e5 (zero-area averages give NaN IoUs)
  cases['all_dummy_m1'] = ([np.array([dummy] * 20, F32)], 0, 5, 256, F32(1))
  cases['all_dummy_m2'] = ([np.array([dummy] * 10, F32), np.array([dummy] * 10, F32)], 0b10, 5, 640,
                           F32(2.5))
  # no dummies: every row real, mirrored second model
  k = 30
  xy = rng.uniform(0, 150, (k, 2))
  wh = rng.uniform(5, 60, (k, 2))
  rows = np.concatenate([np.full((k, 1), 4.0), xy, xy + wh, rng.uniform(0.05, 1, (k, 1)),
                         rng.integers(1, 4, (k, 1))], 1).astype(F32)
  mir = rows.copy()
  mir[:, 1], mir[:, 3] = F32(256 * 1.25) - rows[:, 3] - 1, F32(256 * 1.25) - rows[:, 1] + 1
  cases['no_dummy_m2'] = ([rows, mir.astype(F32)], 0b10, 4, 256, F32(1.25))
  # only rows of class num_classes: nothing to fuse
  cases['nothing_fused'] = ([np.array([_row(3, (1, 1, 5, 5), 0.5)] * 3, F32)], 0, 3, 256, F32(1))
  return cases


def main():
  assert int(np.__version__.split('.')[0]) >= 2, 'NEP 50 promotion rules (numpy >= 2) are assumed'
  wbf, nms_np = import_reference()
  rng = np.random.default_rng(2026)
  cases = nms_pair_cases(nms_np, rng)
  cases.update(hand_cases(rng))
  data = {}
  for name, (blocks, mask, num_classes, width, scale) in cases.items():
    rows = max(len(b) for b in blocks)
    assert all(len(b) == rows for b in blocks), name
    data[name + '/det'] = np.stack(blocks).astype(F32)
    data[name + '/meta'] = np.array([len(blocks), mask, num_classes, width], np.int64)
    data[name + '/scale'] = np.array(scale, F32)
    data[name + '/out'] = run_reference(wbf, blocks, mask, num_classes, width, scale)
    print('%-20s models %d rows %3d -> %3d clusters' % (name, len(blocks), rows, len(data[name + '/out'])))
  np.savez_compressed(os.path.join(HERE, 'wbf.npz'), **data)


if __name__ == '__main__':
  main()
