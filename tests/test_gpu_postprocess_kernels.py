"""The post-processing kernels every Engine.detect() and ServingDriver call runs -- pre-NMS
(edet_pre_nms: class arg-max + sigmoid + box decode, or boxes only), top-k pre-NMS
(edet_pre_nms_topk), NonMaxSuppressionV5 (edet_nms_v5: the shared-memory fast kernel and the
full-queue kernel it hands images to), nms_np's per-class NMS (edet_per_class_nms) and the serving
pre-process (edet_preprocess) -- against the CPU oracle at every registered model's anchor layout,
at class-head configurations other than D0's and on every fallback path of NMS-V5.

Shared rules, with the harness of test_gpu_persistent_kernels.py / test_gpu_memory_bound_kernels.py:
  - every input is carved from an allocation that continues with values a stray read would expose
    (NaN after boxes, anchors and images, +inf after fp16 logits and scores -- a NaN score is never
    a candidate, +inf always is -- an out-of-range value after int32 and uint8 inputs); class-head
    padding columns hold fp16 +inf and box-head padding columns NaN;
  - every output is carved from a sentinel-filled allocation: no sentinel after it may change;
  - every case runs twice and both runs must give the same bits;
  - decoded boxes are held to a bound in float32 units derived from decode_box's operations
    (check_decode), scores to rtol 1e-6, indices, classes and NMS outputs to equality.

The registry (anchor_layouts) and the tests that the case lists cover it need no GPU; every other
test is marked gpu on its own."""
import ctypes
import functools

import numpy as np
import pytest
import torch

from automl_b200 import anchors as anchors_lib
from automl_b200 import hparams_config
from automl_b200 import utils
from automl_b200._lib import EdetError
from oracle import postprocess_oracle as po
from test_gpu_kernels import _nms_inputs, _params, _synthetic_head_outputs
from test_gpu_memory_bound_kernels import Buf
from test_gpu_persistent_kernels import DEV, GUARD, SENTINEL, carve  # noqa: F401  (the shared harness)

U = 2.0**-24                  # fp32 unit roundoff
INT_GUARD = -0x5A5A5A5A       # after / in every int32 buffer: no class, index or count is this
NAN, INF = float('nan'), float('inf')
DET_MODELS = (sorted(hparams_config.efficientdet_model_param_dict) +
              sorted(hparams_config.efficientdet_lite_param_dict))


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _round8(x):
  return (x + 7) // 8 * 8


class Head(object):
  """An anchor + class-head configuration: levels min_level..max_level of image_size,
  A = num_scales x len(aspect_ratios) anchors per location, C classes."""

  def __init__(self, image_size, num_classes=90, num_scales=3, aspect_ratios=(1.0, 2.0, 0.5),
               anchor_scale=4.0, min_level=3, max_level=7):
    self.image_size, self.C = image_size, num_classes
    self.num_scales, self.aspect_ratios, self.anchor_scale = num_scales, tuple(aspect_ratios), anchor_scale
    self.min_level, self.max_level = min_level, max_level
    self.hw = tuple(utils.parse_image_size(image_size))
    fs = utils.get_feat_sizes(image_size, max_level)
    self.level_hw = tuple((fs[l]['height'], fs[l]['width']) for l in range(min_level, max_level + 1))
    self.A = num_scales * len(aspect_ratios)
    self.total_anchors = sum(h * w for h, w in self.level_hw) * self.A
    self.layout = (self.hw, self.level_hw, self.total_anchors)

  def params(self, **nms):
    p = _params(self.image_size, **nms)
    p.update(min_level=self.min_level, max_level=self.max_level, num_scales=self.num_scales,
             aspect_ratios=list(self.aspect_ratios), anchor_scale=self.anchor_scale,
             num_classes=self.C)
    return p

  def anchors(self):
    return anchors_lib.Anchors(self.min_level, self.max_level, self.num_scales,
                               list(self.aspect_ratios), self.anchor_scale, self.image_size).boxes

  def name(self):
    return '%s_A%d_C%d' % ('x'.join(map(str, self.hw)) + ('_l%d' % self.max_level if self.max_level != 7 else ''),
                           self.A, self.C)


@functools.lru_cache(maxsize=None)
def model_head(name):
  c = hparams_config.get_efficientdet_config(name)
  return Head(c.image_size, c.num_classes, c.num_scales, c.aspect_ratios, c.anchor_scale,
              c.min_level, c.max_level)


# ---------------------------------------------------------------------------------------------
# registry (no GPU)
def anchor_layouts():
  """(image (h, w), level sizes, total anchors) of every registered EfficientDet / lite model."""
  return sorted({model_head(name).layout for name in DET_MODELS})


def input_sizes():
  """(h, w) of every registered model's network input."""
  return sorted({model_head(name).hw for name in DET_MODELS})


def _layout_heads():
  """One registered head per anchor layout (the first model that has it)."""
  heads = {}
  for name in DET_MODELS:
    heads.setdefault(model_head(name).layout, model_head(name))
  return [heads[l] for l in anchor_layouts()]


LAYOUT_HEADS = _layout_heads()
# class-head configurations other than D0's on a non-square map: C = 1, 20, 96 (the fused arg-max's
# last width), 97, 200 (ld_cls > 1536: pre-NMS needs more than 48 KB of shared memory); A = 1, 3 and
# 16 (kPrePix * A = 256 threads, every thread of a pre-NMS CTA busy)
A_CFG = {1: (1, (1.0,)), 3: (1, (1.0, 2.0, 0.5)), 9: (3, (1.0, 2.0, 0.5)), 16: (4, (1.0, 2.0, 0.5, 1.5))}
SMALL_HEADS = [Head((96, 160), c, *A_CFG[a]) for a, c in
               [(9, 1), (9, 20), (9, 96), (9, 97), (9, 200), (1, 200), (3, 97), (16, 20), (16, 96), (16, 97)]]


def _batch(head):
  return 1 if head.total_anchors > 100000 else 2


# (head, n, ld_cls, ld_box): every layout at D0's head (alternately the tight and a wider stride),
# every small head at both
PRE_CASES = ([(h, _batch(h), _round8(h.A * h.C) + 24 * (i % 2), _round8(4 * h.A) + 8 * (i % 2))
              for i, h in enumerate(LAYOUT_HEADS)] +
             [(h, 2, _round8(h.A * h.C) + 24 * w, _round8(4 * h.A) + 8 * w) for h in SMALL_HEADS for w in (0, 1)])
TOPK_KS = (1, 1000, 8192)
TINY = 16                     # a 2x2 map and four 1x1 levels: 72 anchors
# (head, n, ld_cls, ld_box, ks)
TOPK_CASES = ([(h, _batch(h), _round8(h.A * h.C) + 24 * (i % 2), _round8(4 * h.A), TOPK_KS)
               for i, h in enumerate(LAYOUT_HEADS)] +
              [(h, 2, _round8(h.A * h.C) + 8 * (i % 2), _round8(4 * h.A),
                tuple(sorted({1, min(1000, h.total_anchors * h.C), min(8192, h.total_anchors * h.C)})))
               for i, h in enumerate(SMALL_HEADS)] +
              # k = every pair: C = 1 (A * C = 9: the second 16-byte vector of a pixel row holds
              # one logit and seven padding columns) and C = 97
              [(Head(TINY, 1), 2, 16, 40, (72,)), (Head(TINY, 97), 2, _round8(9 * 97), 40, (72 * 97,))])
NMS_MAX_OUT = (1, 100, 300, 512)
NMS_CASES = [(h.layout, method, NMS_MAX_OUT[(i + 2 * m) % 4])
             for i, h in enumerate(LAYOUT_HEADS) for m, method in enumerate(('gaussian', 'hard'))]
PREP_SIZES = input_sizes() + [(384, 640), (127, 129)]
PREP_SOURCES = [(480, 640), (640, 480), (1, 1), (7, 1000)]


def _head_id(case):
  h, n, ld_cls, ld_box = case[:4]
  return '%s_n%d_ld%d_%d' % (h.name(), n, ld_cls, ld_box)


def test_anchor_layouts_are_covered():
  layouts = anchor_layouts()
  assert len(layouts) == 11
  assert min(l[2] for l in layouts) == 19206 and max(l[2] for l in layouts) == 442260   # lite0, D7x
  assert {len(l[1]) for l in layouts} == {5, 6}
  for cases in (PRE_CASES, TOPK_CASES):
    assert {c[0].layout for c in cases if c[0].C == 90 and c[0].A == 9} >= set(layouts)
    assert {c[0].C for c in cases} >= {1, 20, 96, 97, 200} and {c[0].A for c in cases} >= {1, 3, 16}
    assert any(c[2] > _round8(c[0].A * c[0].C) for c in cases)            # a wider stride
  assert {l for l, _, _ in NMS_CASES} == set(layouts)
  for method in ('gaussian', 'hard'):
    assert {m for _, meth, m in NMS_CASES if meth == method} == set(NMS_MAX_OUT)
  # the shared-memory-heavy pre-NMS launch (ld_cls > 1536) and the thread-filling A = 16
  assert any(16 * c[2] * 2 > 48 * 1024 for c in PRE_CASES)
  assert any(c[0].A * 16 == 256 for c in PRE_CASES)
  assert len(input_sizes()) == 10 and {320, 1536} <= {h for h, _ in input_sizes()}
  assert set(input_sizes()) <= set(PREP_SIZES)


def topk_order(flat, k):
  """Row-wise first k flat indices of po.topk_class_boxes's order (value descending, lower flat
  index first among equal values; -0 == +0), without sorting every pair."""
  out = []
  for row in flat:
    kth = -np.partition(-row, k - 1)[k - 1]
    cand = np.nonzero(row >= kth)[0]
    out.append(cand[np.argsort(-row[cand], kind='stable')][:k])
  return np.stack(out)


def test_topk_order_is_the_oracle():
  rng = np.random.default_rng(2)
  flat = rng.normal(0, 1, size=(3, 5000)).astype(np.float16).astype(np.float32)
  flat[0, rng.choice(5000, 800, replace=False)] = 0.0
  flat[0, rng.choice(5000, 800, replace=False)] = -0.0
  flat[1, :] = np.round(flat[1] * 4) / 4                  # heavy ties
  params = {'num_classes': 10, 'nms_configs': {'max_nms_inputs': 0}}
  for k in (1, 700, 2500, 5000):
    params['nms_configs']['max_nms_inputs'] = k
    _, _, cls, idx = po.topk_class_boxes(params, flat.reshape(3, 500, 10), np.zeros((3, 500, 4), np.float32))
    np.testing.assert_array_equal(topk_order(flat, k), idx.astype(np.int64) * 10 + cls)


# ---------------------------------------------------------------------------------------------
# shared pieces
def check_decode(got, codes, anchors, what=''):
  """Decoded boxes against float64.  decode_box (common.cuh) from fp16 codes (exact in fp32) and
  fp32 anchors, with every rounding of a correctly rounded fp32 operation <= u = 2^-24 relative and
  expf within 2 ulp (CUDA C Programming Guide) = 4u relative:
    yca = (a0 + a2) * 0.5                  one rounding (the halving is exact):   u |yca|
    ha  = a2 - a0                          u |ha|
    h/2 = expf(th) * ha * 0.5              4u + u + u:                            6u |h/2|
    yc  = ty * ha + yca                    ha, the product, the sum:   2u |ty ha| + u |yca| + u |yc|
    out = yc -/+ h/2                       the above + u |out|
  so |out - exact| <= u (2 |ty ha| + |yca| + |yc| + 6 |h/2| + |out|) to first order (x likewise);
  the factor 1.001 covers the second-order terms and the float64 reference's own rounding."""
  t = np.asarray(codes, np.float64)
  a = np.asarray(anchors, np.float64)
  yca, xca = (a[..., 0] + a[..., 2]) / 2, (a[..., 1] + a[..., 3]) / 2
  ha, wa = a[..., 2] - a[..., 0], a[..., 3] - a[..., 1]
  hh, hw = np.exp(t[..., 2]) * ha / 2, np.exp(t[..., 3]) * wa / 2
  yc, xc = t[..., 0] * ha + yca, t[..., 1] * wa + xca
  ref = np.stack([yc - hh, xc - hw, yc + hh, xc + hw], -1)
  my = 2 * np.abs(t[..., 0] * ha) + np.abs(yca) + np.abs(yc) + 6 * np.abs(hh)
  mx = 2 * np.abs(t[..., 1] * wa) + np.abs(xca) + np.abs(xc) + 6 * np.abs(hw)
  bound = 1.001 * U * (np.stack([my, mx, my, mx], -1) + np.abs(ref))
  err = np.abs(np.asarray(got, np.float64) - ref)
  bad = ~(err <= bound)
  assert not bad.any(), '%s: box off by %g (%d outside the bound), first at %s: got %r, want %r +- %g' % (
      what, float(np.nanmax(err)), int(bad.sum()), tuple(np.argwhere(bad)[0]),
      float(np.asarray(got)[tuple(np.argwhere(bad)[0])]), float(ref[tuple(np.argwhere(bad)[0])]),
      float(bound[tuple(np.argwhere(bad)[0])]))


def head_inputs(head, n, seed, dup=True):
  """fp16 logits N(-4, 2) and box codes N(0, 0.5): per level [N,H,W,A*C] and [N,H,W,A*4].  dup:
  every 5th anchor gets its maximum twice, at two random classes (the first must win)."""
  rng = np.random.default_rng(seed)
  cls, box = _synthetic_head_outputs(rng, n, head.image_size, head.min_level, head.max_level,
                                     head.A, head.C)
  if dup and head.C > 1:
    for t in cls:
      v = t.reshape(-1, head.C)
      rows = np.arange(0, v.shape[0], 5)
      c1 = rng.integers(0, head.C - 1, rows.size)
      c2 = rng.integers(c1 + 1, head.C)
      top = (v[rows].astype(np.float32).max(1) + 1).astype(np.float16)
      v[rows, c1] = top
      v[rows, c2] = top
  return cls, box


def dev_levels(levels, ld, fill):
  """Device copies of [N,H,W,c] fp16 arrays with ld >= c columns; padding columns and GUARD
  elements after each allocation hold `fill`."""
  out = []
  for t in levels:
    full = torch.full(t.shape[:-1] + (ld,), fill, dtype=torch.float16)
    full[..., :t.shape[-1]] = torch.from_numpy(t)
    out.append(Buf(full, fill))
  return out


def _out(shape, dtype=torch.float32):
  fill = SENTINEL if dtype == torch.float32 else INT_GUARD
  return Buf(torch.full(shape, fill, dtype=dtype), fill)


def _same(runs):
  for r in runs[1:]:
    for a, b in zip(runs[0], r):
      assert torch.equal(a, b), 'two runs differ'


# ---------------------------------------------------------------------------------------------
# edet_pre_nms
@pytest.mark.gpu
@pytest.mark.parametrize('case', PRE_CASES, ids=_head_id)
def test_pre_nms(case):
  """Classes exact (first maximum wins), scores within rtol 1e-6 of po.pre_nms, boxes within
  check_decode's bound; the boxes-only form gives the same boxes and writes no score or class."""
  ops = _ops()
  head, n, ld_cls, ld_box = case
  A, C, K = head.A, head.C, head.total_anchors
  cls, box = head_inputs(head, n, seed=K + C + ld_cls)
  dcls, dbox = dev_levels(cls, ld_cls, INF), dev_levels(box, ld_box, NAN)
  anc = head.anchors()
  danc = carve(torch.from_numpy(anc))

  def launch(with_logits):
    boxes, scores, classes = _out((n, K, 4)), _out((n, K)), _out((n, K), torch.int32)
    ops.pre_nms([b.t for b in dcls] if with_logits else None, [b.t for b in dbox], head.level_hw,
                A, C, danc, boxes.t, scores.t, classes.t)
    return boxes.result(), scores.result(), classes.result()

  runs = [launch(True), launch(True)]
  _same(runs)
  boxes, scores, classes = runs[0]
  only = launch(False)
  assert torch.equal(only[0], boxes), 'boxes-only pre-NMS decodes different boxes'
  assert bool((only[1] == SENTINEL).all()) and bool((only[2] == INT_GUARD).all())
  _, ref_scores, ref_classes = po.pre_nms(head.params(), cls, box)
  np.testing.assert_array_equal(classes.numpy(), ref_classes)
  np.testing.assert_allclose(scores.numpy(), ref_scores, rtol=1e-6, atol=1e-7)
  codes = np.concatenate([b.reshape(n, -1, 4) for b in box], 1)
  check_decode(boxes.numpy(), codes, anc, _head_id(case))


@pytest.mark.gpu
@pytest.mark.parametrize('what', ['A17', 'ld_cls', 'levels9'])
def test_pre_nms_refusals(what):
  """17 anchors per location (kPrePix * A > 256 threads), ld_cls % 8 != 0 and 9 levels raise and
  leave every output untouched."""
  ops = _ops()
  a, c = {'A17': (17, 1), 'ld_cls': (9, 91), 'levels9': (9, 4)}[what]
  ld_cls = a * c if what == 'ld_cls' else _round8(a * c)
  levels = 9 if what == 'levels9' else 5
  hw = [(2, 2)] * levels
  cls = [carve(torch.zeros(1, 2, 2, ld_cls, dtype=torch.float16)) for _ in hw]
  box = [carve(torch.zeros(1, 2, 2, _round8(4 * a), dtype=torch.float16)) for _ in hw]
  k = 4 * a * levels
  anc = carve(torch.zeros(k, 4))
  boxes, scores, classes = _out((1, k, 4)), _out((1, k)), _out((1, k), torch.int32)
  with pytest.raises(EdetError):
    ops.pre_nms(cls, box, hw, a, c, anc, boxes.t, scores.t, classes.t)
  assert bool((boxes.result() == SENTINEL).all()) and bool((scores.result() == SENTINEL).all())
  assert bool((classes.result() == INT_GUARD).all())


# ---------------------------------------------------------------------------------------------
# edet_pre_nms_topk
def _topk_launch(head, n, k, dcls, dbox, danc):
  ops = _ops()
  bufs = (_out((n, k, 4)), _out((n, k)), _out((n, k), torch.int32), _out((n, k), torch.int32))
  ops.pre_nms_topk([b.t for b in dcls], [b.t for b in dbox], head.level_hw, head.A, head.C, danc,
                   *[b.t for b in bufs])
  return tuple(b.result() for b in bufs)


@pytest.mark.gpu
@pytest.mark.parametrize('case', TOPK_CASES, ids=_head_id)
def test_pre_nms_topk(case):
  """The first k (anchor, class) pairs in po.topk_class_boxes's order (topk_order): indices and
  classes exact, scores within rtol 1e-6, boxes within check_decode's bound.  Padding columns
  hold +inf: a kernel that ranked one would select it first."""
  head, n, ld_cls, ld_box, ks = case
  C = head.C
  cls, box = head_inputs(head, n, seed=head.total_anchors + 3 * C + ld_cls)
  dcls, dbox = dev_levels(cls, ld_cls, INF), dev_levels(box, ld_box, NAN)
  anc = head.anchors()
  danc = carve(torch.from_numpy(anc))
  flat = np.concatenate([c.reshape(n, -1) for c in cls], 1).astype(np.float32)
  codes = np.concatenate([b.reshape(n, -1, 4) for b in box], 1)
  for k in ks:
    runs = [_topk_launch(head, n, k, dcls, dbox, danc) for _ in range(2)]
    _same(runs)
    boxes, scores, classes, indices = (r.numpy() for r in runs[0])
    order = topk_order(flat, k)
    what = '%s k=%d' % (_head_id(case), k)
    np.testing.assert_array_equal(indices, order // C, err_msg=what)
    np.testing.assert_array_equal(classes, order % C, err_msg=what)
    np.testing.assert_allclose(scores, po.sigmoid_f32(np.take_along_axis(flat, order, 1)),
                               rtol=1e-6, atol=1e-7, err_msg=what)
    check_decode(boxes, np.take_along_axis(codes, (order // C)[..., None], 1), anc[order // C], what)
  if TINY in head.hw:     # k = every pair: the oracle itself
    _, ref_scores, ref_classes = po.pre_nms(head.params(max_nms_inputs=ks[-1]), cls, box)
    np.testing.assert_array_equal(classes, ref_classes)
    np.testing.assert_allclose(scores, ref_scores, rtol=1e-6, atol=1e-7)


def _signed_zero_logits(rng, head, n, positives, zeros):
  """Per image: `positives` logits in [0.5, 8], `zeros` zeros of random sign, the rest negative,
  scattered over the (anchor, class) pairs; split into the head's levels."""
  pairs = head.total_anchors * head.C
  flat = np.empty((n, pairs), np.float16)
  for i in range(n):
    perm = rng.permutation(pairs)
    flat[i, perm[:positives]] = rng.uniform(0.5, 8.0, positives)
    flat[i, perm[positives:positives + zeros]] = np.where(rng.random(zeros) < 0.5, -0.0, 0.0)
    flat[i, perm[positives + zeros:]] = -0.01 - np.abs(rng.normal(0, 4, pairs - positives - zeros))
  cls, at = [], 0
  for h, w in head.level_hw:
    size = h * w * head.A * head.C
    cls.append(flat[:, at:at + size].reshape(n, h, w, head.A * head.C))
    at += size
  return cls


@pytest.mark.gpu
def test_pre_nms_topk_signed_zero():
  """fp16 -0 and +0 are equal logits: tf.math.top_k and the oracle keep the lower flat index
  among them.  The k-th logit is 0, with -0 and +0 both inside and outside the selected set."""
  head = Head(64, 20)
  n, positives, zeros, k = 2, 300, 2000, 1300
  rng = np.random.default_rng(17)
  cls = _signed_zero_logits(rng, head, n, positives, zeros)
  _, box = head_inputs(head, n, seed=18, dup=False)
  params = head.params(max_nms_inputs=k)
  merged_cls, merged_box = po.merge_class_box_level_outputs(
      params, [c.astype(np.float32) for c in cls], [b.astype(np.float32) for b in box])
  _, _, ref_classes, ref_indices = po.topk_class_boxes(params, merged_cls, merged_box)
  flat = merged_cls.reshape(n, -1)
  order = ref_indices.astype(np.int64) * head.C + ref_classes
  for i in range(n):   # the construction: a cut through zeros of both signs
    assert flat[i, order[i, -1]] == 0 and flat[i, order[i, positives - 1]] > 0
    chosen = np.zeros(flat.shape[1], bool)
    chosen[order[i]] = True
    z = flat[i] == 0
    for side in (chosen, ~chosen):
      assert {bool(s) for s in np.signbit(flat[i][z & side])} == {False, True}
  dcls = dev_levels(cls, _round8(head.A * head.C), INF)
  dbox = dev_levels(box, _round8(4 * head.A), NAN)
  danc = carve(torch.from_numpy(head.anchors()))
  runs = [_topk_launch(head, n, k, dcls, dbox, danc) for _ in range(2)]
  _same(runs)
  _, scores, classes, indices = (r.numpy() for r in runs[0])
  np.testing.assert_array_equal(indices, ref_indices)
  np.testing.assert_array_equal(classes, ref_classes)
  _, ref_scores, _ = po.pre_nms(params, cls, box)
  np.testing.assert_allclose(scores, ref_scores, rtol=1e-6, atol=1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize('k', [0, 8193, 73])
def test_pre_nms_topk_refusals(k):
  """k = 0, k > kMaxK = 8192 and k > the number of pairs (72 on the tiny map with C = 1) raise
  and leave every output untouched."""
  head = Head(TINY if k == 73 else 128, 1 if k == 73 else 90)
  n = 1
  cls, box = head_inputs(head, n, seed=5, dup=False)
  dcls, dbox = dev_levels(cls, _round8(head.A * head.C), INF), dev_levels(box, _round8(4 * head.A), NAN)
  danc = carve(torch.from_numpy(head.anchors()))
  bufs = (_out((n, k, 4)), _out((n, k)), _out((n, k), torch.int32), _out((n, k), torch.int32))
  with pytest.raises(EdetError):
    _ops().pre_nms_topk([b.t for b in dcls], [b.t for b in dbox], head.level_hw, head.A, head.C,
                        danc, *[b.t for b in bufs])
  for b in bufs:
    r = b.result()
    assert bool((r == b.fill).all())


# ---------------------------------------------------------------------------------------------
# edet_nms_v5
def run_nms(boxes, scores, classes, scales, id_base, max_out, iou_t, score_t, sigma, clip):
  """Two launches into fresh guarded outputs and workspace; the same bits.  Returns (det, sel,
  valid, flags) as numpy, flags = the fast kernel's hand-over reasons in the last 4n work bytes."""
  ops = _ops()
  n, k = scores.shape
  db, ds = carve(torch.from_numpy(boxes)), Buf(torch.from_numpy(scores), INF)
  dc = Buf(torch.from_numpy(classes), INT_GUARD)
  dsc = carve(torch.from_numpy(scales)) if scales is not None else None
  runs = []
  for _ in range(2):
    det, sel, valid = _out((n, max_out, 7)), _out((n, max_out), torch.int32), _out((n,), torch.int32)
    work = Buf(torch.full((ops.nms_work_bytes(n, k),), 0x5A, dtype=torch.uint8), 0x5A)
    ops.nms_v5(db, ds.t, dc.t, dsc, id_base, max_out, iou_t, score_t, sigma, clip, det.t, sel.t,
               valid.t, work.t)
    w = work.result()
    runs.append((det.result(), sel.result(), valid.result(), w[-4 * n:].clone().view(torch.int32)))
  _same(runs)
  return tuple(r.numpy() for r in runs[0])


def check_nms(res, boxes, scores, classes, scales, id_base, max_out, iou_t, score_t, sigma, clip):
  """Every image bit-exact against po.non_max_suppression_v5: valid count, the padded keep
  indices, scores, clipped and scaled boxes, 1-based classes and image ids."""
  det, sel, valid, _ = res
  for i in range(scores.shape[0]):
    idx, sc, v = po.non_max_suppression_v5(boxes[i], scores[i], max_out, iou_t, score_t, sigma, True)
    assert int(valid[i]) == v, (i, int(valid[i]), v)
    np.testing.assert_array_equal(sel[i], idx, err_msg='image %d' % i)
    np.testing.assert_array_equal(det[i, :, 5], sc, err_msg='image %d' % i)
    s = np.float32(1.0 if scales is None else scales[i])
    ref = po.clip_boxes(boxes[i][idx], (int(clip[0]), int(clip[1]))) * s
    np.testing.assert_array_equal(det[i, :, 1:5], ref, err_msg='image %d' % i)
    np.testing.assert_array_equal(det[i, :, 6], (classes[i][idx] + 1).astype(np.float32))
    np.testing.assert_array_equal(det[i, :, 0], np.full(max_out, id_base + i, np.float32))


def _nms_args(method, score_thresh=None):
  params = _params(512, method=method, score_thresh=score_thresh)
  return po.nms_v5_params(params['nms_configs'])


@pytest.mark.gpu
@pytest.mark.parametrize('case', NMS_CASES, ids=lambda c: '%dx%d_K%d_%s_max%d' % (
    c[0][0] + (c[0][2], c[1], c[2])))
def test_nms_v5_layouts(case):
  """K = every registered layout's anchor count (up to 442 260), gaussian and hard, every
  max_output_size from 1 to 512, a non-square clip, image ids from 7, per-image scales: bit-exact
  whichever kernel settles each image."""
  layout, method, max_out = case
  (h, w), _, k = layout
  n = 2
  rng = np.random.default_rng(k + max_out + len(method))
  boxes, scores, classes = _nms_inputs(rng, n, k, image=float(max(h, w)))
  iou_t, score_t, sigma = _nms_args(method, 0.0 if method == 'gaussian' else None)
  scales = np.asarray([1.25, 0.5], np.float32)
  clip = (float(h), float(3 * w // 4))
  res = run_nms(boxes, scores, classes, scales, 7, max_out, iou_t, score_t, sigma, clip)
  assert set(res[3].tolist()) <= {0, 1, 2, 3, 4}, res[3]
  check_nms(res, boxes, scores, classes, scales, 7, max_out, iou_t, score_t, sigma, clip)


def _grid_boxes(k):
  """k disjoint 4 x 4 boxes on a 6-pixel grid."""
  side = int(np.ceil(np.sqrt(k)))
  r, c = np.divmod(np.arange(k), side)
  y, x = 6.0 * r, 6.0 * c
  return np.stack([y, x, y + 4, x + 4], -1).astype(np.float32)


def _shifted(rng, base, lo, hi, count):
  """count boxes of base's size moved by lo..hi pixels along x or y, either way."""
  d = rng.uniform(lo, hi, count) * rng.choice([-1.0, 1.0], count)
  along_x = rng.random(count) < 0.5
  out = np.repeat(base[None], count, 0).astype(np.float64)
  out[along_x, 1] += d[along_x]
  out[along_x, 3] += d[along_x]
  out[~along_x, 0] += d[~along_x]
  out[~along_x, 2] += d[~along_x]
  return out.astype(np.float32)


def _distinct(rng, lo, hi, count):
  """count distinct float32 values in (lo, hi), shuffled."""
  v = (lo + (hi - lo) * (np.arange(count) + 1.0) / (count + 1)).astype(np.float32)
  assert np.unique(v).size == count
  return rng.permutation(v)


BEST = np.asarray([100.0, 100.0, 200.0, 200.0], np.float32)


def fallback_image(reason, rng):
  """(method, score_thresh, boxes [k,4], scores [k]) of one image the fast kernel must hand to the
  full-queue kernel with flag `reason`:
    1 (ties overflow the 8192-candidate capacity): 9000 boxes, every score 0.25;
    2 (the queue runs out while excluded candidates remain): hard, 20 000 copies of one box with
      distinct scores: the top one is selected, the 8191 others of the queue are suppressed, none
      is re-queued, and the excluded ~12 000 remain;
    3 (the exactness bound fails): gaussian, score_thresh 0.5.  The best box (0.70), 50 boxes at
      IoU 0.3 with it (0.695-0.70), 8141 near-copies (IoU > 0.9, 0.65-0.695) and 11 808 scattered
      boxes (0.60-0.65).  The near-copies decay to < 0.15 and drop out; the 50 re-queue at about
      0.58, below every excluded candidate, and the first of them the queue reaches fails the bound;
    4 (the re-queue array overflows): gaussian, 8000 boxes at IoU 0.6 with the best one, scores
      0.90-0.91: all 7999 decay to about 0.44 and re-queue in one period, 64 per chunk, past 4096."""
  if reason == 1:
    boxes, _, _ = _nms_inputs(rng, 1, 9000, clustered=False)
    return 'gaussian', None, boxes[0], np.full(9000, 0.25, np.float32)
  if reason == 2:
    return 'hard', None, np.repeat(BEST[None], 20000, 0), _distinct(rng, 0.2, 0.9, 20000)
  if reason == 3:
    scattered, _, _ = _nms_inputs(rng, 1, 11808, image=1000.0, clustered=False)
    boxes = np.concatenate([BEST[None], _shifted(rng, BEST, 53.0, 54.5, 50),
                            _shifted(rng, BEST, 0.0, 2.5, 8141), scattered[0]])
    scores = np.concatenate([[0.70], _distinct(rng, 0.695, 0.6999, 50), _distinct(rng, 0.65, 0.695, 8141),
                             _distinct(rng, 0.60, 0.65, 11808)]).astype(np.float32)
    return 'gaussian', 0.5, boxes, scores
  boxes = np.concatenate([BEST[None], _shifted(rng, BEST, 24.5, 25.5, 7999)])
  return 'gaussian', None, boxes, np.concatenate([[0.91], _distinct(rng, 0.90, 0.9099, 7999)]).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize('reason', [1, 2, 3, 4])
def test_nms_v5_fallback_reasons(reason):
  """Each hand-over reason of the fast kernel, flagged with its own value, and the full-queue
  kernel's result bit-exact."""
  rng = np.random.default_rng(40 + reason)
  method, thr, boxes, scores = fallback_image(reason, rng)
  iou_t, score_t, sigma = _nms_args(method, thr)
  k = scores.size
  classes = rng.integers(0, 90, size=(1, k)).astype(np.int32)
  scales = np.asarray([0.75], np.float32)
  res = run_nms(boxes[None], scores[None], classes, scales, 3, 100, iou_t, score_t, sigma, (1024.0, 768.0))
  assert res[3].tolist() == [reason]
  check_nms(res, boxes[None], scores[None], classes, scales, 3, 100, iou_t, score_t, sigma, (1024.0, 768.0))


@pytest.mark.gpu
@pytest.mark.parametrize('method,reasons', [('hard', (0, 2)), ('gaussian', (3, 0))])
def test_nms_v5_mixed_batch(method, reasons):
  """One image settled by the fast kernel (disjoint boxes, distinct scores) and one handed to the
  full-queue kernel in the same launch: both exact."""
  rng = np.random.default_rng(50 + len(method))
  boxes, scores = [], []
  thr = None
  for r in reasons:
    if r:
      m, thr, b, s = fallback_image(r, rng)
      assert m == method
    else:
      b, s = _grid_boxes(20000), _distinct(rng, 0.0, 1.0, 20000)
    boxes.append(b)
    scores.append(s)
  boxes, scores = np.stack(boxes), np.stack(scores)
  iou_t, score_t, sigma = _nms_args(method, thr)
  classes = rng.integers(0, 90, size=scores.shape).astype(np.int32)
  scales = np.asarray([1.5, 0.5], np.float32)
  res = run_nms(boxes, scores, classes, scales, 11, 100, iou_t, score_t, sigma, (1024.0, 768.0))
  assert tuple(res[3].tolist()) == reasons
  check_nms(res, boxes, scores, classes, scales, 11, 100, iou_t, score_t, sigma, (1024.0, 768.0))


@pytest.mark.gpu
def test_nms_v5_signed_zero_scores():
  """-0 and +0 are equal scores: TF's heap and the full-queue kernel pop them in index order, so
  the fast kernel must too.  hard NMS of disjoint boxes keeps every candidate (score > -inf), in
  score order.  The sign of a selected zero score is not compared."""
  rng = np.random.default_rng(60)
  n, k = 2, 64
  boxes = np.repeat(_grid_boxes(k)[None], n, 0)
  scores = rng.choice(np.asarray([-0.0, 0.0, -0.25, -1.0, -3.5], np.float32), size=(n, k))
  for i in range(n):
    z = scores[i] == 0
    assert {bool(s) for s in np.signbit(scores[i][z])} == {False, True}
  classes = rng.integers(0, 90, size=(n, k)).astype(np.int32)
  iou_t, score_t, sigma = _nms_args('hard')
  res = run_nms(boxes, scores, classes, None, 0, 100, iou_t, score_t, sigma, (512.0, 512.0))
  assert res[3].tolist() == [0, 0]       # the fast kernel settled both images
  check_nms(res, boxes, scores, classes, None, 0, 100, iou_t, score_t, sigma, (512.0, 512.0))


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['gaussian', 'hard'])
def test_nms_v5_nan_and_neg_inf_never_selected(method):
  rng = np.random.default_rng(70)
  n, k = 2, 3000
  boxes, scores, classes = _nms_inputs(rng, n, k)
  scores[:, ::7] = np.nan
  scores[:, 3::11] = -np.inf
  iou_t, score_t, sigma = _nms_args(method, 0.0 if method == 'gaussian' else None)
  res = run_nms(boxes, scores, classes, None, 0, 300, iou_t, score_t, sigma, (512.0, 512.0))
  check_nms(res, boxes, scores, classes, None, 0, 300, iou_t, score_t, sigma, (512.0, 512.0))
  det, sel, valid, _ = res
  for i in range(n):
    assert np.isfinite(scores[i][sel[i, :valid[i]]]).all()


@pytest.mark.gpu
@pytest.mark.parametrize('max_out', [0, 513])
def test_nms_v5_refusals(max_out):
  ops = _ops()
  rng = np.random.default_rng(0)
  boxes, scores, classes = _nms_inputs(rng, 1, 50)
  m = max(max_out, 1)
  det, sel, valid = _out((1, m, 7)), _out((1, m), torch.int32), _out((1,), torch.int32)
  work = torch.empty(ops.nms_work_bytes(1, 50), dtype=torch.uint8, device=DEV)
  with pytest.raises(EdetError):
    ops.nms_v5(carve(torch.from_numpy(boxes)), carve(torch.from_numpy(scores)),
               Buf(torch.from_numpy(classes), INT_GUARD).t, None, 0, max_out, 0.5, 0.001, 0.25,
               (512.0, 512.0), det.t, sel.t, valid.t, work)
  assert bool((det.result() == SENTINEL).all()) and bool((sel.result() == INT_GUARD).all())
  assert bool((valid.result() == INT_GUARD).all())


# ---------------------------------------------------------------------------------------------
# edet_per_class_nms
PCN_METHODS = ('hard', 'diou', 'gaussian', 'linear')
PCN_CASES = [(m, mb) for m in PCN_METHODS for mb in (1, 37, 256)]


def _pcn_inputs(rng, k, num_classes):
  """3 images of k candidates with distinct scores: (0) boxes around 40 centres, class ids in
  -3..num_classes+2 (the out-of-range ones must be ignored); (1) boxes around 5 centres in 3
  classes, so that hard NMS keeps few per 2048-candidate round and needs several rounds; (2) no
  valid class id at all."""
  boxes, scores, classes = [], [], []
  for i in range(3):
    b, _, _ = _nms_inputs(rng, 1, k, image=512.0)
    if i == 1:
      centres = rng.uniform(100, 400, size=(5, 2))
      c = centres[rng.integers(0, 5, k)] + rng.normal(0, 4, size=(k, 2))
      wh = rng.uniform(40, 60, size=(k, 2))
      b = np.concatenate([c - wh / 2, c + wh / 2], -1).astype(np.float32)[None]
    boxes.append(b[0])
    scores.append(_distinct(rng, 0.0, 1.0, k))
    if i == 0:
      classes.append(rng.integers(-3, num_classes + 3, k))
    elif i == 1:
      classes.append(rng.integers(0, 3, k))
    else:
      classes.append(np.where(rng.random(k) < 0.5, -1, num_classes))
  return np.stack(boxes), np.stack(scores), np.stack(classes).astype(np.int32)


def _pcn_launch(boxes, scores, classes, ids, scl, num_classes, max_boxes, method):
  ops = _ops()
  n, k = scores.shape
  db, ds, dc = carve(torch.from_numpy(boxes)), Buf(torch.from_numpy(scores), INF), Buf(torch.from_numpy(classes), INT_GUARD)
  runs = []
  for _ in range(2):
    det, keep, valid = _out((n, max_boxes, 7)), _out((n, max_boxes), torch.int32), _out((n,), torch.int32)
    work = _out((n, k))
    ops.per_class_nms(db, ds.t, dc.t, ids, scl, num_classes, max_boxes, method, None, det.t, keep.t,
                      valid.t, work=work.t)
    work.result()
    runs.append((det.result(), keep.result(), valid.result()))
  _same(runs)
  return tuple(r.numpy() for r in runs[0])


def _pcn_check(method, got, ref, what):
  if method == 'gaussian':
    np.testing.assert_array_equal(got[:, [0, 1, 2, 3, 4, 6]], ref[:, [0, 1, 2, 3, 4, 6]], err_msg=what)
    np.testing.assert_allclose(got[:, 5], ref[:, 5], rtol=1e-6, atol=0, err_msg=what)
  else:
    np.testing.assert_array_equal(got, ref, err_msg=what)


@pytest.mark.gpu
@pytest.mark.parametrize('method,max_boxes', PCN_CASES)
def test_per_class_nms(method, max_boxes):
  """Rows against po.per_class_nms (gaussian: every column equal but the score, within rtol 1e-6,
  as for the reference module's goldens); out-of-range class ids ignored; an image without a valid
  class id gives max_boxes dummy rows; keep indices point at the rows' candidates."""
  rng = np.random.default_rng(80 + max_boxes + len(method))
  k, num_classes = 3000, 20
  boxes, scores, classes = _pcn_inputs(rng, k, num_classes)
  ids = np.asarray([5.0, 6.0, 7.0], np.float32)
  scl = np.asarray([1.0, 2.5, 0.5], np.float32)
  det, keep, valid = _pcn_launch(boxes, scores, classes, carve(torch.from_numpy(ids)),
                                 carve(torch.from_numpy(scl)), num_classes, max_boxes, method)
  cfg = {'method': method, 'iou_thresh': None, 'sigma': None, 'score_thresh': None}
  for i in range(3):
    ref = po.per_class_nms(boxes[i], scores[i], classes[i], ids[i:i + 1], scl[i], num_classes,
                           max_boxes, cfg)
    what = '%s max_boxes=%d image %d' % (method, max_boxes, i)
    _pcn_check(method, det[i], ref, what)
    nv = int((ref[:, 5] > -1e4).sum())
    assert int(valid[i]) == nv, what
    assert (keep[i, nv:] == -1).all(), what
    kp = keep[i, :nv]
    assert ((classes[i][kp] >= 0) & (classes[i][kp] < num_classes)).all(), what
    np.testing.assert_array_equal(classes[i][kp] + 1, det[i, :nv, 6], err_msg=what)
    np.testing.assert_array_equal(boxes[i][kp][:, [1, 0, 3, 2]] * scl[i], det[i, :nv, 1:5], err_msg=what)
  assert int(valid[2]) == 0
  assert int(valid[1]) == max_boxes or max_boxes > 37     # image 1 runs out of survivors at 256


@pytest.mark.gpu
@pytest.mark.parametrize('method', PCN_METHODS)
def test_per_class_nms_default_ids_and_scales(method):
  """image_ids / image_scales = None: the id is the batch index and the scale 1."""
  rng = np.random.default_rng(90)
  k, num_classes, max_boxes = 500, 20, 37
  boxes, scores, classes = _pcn_inputs(rng, k, num_classes)
  det, _, _ = _pcn_launch(boxes, scores, classes, None, None, num_classes, max_boxes, method)
  cfg = {'method': method, 'iou_thresh': None, 'sigma': None, 'score_thresh': None}
  for i in range(3):
    ref = po.per_class_nms(boxes[i], scores[i], classes[i], np.asarray([float(i)], np.float32),
                           np.float32(1.0), num_classes, max_boxes, cfg)
    _pcn_check(method, det[i], ref, '%s image %d' % (method, i))


@pytest.mark.gpu
@pytest.mark.parametrize('method', PCN_METHODS)
def test_per_class_nms_tie_order(method):
  """Equal scores: hard / diou take the higher index first (a stable argsort then [::-1]); the soft
  methods the lower index first (the first arg-max).  Boxes 0 and 1 are disjoint at 0.5, boxes 2
  and 3 identical at 0.7, all of class 0."""
  boxes = np.asarray([[[0, 0, 10, 10], [100, 100, 110, 110], [50, 50, 70, 70], [50, 50, 70, 70]]], np.float32)
  scores = np.asarray([[0.5, 0.5, 0.7, 0.7]], np.float32)
  classes = np.zeros((1, 4), np.int32)
  _, keep, valid = _pcn_launch(boxes, scores, classes, None, None, 1, 4, method)
  if method in ('hard', 'diou'):
    assert keep[0].tolist() == [3, 1, 0, -1] and int(valid[0]) == 3
  elif method == 'linear':                     # IoU 1 -> weight 0: box 3 drops out
    assert keep[0].tolist() == [2, 0, 1, -1] and int(valid[0]) == 3
  else:                                        # gaussian: box 3 decays to 0.7 e^-2
    assert keep[0].tolist() == [2, 0, 1, 3] and int(valid[0]) == 4


def _pcn_raw(n, k, max_boxes, method_code, sigma, det, keep, valid, work):
  from automl_b200 import _lib
  z = torch.zeros(n, k, 4, device=DEV)
  s = torch.rand(n, k, device=DEV)
  c = torch.zeros(n, k, dtype=torch.int32, device=DEV)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  _lib.call('edet_per_class_nms', p(z), p(s), p(c), None, None, n, k, 90, max_boxes, method_code,
            ctypes.c_float(0.5), ctypes.c_float(sigma), ctypes.c_float(0.001), p(work), p(det),
            p(keep), p(valid), None)


@pytest.mark.gpu
@pytest.mark.parametrize('what', ['max_boxes257', 'sigma0', 'sigma_neg', 'method99'])
def test_per_class_nms_refusals(what):
  """max_boxes_to_draw = 257, a soft method with sigma <= 0 and an unknown method code raise and
  leave every output untouched."""
  from automl_b200 import _lib
  n, k = 1, 64
  mb = 257 if what == 'max_boxes257' else 100
  code = {'max_boxes257': _lib.NMS_HARD, 'sigma0': _lib.NMS_GAUSSIAN, 'sigma_neg': _lib.NMS_LINEAR,
          'method99': 99}[what]
  sigma = {'sigma0': 0.0, 'sigma_neg': -1.0}.get(what, 0.5)
  det, keep, valid, work = _out((n, mb, 7)), _out((n, mb), torch.int32), _out((n,), torch.int32), _out((n, k))
  with pytest.raises(EdetError):
    _pcn_raw(n, k, mb, code, sigma, det.t, keep.t, valid.t, work.t)
  for b in (det, keep, valid, work):
    assert bool((b.result() == b.fill).all())


# ---------------------------------------------------------------------------------------------
# edet_preprocess
PREP_MEAN, PREP_STD = [100.5, 120.25, 90.75], [50.0, 60.5, 70.125]


def _scaled_hw(src, size):
  """dataloader.py's float32 scaled size of a (h, w) source in an output of `size`."""
  (h, w), (oh, ow) = src, size
  s = min(np.float32(oh) / np.float32(h), np.float32(ow) / np.float32(w))
  return int(np.float32(h) * s), int(np.float32(w) * s)


@pytest.mark.gpu
@pytest.mark.parametrize('src', PREP_SOURCES, ids=lambda s: 'src%dx%d' % s)
@pytest.mark.parametrize('size', PREP_SIZES, ids=lambda s: '%dx%d' % s)
def test_preprocess(size, src):
  """Bit-identical to po.image_preprocess, zero pad included (the kernel does the oracle's float32
  operations in the oracle's order), at every registered input size (2-6 column blocks of 256) for
  down- and up-scaled sources; an image that collapses to zero rows is refused."""
  ops = _ops()
  n = 3
  rng = np.random.default_rng(size[0] * 7 + src[1])
  imgs = rng.integers(0, 256, size=(n,) + src + (3,), dtype=np.uint8)
  raw = Buf(torch.from_numpy(imgs), 0xA5)
  runs = []
  collapses = min(_scaled_hw(src, size)) == 0
  for _ in range(2):
    out = _out((n,) + tuple(size) + (3,))
    if collapses:
      with pytest.raises(EdetError):
        ops.preprocess(raw.t, out.t, PREP_MEAN, PREP_STD)
      assert bool((out.result() == SENTINEL).all())
      return
    scale = ops.preprocess(raw.t, out.t, PREP_MEAN, PREP_STD)
    runs.append((out.result(),))
  _same(runs)
  got = runs[0][0].numpy()
  for i in range(n):
    ref, ref_scale = po.image_preprocess(imgs[i], size, PREP_MEAN, PREP_STD)
    np.testing.assert_array_equal(got[i], ref, err_msg='image %d' % i)
    assert np.float32(scale) == ref_scale


def test_preprocess_cases_collapse_somewhere():
  """The case list reaches the refusal: 7 x 1000 into 127 x 129 has a zero-row scaled image."""
  assert _scaled_hw((7, 1000), (127, 129))[0] == 0
  assert all(min(_scaled_hw(s, z)) > 0 for s in PREP_SOURCES[:3] for z in PREP_SIZES)


# ---------------------------------------------------------------------------------------------
# Engine.detect() at non-default head configurations
DETECT_CONFIGS = [
    ('classes1', {'num_classes': 1}, {}),
    ('classes20', {'num_classes': 20}, {}),
    ('classes97', {'num_classes': 97}, {}),          # past the fused arg-max: stored logits
    ('aspect1', {'aspect_ratios': [1.0]}, {}),
    ('max300', {}, {'max_output_size': 300}),
    ('hard', {}, {'method': 'hard'}),
]


@pytest.mark.gpu
@pytest.mark.parametrize('name,over,nms_over', DETECT_CONFIGS, ids=[c[0] for c in DETECT_CONFIGS])
def test_detect_head_configs(name, over, nms_over):
  """D0 at 128 px: detect() twice (graph replay) gives the same bits; its pre-NMS matches the
  oracle's on the engine's own head outputs (sliced with A * C and A * 4), and its detections are
  the oracle's NMS of its own pre-NMS tensors, bit for bit."""
  from test_gpu_network import _engine, _setup
  c, a, w, x = _setup('efficientdet-d0', 128, 2, seed=5, **over)
  for key, v in nms_over.items():
    setattr(c.nms_configs, key, v)
  eng = _engine(c, w, 2, use_cuda_graph=True, image_id_base=4)
  scales = np.asarray([1.25, 0.5], np.float32)
  det1 = eng.detect(torch.from_numpy(x), scales).cpu().numpy().copy()
  det2 = eng.detect(torch.from_numpy(x), scales).cpu().numpy().copy()
  np.testing.assert_array_equal(det1, det2)
  params = c.as_dict()
  max_out = params['nms_configs']['max_output_size']
  assert det1.shape == (2, max_out, 7)
  np.testing.assert_array_equal(det1[:, :, 0], np.asarray([[4.0] * max_out, [5.0] * max_out], np.float32))
  A, C = a.num_anchors, a.num_classes
  assert eng.fuse_class_argmax == (C <= 96)
  eng.forward(torch.from_numpy(x))
  torch.cuda.synchronize()
  cls_l = [eng.cls_out[l][..., :A * C].float().cpu().numpy() for l in a.levels]
  box_l = [eng.box_out[l][..., :A * 4].float().cpu().numpy() for l in a.levels]
  _, ref_scores, ref_classes = po.pre_nms(params, cls_l, box_l)
  np.testing.assert_array_equal(eng.classes.cpu().numpy(), ref_classes)
  np.testing.assert_allclose(eng.scores.cpu().numpy(), ref_scores, rtol=1e-6, atol=1e-7)
  gb, gs, gc = eng.boxes.cpu().numpy(), eng.scores.cpu().numpy(), eng.classes.cpu().numpy()
  codes = np.concatenate([b.reshape(2, -1, 4) for b in box_l], 1)
  check_decode(gb, codes, eng.anchors.boxes, name)
  iou_t, score_t, tf_sigma = po.nms_v5_params(params['nms_configs'])
  for i in range(2):
    idx, sc, v = po.non_max_suppression_v5(gb[i], gs[i], max_out, iou_t, score_t, tf_sigma, True)
    assert int(eng.valid[i]) == v
    np.testing.assert_array_equal(eng.sel_index[i].cpu().numpy(), idx)
    np.testing.assert_array_equal(det1[i, :, 5], sc)
    np.testing.assert_array_equal(det1[i, :, 1:5], po.clip_boxes(gb[i][idx], 128) * scales[i])
    np.testing.assert_array_equal(det1[i, :, 6], (gc[i][idx] + 1).astype(np.float32))
