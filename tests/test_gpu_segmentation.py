"""The segmentation head on the GPU, end to end (tf2/efficientdet_keras.py:644-706, 875-915):
parity of the seg logits with the CPU oracle (tests/seg_oracle.py on
oracle/efficientdet_oracle.py's backbone and BiFPN), detection outputs unchanged by the extra
head, a segmentation-only network without head / NMS launches, pipelined and graph execution,
and EfficientDetNet's output tuple."""
import numpy as np
import pytest
import torch

import precision_model as pm
import seg_oracle
from automl_b200 import arch
from automl_b200 import hparams_config
from automl_b200 import weights

pytestmark = pytest.mark.gpu
REL_TOL = 1e-3
BOTH = ['object_detection', 'segmentation']


def rel_l2(a, b):
  a, b = a.double().flatten(), b.double().flatten()
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


def _setup(name, image_size, n, heads, seed=0):
  c = hparams_config.get_efficientdet_config(name)
  c.override(dict(image_size=image_size, heads=heads))
  a = arch.DetArch(c)
  w = weights.synthetic_weights(a, seed)
  h, wd = a.image_hw
  x = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, size=(n, h, wd, 3)).astype(np.float32)
  return c, a, w, x


def _engine(c, w, n, **kw):
  from automl_b200.engine import Engine
  return Engine(c, w, n, **kw)


def seg_device_weights(a, w):
  """pm.device_weights plus the segmentation head: BN folded into the Conv2DTranspose kernels
  (per output channel, axis 2 of the Keras layout) in float64, then rounded to fp16."""
  out = pm.device_weights(a, w)
  for st in a.seg_stages:
    k = np.float64(w[st.kernel_scope + '/kernel'])
    if st.bn_scope:
      g, b = np.float64(w[st.bn_scope + '/gamma']), np.float64(w[st.bn_scope + '/beta'])
      m, v = np.float64(w[st.bn_scope + '/moving_mean']), np.float64(w[st.bn_scope + '/moving_variance'])
      s = g / np.sqrt(v + pm.EPS)
      k = k * s.reshape(1, 1, -1, 1)
      out[st.bn_scope + '/gamma'] = np.ones_like(g, np.float32)
      out[st.bn_scope + '/moving_variance'] = np.full(g.shape, 1.0 - pm.EPS, np.float32)
      out[st.bn_scope + '/moving_mean'] = np.zeros_like(g, np.float32)
      out[st.bn_scope + '/beta'] = (b - m * s).astype(np.float32)
    out[st.kernel_scope + '/kernel'] = pm._r16(k)  # pylint: disable=protected-access
  return out


@pytest.mark.parametrize('name,image_size,n', [
    ('efficientdet-d0', 256, 2),
    ('efficientdet-d0', 640, 2),
    ('efficientdet-d1', 128, 1),            # F = 88: K padded to the k-block
    ('efficientdet-d0', '640x384', 1),      # non-square
])
def test_seg_logits_match_oracle(name, image_size, n):
  c, a, w, x = _setup(name, image_size, n, ['segmentation'])
  eng = _engine(c, w, n, use_cuda_graph=False)
  eng.forward(torch.from_numpy(x))
  got = eng.seg_logits.float().cpu()
  torch.cuda.synchronize()
  ref = seg_oracle.seg_logits(c, w, x, torch.float32)
  h, wd = a.level_hw[c.min_level]
  assert tuple(got.shape) == tuple(ref.shape) == (n, 2 * h, 2 * wd, c.seg_num_classes)
  assert rel_l2(got, ref) < REL_TOL
  # the padding channels of the round8 buffer are zero
  assert bool((eng.seg_out[..., c.seg_num_classes:] == 0).all())


def test_seg_logits_lite0_within_format_error():
  """lite0 (relu6, 'sum' fusion) with random weights is badly conditioned (test_gpu_network.py's
  lite3 test): the fp16 storage format alone is about 1e-3 off, so the device must stay within
  precision_model.bar() of the format model (the oracle with fp16 stores and fp16 folded weights)."""
  c, a, w, x = _setup('efficientdet-lite0', 256, 1, BOTH)
  eng = _engine(c, w, 1, use_cuda_graph=False)
  eng.forward(torch.from_numpy(x))
  got = eng.seg_logits.float().cpu()
  torch.cuda.synchronize()
  ref = seg_oracle.seg_logits(c, w, x, torch.float32)
  model = seg_oracle.seg_logits(c, seg_device_weights(a, w), x, torch.float32, store=pm.eo.fp16_store)
  assert rel_l2(got, ref) < pm.bar(rel_l2(model, ref))


def test_detection_outputs_unchanged_by_the_segmentation_head():
  c2, a, w2, x = _setup('efficientdet-d0', 256, 2, BOTH, seed=3)
  c1, _, w1, _ = _setup('efficientdet-d0', 256, 2, ['object_detection'], seed=3)
  xt = torch.from_numpy(x)
  both, det = _engine(c2, w2, 2), _engine(c1, w1, 2)
  cb, bb = both.forward(xt)
  cd, bd = det.forward(xt)
  torch.cuda.synchronize()
  for l in a.levels:
    assert torch.equal(cb[l], cd[l]) and torch.equal(bb[l], bd[l])
  assert torch.equal(both.detect(xt).clone(), det.detect(xt).clone())


def test_segmentation_only_network():
  c2, a, w2, x = _setup('efficientdet-d0', 256, 2, BOTH, seed=5)
  c1, _, _, _ = _setup('efficientdet-d0', 256, 2, ['segmentation'], seed=5)
  xt = torch.from_numpy(x)
  both, seg = _engine(c2, w2, 2), _engine(c1, w2, 2)   # the segmentation variables of w2
  both.forward(xt)
  cls_out, box_out = seg.forward(xt)
  torch.cuda.synchronize()
  assert torch.equal(seg.seg_logits, both.seg_logits)
  assert cls_out == {} and box_out == {}
  names = seg.op_names()
  assert not any(n.startswith(('class_net', 'box_net')) or n in ('pre_nms', 'nms') for n in names)
  assert sum(n.startswith('segmentation_head/') for n in names) == len(a.seg_stages)
  with pytest.raises(ValueError):
    seg.detect(xt)


@pytest.mark.parametrize('graph', [True, False])
def test_pipelined_and_graph_runs_equal_eager_sequential(graph):
  c, a, w, _ = _setup('efficientdet-d0', 256, 2, BOTH, seed=11)
  rng = np.random.default_rng(12)
  xs = [torch.from_numpy(rng.uniform(-2, 2, size=(2, 256, 256, 3)).astype(np.float32)).cuda()
        for _ in range(3)]
  ref = _engine(c, w, 2, use_cuda_graph=False, pipeline=False)
  want_seg, want_det = [], []
  for x in xs:
    want_det.append(ref.detect(x).clone())
    want_seg.append(ref.seg_logits.clone())
  ref.forward(xs[0])
  torch.cuda.synchronize()
  assert torch.equal(ref.seg_logits, want_seg[0])
  for pipeline in (False, True):
    eng = _engine(c, w, 2, use_cuda_graph=graph, pipeline=pipeline)
    for i, x in enumerate(xs):
      got = eng.detect(x)
      torch.cuda.synchronize()
      assert torch.equal(got, want_det[i]), (pipeline, i)
      assert torch.equal(eng.seg_logits, want_seg[i]), (pipeline, i)
    eng.forward(xs[1])
    torch.cuda.synchronize()
    assert torch.equal(eng.seg_logits, want_seg[1])


@pytest.mark.parametrize('heads', [BOTH, ['segmentation'], ['object_detection']])
def test_efficientdetnet_output_tuple(heads):
  from automl_b200 import efficientdet_arch
  from automl_b200.efficientdet_keras import EfficientDetNet
  c, a, w, x = _setup('efficientdet-d0', 256, 1, heads, seed=7)
  net = EfficientDetNet(config=c, weights=w)
  out = net(x, training=False)
  torch.cuda.synchronize()
  n_det = 2 if 'object_detection' in heads else 0
  assert len(out) == n_det + ('segmentation' in heads)
  if n_det:
    cls_l, box_l = out[0], out[1]
    assert len(cls_l) == len(box_l) == len(a.levels)
    for l, tc, tb in zip(a.levels, cls_l, box_l):
      hh, ww = a.level_hw[l]
      assert tc.dtype == torch.float32 and tuple(tc.shape) == (1, hh, ww, a.num_anchors * a.num_classes)
      assert tuple(tb.shape) == (1, hh, ww, 4 * a.num_anchors)
  if 'segmentation' in heads:
    seg = out[-1]
    assert seg.dtype == torch.float32 and tuple(seg.shape) == (1, 64, 64, c.seg_num_classes)
    ref = seg_oracle.seg_logits(c, w, x, torch.float32)
    assert rel_l2(seg.cpu(), ref) < REL_TOL
  # the legacy graph keeps its two dicts of detection outputs for every config
  cls_d, box_d = efficientdet_arch.efficientdet(x, config=c)
  assert sorted(cls_d) == sorted(box_d) == a.levels
  efficientdet_arch.clear_engines()
