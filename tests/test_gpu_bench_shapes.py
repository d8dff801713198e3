"""Parity at the shapes that are BENCHMARKED (BASELINE.json configs 2-5), not only at toy sizes:

  * EfficientDet-D0 640x640 batch 32 (the headline): every block / BiFPN / head tensor against the
    oracle at the 1e-3 bar, and the detections of the graph-replayed engine bit-equal to the
    oracle's NMS-V5 on the engine's own pre-NMS tensors (K = 76 725 anchors, gaussian);
  * EfficientDet-D4 1024x1024 and D7x 1536x1536 (batch 1 of the per-GPU batch);
  * EfficientNetV2-S 384x384;
  * the NMS-V5 kernel alone at K = 76 725 (gaussian and hard).

The measured errors are written to parity_bench_shapes.json in the system temporary directory.
"""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from automl_b200 import arch
from automl_b200 import hparams_config
from automl_b200 import weights
from oracle import efficientdet_oracle as eo
from oracle import postprocess_oracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT = os.path.join(tempfile.gettempdir(), 'parity_bench_shapes.json')


def rel_l2(a, b):
  a, b = a.double().flatten(), b.double().flatten()
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


def _record(key, value):
  os.makedirs(os.path.dirname(REPORT), exist_ok=True)
  data = {}
  if os.path.exists(REPORT):
    with open(REPORT) as f:
      data = json.load(f)
  data[key] = value
  with open(REPORT, 'w') as f:
    json.dump(data, f, indent=1, sort_keys=True)


def _network_errors(name, image_size, n, seed=0):
  from automl_b200.engine import Engine
  c = hparams_config.get_efficientdet_config(name)
  c.override(dict(image_size=image_size))
  a = arch.DetArch(c)
  w = weights.synthetic_weights(a, seed)
  h, wd = a.image_hw
  x = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, size=(n, h, wd, 3)).astype(np.float32)
  torch.set_num_threads(min(32, os.cpu_count() or 1))
  orc = eo.Oracle(c, w, torch.float32)
  cls_ref, box_ref = orc(x)
  eng = Engine(c, w, n)
  cls_out, box_out = eng.forward(torch.from_numpy(x))
  torch.cuda.synchronize()
  errs = {'blocks': {}, 'fpn': {}, 'cls': {}, 'box': {}}
  for b in a.blocks:
    got = eng.buffers[b.name + '/out'].float().cpu().permute(0, 3, 1, 2)
    errs['blocks'][b.name] = rel_l2(got, orc.endpoints[b.name])
  for l in a.levels:
    errs['fpn'][str(l)] = rel_l2(eng.fpn_feats[l].float().cpu().permute(0, 3, 1, 2),
                                 orc.endpoints['fpn_%d' % l])
    errs['cls'][str(l)] = rel_l2(cls_out[l].float().cpu(), cls_ref[l])
    errs['box'][str(l)] = rel_l2(box_out[l].float().cpu(), box_ref[l])
  return c, a, eng, x, errs


def _worst(errs):
  return {k: max(v.values()) for k, v in errs.items()}


def test_d0_640_batch32_network_and_detections():
  """BASELINE config 2 exactly as bench.py runs it."""
  c, a, eng, x, errs = _network_errors('efficientdet-d0', 640, 32)
  worst = _worst(errs)
  _record('efficientdet-d0 640x640 batch 32', dict(worst, anchors=eng.total_anchors))
  for group, e in worst.items():
    assert e < 1e-3, (group, errs[group])
  # detections: CUDA graph replay (the benchmarked path) vs the oracle post-process run on the
  # engine's own pre-NMS tensors -> bit-equal indices, soft scores, boxes, classes
  assert eng.total_anchors == 76725
  scales = np.linspace(0.5, 2.0, 32).astype(np.float32)
  det = eng.detect(torch.from_numpy(x), scales).cpu().numpy().copy()
  det2 = eng.detect(torch.from_numpy(x), scales).cpu().numpy()
  np.testing.assert_array_equal(det, det2)
  gb, gs, gc = eng.boxes.cpu().numpy(), eng.scores.cpu().numpy(), eng.classes.cpu().numpy()
  params = c.as_dict()
  cls_l = [eng.cls_out[l][..., :810].float().cpu().numpy() for l in a.levels]
  box_l = [eng.box_out[l][..., :36].float().cpu().numpy() for l in a.levels]
  ref_boxes, ref_scores, ref_classes = po.pre_nms(params, cls_l, box_l)
  np.testing.assert_array_equal(gc, ref_classes)
  np.testing.assert_allclose(gs, ref_scores, rtol=1e-6, atol=1e-7)
  np.testing.assert_allclose(gb, ref_boxes, rtol=1e-5, atol=2e-4)
  iou_t, score_t, tf_sigma = po.nms_v5_params(params['nms_configs'])
  sel, valid = eng.sel_index.cpu().numpy(), eng.valid.cpu().numpy()
  for i in range(0, 32, 3):     # 11 of the 32 images (the Python heap oracle takes ~1 s each)
    idx, sc, v = po.non_max_suppression_v5(gb[i], gs[i], 100, iou_t, score_t, tf_sigma, True)
    assert valid[i] == v
    np.testing.assert_array_equal(sel[i], idx)
    np.testing.assert_array_equal(det[i, :, 5], sc)
    np.testing.assert_array_equal(det[i, :, 1:5], po.clip_boxes(gb[i][idx], 640) * scales[i])
    np.testing.assert_array_equal(det[i, :, 6], (gc[i][idx] + 1).astype(np.float32))
  _record('efficientdet-d0 640x640 batch 32 nms', {'images_checked': 11,
                                                    'full_queue_images': eng.nms_fallback_count()})


def test_d4_1024():
  """BASELINE config 4 (one image of the per-GPU batch of 8)."""
  _, _, _, _, errs = _network_errors('efficientdet-d4', 1024, 1)
  worst = _worst(errs)
  _record('efficientdet-d4 1024x1024 batch 1', worst)
  for group, e in worst.items():
    assert e < 1e-3, (group, errs[group])


def test_d7x_1536():
  """BASELINE config 5.  55 MBConv blocks and 8 un-normalised 'sum' BiFPN cells on random
  weights: this model does NOT meet the 1e-3 bar with fp16 activation / weight storage, kernels
  aside -- the fp32 oracle with nothing but the engine's rounding sites applied (fp16 tensors in
  HBM, BN folded into fp16 GEMM weights: tests/precision_model.py) is itself that far from the
  plain fp32 oracle.  DESIGN.md section 6 has the per-rounding-site budget and why only a
  split-precision (fp16 hi + lo) storage mode -- not built -- can reach 1e-3 here.  Asserted: every
  tensor within 1.5x the format model + 1e-4 (the kernels add nothing beyond the format), plus
  absolute regression guards."""
  import precision_model as pm
  c, a, eng, x, errs = _network_errors('efficientdet-d7x', 1536, 1)
  w = weights.synthetic_weights(a, 0)
  model = eo.Oracle(c, pm.device_weights(a, w), torch.float32, store=eo.fp16_store)
  cls_m, box_m = model(x)
  ref = eo.Oracle(c, w, torch.float32)
  cls_r, box_r = ref(x)
  merr = {'blocks': {b.name: rel_l2(model.endpoints[b.name], ref.endpoints[b.name]) for b in a.blocks},
          'fpn': {str(l): rel_l2(model.endpoints['fpn_%d' % l], ref.endpoints['fpn_%d' % l]) for l in a.levels},
          'cls': {str(l): rel_l2(cls_m[l], cls_r[l]) for l in a.levels},
          'box': {str(l): rel_l2(box_m[l], box_r[l]) for l in a.levels}}
  worst = _worst(errs)
  _record('efficientdet-d7x 1536x1536 batch 1', dict(worst, format_model=_worst(merr)))
  for group in errs:
    for k, dev in errs[group].items():
      assert dev < pm.bar(merr[group][k]), (group, k, dev, merr[group][k])
  assert worst['blocks'] < 3.5e-3, errs['blocks']
  assert worst['fpn'] < 3.8e-3, errs['fpn']
  assert worst['cls'] < 5e-3, errs['cls']
  assert worst['box'] < 6.2e-3, errs['box']


def test_effnetv2_s_384():
  """BASELINE config 3 at its own resolution (batch 2 of the 128): every endpoint within 2e-3
  absolute and within 1.5x the format model (tests/precision_model.py) + 1e-4."""
  from automl_b200.efficientnetv2 import effnetv2_model
  name = 'efficientnetv2-s'
  a = effnetv2_model.EffNetV2Arch(name)
  w = effnetv2_model.synthetic_weights(a, 11)
  model = effnetv2_model.get_model(name, weights=w, batch_size=2, image_size=384)
  x = np.random.default_rng(3).uniform(-1, 1, size=(2, 384, 384, 3)).astype(np.float32)
  model(torch.from_numpy(x), with_endpoints=True)
  torch.cuda.synchronize()
  import precision_model as pm
  merr, ref = pm.effnetv2_format_errors(a, w, x)     # what fp16 storage alone costs (no kernel)
  errs = {k: rel_l2(t.float().cpu().permute(0, 3, 1, 2), ref[k]) for k, t in model.endpoints.items()}
  _record('efficientnetv2-s 384x384 batch 2', {'worst': max(errs.values()),
                                              'stem_to_stage2': max(errs[k] for k in errs if k in ('stem', 'reduction_1', 'reduction_2')),
                                              'format_model_worst': max(merr.values())})
  assert max(errs.values()) < 2e-3, errs
  for k, e in errs.items():       # the last stage is past 1e-3 because the FORMAT is (1.59e-3 in the model)
    assert e < pm.bar(merr[k]), (k, e, merr[k])


@pytest.mark.parametrize('method', ['gaussian', 'hard'])
def test_nms_v5_at_bench_k(method):
  """The NMS kernel alone at K = 76 725 candidates per image (D0 / D1 at 640): fast path with its
  16 384-candidate compaction, run-time exactness proof and full-queue fallback."""
  from automl_b200 import ops
  import test_gpu_kernels as tk
  k, n = 76725, 4
  rng = np.random.default_rng(76725 + len(method))
  boxes, scores, classes = tk._nms_inputs(rng, n, k, image=640.0)   # pylint: disable=protected-access
  if method == 'hard':
    scores[:, 1::11] = scores[:, 0:1]
  params = tk._params(640, method=method, score_thresh=None)        # pylint: disable=protected-access
  iou_t, score_t, tf_sigma = po.nms_v5_params(params['nms_configs'])
  dev = 'cuda:0'
  det = torch.empty(n, 100, 7, device=dev)
  sel = torch.empty(n, 100, dtype=torch.int32, device=dev)
  valid = torch.empty(n, dtype=torch.int32, device=dev)
  work = torch.empty(ops.nms_work_bytes(n, k), dtype=torch.uint8, device=dev)
  ops.nms_v5(torch.from_numpy(boxes).to(dev), torch.from_numpy(scores).to(dev),
             torch.from_numpy(classes).to(dev), None, 0, 100, iou_t, score_t, tf_sigma,
             (640.0, 640.0), det, sel, valid, work)
  torch.cuda.synchronize()
  for i in range(n):
    idx, sc, v = po.non_max_suppression_v5(boxes[i], scores[i], 100, iou_t, score_t, tf_sigma, True)
    assert int(valid[i]) == v
    np.testing.assert_array_equal(sel[i].cpu().numpy(), idx)
    np.testing.assert_array_equal(det[i, :, 5].cpu().numpy(), sc)
    np.testing.assert_array_equal(det[i, :, 1:5].cpu().numpy(), po.clip_boxes(boxes[i][idx], 640))
