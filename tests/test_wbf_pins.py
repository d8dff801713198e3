"""Weighted box fusion pins, without a GPU: the numpy oracle (tests/wbf_oracle.py) equals, bit for
bit, every golden the unmodified reference wbf.py recorded (tests/golden/make_wbf_golden.py), the
goldens show the reference's class-range behaviour the kernel keeps, and csrc/wbf.cu compiles for
sm_90a without spills."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import wbf_oracle as wo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'wbf.npz')


def _cases():
  data = np.load(GOLDEN)
  names = sorted({k.split('/')[0] for k in data.files})
  return {n: (data[n + '/det'], data[n + '/meta'], data[n + '/scale'], data[n + '/out']) for n in names}


CASES = _cases()


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_equals_reference_golden(name):
  det, (num_models, mask, num_classes, width), scale, want = CASES[name]
  assert det.shape[0] == num_models
  rows = wo.stack_models(list(det), int(mask), scale, int(width))
  got = wo.ensemble(rows, int(num_classes), int(num_models))
  assert wo.same_bits(got, want), (name, got, want)


def test_goldens_cover_the_cases():
  names = set(CASES)
  for method in ('hard', 'gaussian', 'linear'):
    for m in (1, 2, 3):
      assert 'nms_%s_m%d' % (method, m) in names
  assert {'ties', 'equidistant', 'iou_below', 'iou_above', 'big_cluster_m1', 'empty_and_dropped',
          'all_dummy_m1', 'no_dummy_m2', 'nothing_fused'} <= names


def test_class_range_quirk_is_the_reference_behaviour():
  """nms_np's classes are 1-based: wbf.py fuses range(num_classes), so class num_classes is
  dropped and class 0 (nms_np's dummy rows) becomes one cluster at score -1e5."""
  det, (_, _, num_classes, _), _, out = CASES['empty_and_dropped']
  assert (det[0][:, 6] == num_classes).any() and not (out[:, 6] == num_classes).any()
  for name in ('all_dummy_m1', 'all_dummy_m2'):
    out = CASES[name][3]
    assert out.shape == (1, 7) and out[0, 5] == np.float32(-1e5) and out[0, 6] == 0
  for name in [n for n in CASES if n.startswith('nms_')]:
    det, (_, _, num_classes, _), _, out = CASES[name]
    dummies = (det[..., 5] == np.float32(-1e5)).any()
    assert ((out[:, 6] == 0).sum() == 1) == dummies, name
    assert not (out[:, 6] == num_classes).any(), name
  assert CASES['nothing_fused'][3].shape == (0, 7)


def test_ties_keep_class_then_creation_order():
  out = CASES['ties'][3]
  half = out[out[:, 5] == np.float32(0.5)]
  # the class-1 clusters (created in input order), then the two class-2 ones
  assert half[:, 6].tolist() == [1, 1, 2, 2]
  assert half[0, 1] == 50 and half[1, 1] == 0 and half[2, 1] == 0 and half[3, 1] == 100


def test_iou_threshold_is_strict_at_0_55f():
  base = CASES['iou_below'][0][0][0]
  below, above = CASES['iou_below'][0][0][1], CASES['iou_above'][0][0][1]
  with np.errstate(all='ignore'):
    assert wo.iou(base, below) < wo.THRESH <= wo.iou(base, above)
  assert len(CASES['iou_below'][3]) == 2 and len(CASES['iou_above'][3]) == 1


def test_oracle_single_member_is_not_a_shortcut():
  """(x * s) / s is not always x in float32: a one-member cluster is averaged like any other."""
  rng = np.random.default_rng(0)
  x = rng.uniform(0, 1000, 20000).astype(np.float32)
  s = rng.uniform(0, 1, 20000).astype(np.float32)
  assert ((x * s) / s != x).any()


def test_wbf_compiles_without_spills():
  from automl_b200 import build
  src = os.path.join(build.CSRC, 'wbf.cu')
  with tempfile.TemporaryDirectory() as tmp:
    res = subprocess.run([build.NVCC] + [f for f in build.FLAGS if f != '--shared'] +
                         ['-Xptxas', '-v', '-c', src, '-o', os.path.join(tmp, 'wbf.o')],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  assert res.returncode == 0, res.stdout
  assert "for 'sm_90a'" in res.stdout
  spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', res.stdout)
  assert spills and all(s == ('0', '0') for s in spills), res.stdout


def test_row_limit_covers_every_registered_config():
  """EDET_WBF_MAX_ROWS holds two models of the largest max_output_size of any registered config."""
  from automl_b200 import hparams_config
  with open(os.path.join(ROOT, 'include', 'automl_b200.h')) as f:
    limit = int(re.search(r'#define EDET_WBF_MAX_ROWS (\d+)', f.read()).group(1))
  names = list(hparams_config.efficientdet_model_param_dict) + list(hparams_config.efficientdet_lite_param_dict)
  biggest = max(int(hparams_config.get_detection_config(n).nms_configs.max_output_size) for n in names)
  assert limit >= 2 * biggest >= 200
