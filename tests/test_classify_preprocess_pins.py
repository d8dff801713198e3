"""CPU pins of the EfficientNet V1 / V2 classification serving path: the eval recipe each registered
model uses, the crop rule, TF's bicubic coefficient table, hand-derived resize fixtures, and the
oracle (tests/classify_oracle.py) against plain float64 loops, in the style of
tests/test_oracle_definitions.py.

The recipe per model comes from the REAL reference config: tests/golden/classify_configs.json
records cfg.data.augname and cfg.eval.isize of every registered name
(tests/golden/make_classify_golden.py).
"""
import json
import math
import os

import numpy as np
import pytest
import torch

import classify_oracle as co
from automl_b200.efficientnetv2 import effnetv2_configs
from automl_b200.efficientnetv2 import preprocessing

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                       'classify_configs.json')) as _f:
  GOLDEN = json.load(_f)


# ---- configs ------------------------------------------------------------------------------------
def test_golden_covers_every_registered_model():
  assert len(GOLDEN) == 18
  legacy = sorted(m for m, g in GOLDEN.items() if g['augname'].startswith('effnetv1_'))
  assert len(legacy) == 14
  assert sorted(set(GOLDEN) - set(legacy)) == ['efficientnetv2-%s' % s for s in ('l', 'm', 's', 'xl')]


@pytest.mark.parametrize('model', sorted(GOLDEN))
def test_augname_and_eval_size_match_the_reference(model):
  cfg = effnetv2_configs.get_model_config(model)
  assert cfg.data.augname == GOLDEN[model]['augname']
  assert cfg.eval.isize == GOLDEN[model]['isize']
  assert sorted(cfg.data.as_dict()) == ['augname']      # no training-only fields
  assert preprocessing.is_legacy(cfg.data.augname) == (model not in (
      'efficientnetv2-s', 'efficientnetv2-m', 'efficientnetv2-l', 'efficientnetv2-xl'))


# ---- crop rule ----------------------------------------------------------------------------------
def test_crop_window_of_an_imagenet_decode():
  """375 x 500 at S = 224: side int(0.875 * 375) = 328; the odd margin 47 splits 23 / 24."""
  for fn in (preprocessing.crop_window, co.crop_window):
    assert fn(375, 500, 224, False) == (23, 86, 328, 328)
    assert fn(375, 500, 224, True) == (24, 86, 328, 328)


def test_crop_side_truncates_the_float32_product():
  """252 / 284 * 71 is 63 exactly, but float32(252 / 284) * 71 rounds to just below 63."""
  prod = np.float32(252 / 284) * np.float32(71)
  assert prod < 63 and 252 * 71 == 63 * 284
  for fn in (preprocessing.crop_window, co.crop_window):
    assert fn(71, 100, 252, False) == (4, 19, 62, 62)
    assert fn(71, 100, 252, True) == (5, 19, 62, 62)


def test_bilinear_recipe_crops_only_below_320():
  for fn in (preprocessing.crop_window, co.crop_window):
    assert fn(375, 500, 320, False) == (0, 0, 375, 500)
    assert fn(375, 500, 384, False) == (0, 0, 375, 500)
    assert fn(375, 500, 319, False)[2] == int(np.float32(319 / 351) * np.float32(375))
    assert fn(375, 500, 384, True) == (15, 77, 346, 346)   # the legacy recipe always crops


def test_product_crop_window_equals_the_oracle():
  rng = np.random.default_rng(0)
  for _ in range(2000):
    h, w = (int(v) for v in rng.integers(2, 1500, size=2))
    s = int(rng.integers(32, 801))
    for legacy in (False, True):
      try:
        want = co.crop_window(h, w, s, legacy)
      except ValueError:
        with pytest.raises(ValueError):
          preprocessing.crop_window(h, w, s, legacy)
        continue
      assert preprocessing.crop_window(h, w, s, legacy) == want, (h, w, s, legacy)


def test_empty_crop_is_refused():
  with pytest.raises(ValueError):
    preprocessing.crop_window(1, 500, 224, True)
  with pytest.raises(ValueError):
    preprocessing.crop_window(500, 1, 224, False)
  assert preprocessing.crop_window(1, 500, 384, False) == (0, 0, 1, 500)


def test_image_table_rows():
  desc, total = preprocessing.image_table([(375, 500), (10, 7), (224, 224)], 224, True)
  assert desc.dtype == np.int32 and desc.shape == (3, 8)
  assert list(desc[:, :2].copy().view(np.int64)[:, 0]) == [0, 375 * 500 * 3, 375 * 500 * 3 + 210]
  assert total == 3 * (375 * 500 + 70 + 224 * 224)
  assert list(desc[0, 2:]) == [375, 500, 24, 86, 328, 328]
  assert list(desc[2, 2:]) == [224, 224, 14, 14, 196, 196]   # 0.875 * 224 = 196 exactly


# ---- bicubic table ------------------------------------------------------------------------------
def _weights(off):
  t = co.TABLE
  return [t[2 * off + 1], t[2 * off], t[2 * (1024 - off)], t[2 * (1024 - off) + 1]]


def test_bicubic_table():
  assert co.TABLE.dtype == np.float32 and co.TABLE.shape == (2050,)
  assert np.array_equal(preprocessing.bicubic_table().view(np.int32), co.TABLE.view(np.int32))
  assert _weights(0) == [0, 1, 0, 0]
  assert _weights(512) == [-0.09375, 0.59375, 0.59375, -0.09375]
  for off in range(0, 1025, 7):                         # the Keys kernel is a partition of unity
    assert abs(sum(float(v) for v in _weights(off)) - 1) < 1e-6


def test_table_offset_rounds_half_to_even():
  """1 -> 2048 pixels: dst d samples d / 2048, i.e. (d / 2) / 1024 of a table step."""
  fi, off = co.bicubic_offsets(2048, 1)
  assert list(fi[:8]) == [0] * 8
  assert list(off[:8]) == [0, 0, 1, 2, 2, 2, 3, 4]      # .5 -> 0, 1.5 -> 2, 2.5 -> 2, 3.5 -> 4


# ---- hand-derived fixtures ----------------------------------------------------------------------
def test_bilinear_fixture():
  img = np.zeros((1, 2, 3), np.uint8)
  img[0, 1] = 255
  got = co.resize_bilinear(img.astype(np.float32), 1, 4)[0, :, 0]
  assert list(got) == [0, 63.75, 191.25, 255]
  out = co.preprocess_window(img, 4, False, (0, 0, 1, 2))
  assert np.array_equal(out[:, :, 0], np.tile((np.float32([0, 63.75, 191.25, 255]) - 128) / 128, (4, 1)))


def test_bicubic_at_scale_one_is_the_identity():
  img = np.random.default_rng(1).integers(0, 256, size=(9, 13, 3)).astype(np.float32)
  assert np.array_equal(co.resize_bicubic(img, 9, 13), img)
  out = co.preprocess_window(img.astype(np.uint8), 9, True, (0, 2, 9, 9))
  assert np.array_equal(out, (img[:, 2:11] - co.MEAN_RGB) / co.STDDEV_RGB)


def test_bicubic_step_clamps_at_the_edges():
  """[0, 0, 255, 255] -> 8 pixels: the overshoot of the Keys kernel shows on both sides of the step,
  and at the last pixel the taps beyond the edge repeat 255, so there is none."""
  img = np.zeros((1, 4, 3), np.float32)
  img[0, 2:] = 255
  got = co.resize_bicubic(img, 1, 8)[0, :, 0]
  assert list(got) == [0, -23.90625, 0, 127.5, 255, 278.90625, 255, 255]


# ---- the oracle against plain float64 loops -----------------------------------------------------
def _loop_bilinear(img, s):
  h, w = img.shape[:2]
  out = np.zeros((s, s, 3))
  for y in range(s):
    fy = (y + 0.5) * h / s - 0.5
    y0, y1, ly = max(math.floor(fy), 0), min(math.ceil(fy), h - 1), fy - math.floor(fy)
    for x in range(s):
      fx = (x + 0.5) * w / s - 0.5
      x0, x1, lx = max(math.floor(fx), 0), min(math.ceil(fx), w - 1), fx - math.floor(fx)
      for c in range(3):
        top = img[y0, x0, c] * (1 - lx) + img[y0, x1, c] * lx
        bot = img[y1, x0, c] * (1 - lx) + img[y1, x1, c] * lx
        out[y, x, c] = (top * (1 - ly) + bot * ly - 128) / 128
  return out


def _keys(t, a=-0.75):
  t = abs(t)
  if t <= 1:
    return ((a + 2) * t - (a + 3)) * t * t + 1
  if t < 2:
    return ((a * t - 5 * a) * t + 8 * a) * t - 4 * a
  return 0.0


def _loop_bicubic(img, s):
  h, w = img.shape[:2]
  mean = [0.485 * 255, 0.456 * 255, 0.406 * 255]
  std = [0.229 * 255, 0.224 * 255, 0.225 * 255]

  def taps(d, n_in):
    src = d * n_in / s
    i = math.floor(src)
    frac = round((src - i) * 1024) / 1024          # TF samples its kernel on 1024 steps
    return [(min(max(i + j, 0), n_in - 1), _keys(frac - j)) for j in (-1, 0, 1, 2)]

  out = np.zeros((s, s, 3))
  for y in range(s):
    ty = taps(y, h)
    for x in range(s):
      tx = taps(x, w)
      for c in range(3):
        v = sum(wy * wx * img[iy, ix, c] for iy, wy in ty for ix, wx in tx)
        out[y, x, c] = (v - mean[c]) / std[c]
  return out


@pytest.mark.parametrize('shape,s,legacy', [((37, 53), 20, False), ((53, 37), 20, True),
                                            ((11, 9), 20, False), ((30, 31), 17, True),
                                            ((1, 25), 12, True), ((25, 1), 12, False)])
def test_oracle_recipes_equal_float64_loops(shape, s, legacy):
  img = np.random.default_rng(shape[0] * 100 + shape[1]).integers(0, 256, size=shape + (3,)).astype(np.uint8)
  h, w = shape
  window = co.crop_window(h, w, s, legacy) if min(h, w) > 1 else (0, 0, h, w)
  got = co.preprocess_window(img, s, legacy, window)
  y0, x0, ch, cw = window
  crop = img[y0:y0 + ch, x0:x0 + cw].astype(np.float64)
  ref = _loop_bicubic(crop, s) if legacy else _loop_bilinear(crop, s)
  assert got.dtype == np.float32 and got.shape == (s, s, 3)
  assert np.abs(got - ref).max() < 1e-4


def test_softmax_topk_oracle():
  x = np.array([[1, 3, 3, 2, 3], [0, 0, 0, 0, 0]], np.float32)
  p, c = co.softmax_topk(x, 4)
  assert c.tolist() == [[1, 2, 4, 3], [0, 1, 2, 3]]
  e = np.exp(np.array([1, 3, 3, 2, 3], np.float64) - 3)
  assert np.allclose(p[0], e[[1, 2, 4, 3]] / e.sum(), rtol=1e-15)
  assert np.allclose(p[1], 0.2, rtol=1e-15)


# ---- errors before any device work ---------------------------------------------------------------
def test_preprocess_image_refuses_what_it_cannot_do():
  img = np.zeros((10, 12, 3), np.uint8)
  with pytest.raises(NotImplementedError):
    preprocessing.preprocess_image(img, 224, is_training=True)
  for dtype in (np.float16, torch.bfloat16, 'uint8'):
    with pytest.raises(ValueError):
      preprocessing.preprocess_image(img, 224, image_dtype=dtype)
  for bad in (img.astype(np.float32), img[..., :2], img[..., 0], torch.zeros(10, 12, 3)):
    with pytest.raises(ValueError):
      preprocessing.preprocess_image(bad, 224)
  with pytest.raises(ValueError):
    preprocessing.preprocess_image(np.zeros((1, 12, 3), np.uint8), 224, augname='effnetv1_autoaug')
