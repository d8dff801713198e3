"""Host side of the segmentation masks (no GPU): the integer cell rule of edet_seg_masks against a
float64 restatement, the mask table the driver uploads, and the requests it refuses before
anything is enqueued."""
import numpy as np
import pytest
import torch

import seg_mask_oracle as smo

# D0 and lite0 at their registered image sizes, with the logits grid of min_level 3 (f = 4)
CONFIGS = [('efficientdet-d0', 512), ('efficientdet-lite0', 320)]
F = 4


def _sweep():
  """(h, w): 1x1, single rows and columns, images smaller and larger than the network, odd and
  even sides, and a seeded spread."""
  shapes = [(1, 1), (1, 5000), (5000, 1), (2, 2), (3, 5), (7, 640), (480, 640), (640, 480),
            (427, 640), (375, 500), (612, 612), (512, 512), (320, 320), (511, 513), (1023, 1024),
            (4000, 3000), (2999, 4001), (64, 48), (127, 129)]
  rng = np.random.default_rng(11)
  shapes += [tuple(int(v) for v in rng.integers(1, 2048, size=2)) for _ in range(60)]
  return shapes


def _scaled(h, w, size):
  """Scaled size by the float32 scale-to-fit of edet_preprocess (may be 0 for extreme aspects)."""
  s = min(np.float32(size) / np.float32(h), np.float32(size) / np.float32(w))
  return int(np.float32(h) * s), int(np.float32(w) * s)


@pytest.mark.parametrize('name,size', CONFIGS)
def test_cell_rule_equals_float64_restatement(name, size):
  from automl_b200 import hparams_config
  c = hparams_config.get_efficientdet_config(name)
  assert c.image_size == size and 2 ** (c.min_level - 1) == F
  grid = size // F
  for h, w in _sweep():
    for n, scaled in zip((h, w), _scaled(h, w, size)):
      scaled = max(scaled, 1)      # collapsing images are refused; the rule is pinned regardless
      got = smo.cells(n, scaled, F, grid)
      np.testing.assert_array_equal(got, smo.cells_float64(n, scaled, F, grid), err_msg=str((h, w)))
      assert got[0] >= 0 and got[-1] <= (scaled - 1) // F   # never a padding cell
      assert (np.diff(got) >= 0).all()


@pytest.mark.parametrize('name,size', CONFIGS)
def test_mask_table_layout(name, size):
  """Rows of 24 bytes (int64 offset, h, w, scaled_h, scaled_w), masks back to back, the scaled
  size of the pre-process table."""
  from automl_b200 import inference, ops
  shapes = [(h, w) for h, w in _sweep() if min(_scaled(h, w, size)) >= 1]
  assert len(shapes) > 60
  table, total = inference.seg_mask_table(shapes, size)
  desc, _, _ = inference.preprocess_table(shapes, size)
  assert table.dtype == np.int32 and table.shape == (len(shapes), ops.SEG_MASK_WORDS)
  assert table.nbytes == 24 * len(shapes)
  offsets = table[:, :2].copy().view(np.int64)[:, 0]
  areas = np.array([h * w for h, w in shapes], np.int64)
  np.testing.assert_array_equal(offsets, np.concatenate([[0], np.cumsum(areas)[:-1]]))
  assert total == int(areas.sum())
  np.testing.assert_array_equal(table[:, 2:4], shapes)
  np.testing.assert_array_equal(table[:, 4:], desc[:, 4:])
  for (h, w), (sh, sw) in zip(shapes, table[:, 4:]):
    assert (sh, sw) == _scaled(h, w, size)


def test_mask_table_offsets_past_2_31():
  from automl_b200 import inference
  table, total = inference.seg_mask_table([(30000, 30000)] * 3, 512)
  offsets = table[:, :2].copy().view(np.int64)[:, 0]
  assert list(offsets) == [0, 9 * 10 ** 8, 18 * 10 ** 8] and total == 27 * 10 ** 8 > 2 ** 31


def test_uniform_tensor_request():
  from automl_b200 import inference
  shapes, table, total = inference.segment_request(torch.zeros(4, 48, 64, 3, dtype=torch.uint8), 512, 3)
  assert shapes == [(48, 64)] * 4 and total == 4 * 48 * 64
  np.testing.assert_array_equal(table[:, 4:], [(384, 512)] * 4)


@pytest.mark.parametrize('num_classes', [0, 257, 1000])
def test_class_count_outside_uint8_raises(num_classes):
  from automl_b200 import inference
  with pytest.raises(ValueError):
    inference.segment_request([np.zeros((8, 8, 3), np.uint8)], 512, num_classes)


@pytest.mark.parametrize('num_classes', [257, 0])
def test_op_refuses_class_count_before_any_launch(num_classes):
  from automl_b200 import ops
  logits = torch.zeros(1, 4, 4, 264, dtype=torch.float16)
  table = torch.zeros(1, ops.SEG_MASK_WORDS, dtype=torch.int32)
  with pytest.raises(ValueError):
    ops.seg_masks(logits, num_classes, 4, table, (16, 16), torch.zeros(256, dtype=torch.uint8))


@pytest.mark.parametrize('images', [
    [np.zeros((8, 8, 3), np.float32)],
    [np.zeros((8, 8, 3), np.uint8), np.zeros((8, 8, 3), np.int16)],
    [np.zeros((8, 8), np.uint8)],
    [np.zeros((8, 8, 4), np.uint8)],
    torch.zeros(2, 8, 8, 3, dtype=torch.float32),
    [],
    [np.zeros((0, 8, 3), np.uint8)],
    [np.zeros((1, 5000, 3), np.uint8)],       # collapses to zero rows at 512
], ids=['float32', 'int16', 'gray', 'rgba', 'float_tensor', 'empty_request', 'empty_image',
        'collapses'])
def test_invalid_requests_raise(images):
  """Each entry point's host checks, before anything is enqueued: decoded_images, then the table
  builder (detection of ragged requests and TTA: preprocess_table, segmentation: segment_request,
  classification: image_table, with the request's count)."""
  from automl_b200 import inference, staging
  from automl_b200.efficientnetv2 import preprocessing
  forms = {
      'detection': lambda: inference.preprocess_table(staging.decoded_images(images).shapes, 512),
      'segmentation': lambda: inference.segment_request(images, 512, 3),
      'tta': lambda: inference.preprocess_table(staging.decoded_images(images).shapes, 512),
      'classification': lambda: preprocessing.image_table(
          staging.decoded_images(images, n=len(images) or 1).shapes, 224, False),
  }
  for check in forms.values():
    with pytest.raises(ValueError):
      check()


def test_detection_only_driver_refuses_masks():
  """Checked before anything is built: no GPU needed."""
  from automl_b200 import inference
  drv = inference.ServingDriver('efficientdet-d0', '_', batch_size=1)
  with pytest.raises(ValueError):
    drv.segment_images([np.zeros((8, 8, 3), np.uint8)])
  seg = inference.ServingDriver('efficientdet-d0', '_', batch_size=1,
                                model_params={'heads': ['segmentation']})
  with pytest.raises(NotImplementedError):
    seg.segment_images([np.zeros((8, 8, 3), np.uint8)], resize='bilinear')


def test_oracle_argmax_rule():
  """First index on ties and the first NaN wins, as np.argmax (and tf.argmax) decide."""
  lg = np.array([[[[1, 3, 3, 0], [0, -0.0, 0, 0], [2, np.nan, 5, np.nan]]]], np.float16)
  assert smo.class_map(lg, 4).tolist() == [[[1, 0, 1]]]
  assert smo.class_map(lg, 1).tolist() == [[[0, 0, 0]]]
  m = smo.masks(lg, 3, 1, [(1, 3, 1, 3)])[0]
  assert m.tolist() == [[1, 0, 1]]
