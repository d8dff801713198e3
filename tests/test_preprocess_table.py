"""The host table of the ragged serving pre-process (inference.preprocess_table) against the oracle's
scale-to-fit (oracle/postprocess_oracle.py::image_preprocess): the same image_scale_to_original
bits, and the scaled size the oracle fills before its zero padding."""
import numpy as np
import pytest

from oracle import postprocess_oracle as po

MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]


def _shapes():
  """A seeded few hundred (h, w): COCO-like sizes, small and large, odd and extreme aspects."""
  rng = np.random.default_rng(7)
  shapes = [(480, 640), (640, 480), (427, 640), (375, 500), (612, 612), (1, 1), (1, 700), (700, 1),
            (2, 900), (900, 3), (33, 1), (1, 47), (129, 127)]
  shapes += [tuple(int(v) for v in rng.integers(1, 800, size=2)) for _ in range(200)]
  shapes += [tuple(int(v) for v in rng.integers(1, 48, size=2)) for _ in range(80)]
  return shapes


@pytest.mark.parametrize('image_size', [64, 128, '96x64', (50, 90)])
def test_table_matches_oracle_scale(image_size):
  from automl_b200 import inference, ops, utils
  oh, ow = utils.parse_image_size(image_size)
  shapes = _shapes()
  keep = []
  for h, w in shapes:        # the oracle collapses some extreme aspects to zero size: skip those
    s = min(np.float32(oh) / np.float32(h), np.float32(ow) / np.float32(w))
    if int(np.float32(h) * s) >= 1 and int(np.float32(w) * s) >= 1:
      keep.append((h, w))
  assert len(keep) >= 250
  desc, total, scales = inference.preprocess_table(keep, image_size)
  assert desc.dtype == np.int32 and desc.shape == (len(keep), ops.PRE_DESC_WORDS)
  assert scales.dtype == np.float32 and scales.shape == (len(keep),)
  offsets = desc[:, :2].copy().view(np.int64)[:, 0]
  nbytes = [3 * h * w for h, w in keep]
  assert offsets[0] == 0 and (offsets % 16 == 0).all()
  np.testing.assert_array_equal(np.diff(offsets), [(b + 15) // 16 * 16 for b in nbytes[:-1]])
  assert total == offsets[-1] + nbytes[-1]
  np.testing.assert_array_equal(desc[:, 2:4], keep)
  for i, (h, w) in enumerate(keep):
    out, ref_scale = po.image_preprocess(np.zeros((h, w, 3), np.uint8), image_size, MEAN, STD)
    assert scales[i].tobytes() == np.float32(ref_scale).tobytes(), (h, w, scales[i], ref_scale)
    filled = out[:, :, 0] != 0       # zero pixels normalise to -mean / std, the padding to 0
    sh, sw = int(filled[:, 0].sum()), int(filled[0].sum())
    assert (sh, sw) == (desc[i, 4], desc[i, 5]), (h, w)
    assert 1 <= sh <= oh and 1 <= sw <= ow


@pytest.mark.parametrize('shape', [(1, 2000), (3000, 1), (0, 5), (5, 0)])
def test_table_rejects_collapsing_or_empty_images(shape):
  from automl_b200 import inference
  with pytest.raises(ValueError):
    inference.preprocess_table([(64, 64), shape], 64)


def test_table_of_one_size_is_uniform():
  """All sizes equal: back to back like edet_preprocess's [N, h, w, 3] batch (3 h w is a multiple
  of 16 here), one scale for every image."""
  from automl_b200 import inference
  desc, total, scales = inference.preprocess_table([(480, 640)] * 5, 640)
  assert total == 5 * 3 * 480 * 640
  np.testing.assert_array_equal(desc[:, :2].copy().view(np.int64)[:, 0], np.arange(5) * 3 * 480 * 640)
  assert (scales == scales[0]).all() and (desc[:, 4:] == (480, 640)).all()
