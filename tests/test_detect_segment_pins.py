"""Host side of ServingDriver.submit_with_masks (no GPU): every request it refuses is refused before
the driver builds an engine or enqueues anything, with the words of submit() and submit_segment()."""
import numpy as np
import pytest
import torch

BOTH = ['object_detection', 'segmentation']
IMAGE = [np.zeros((8, 8, 3), np.uint8)]


def _driver(heads=None, batch_size=1, **params):
  from automl_b200 import inference
  if heads is not None:
    params['heads'] = heads
  return inference.ServingDriver('efficientdet-d0', '_', batch_size=batch_size, model_params=params)


def _refused(drv, error, images=IMAGE, match=None, **kwargs):
  """Each entry point raises `error` and leaves the driver unbuilt."""
  for call in (drv.submit_with_masks, drv.serve_images_with_masks,
               lambda r, **kw: list(drv.serve_stream_with_masks([r]))):
    with pytest.raises(error, match=match):
      call(images, **kwargs)
  assert drv._engines is None                                       # pylint: disable=protected-access


@pytest.mark.parametrize('heads', [None, ['object_detection'], ['segmentation'], []],
                         ids=['default', 'detection', 'segmentation', 'none'])
def test_both_heads_needed(heads):
  _refused(_driver(heads), ValueError, match="'object_detection' and 'segmentation' in heads")


@pytest.mark.parametrize('num_classes', [257, 1000, 0])
def test_class_count_outside_uint8_raises(num_classes):
  _refused(_driver(BOTH, seg_num_classes=num_classes), ValueError, match='uint8 masks hold')


def test_bilinear_masks_not_built():
  drv = _driver(BOTH)
  with pytest.raises(NotImplementedError, match='only nearest sampling'):
    drv.submit_with_masks(IMAGE, resize='bilinear')
  assert drv._engines is None                                       # pylint: disable=protected-access


def test_not_built_under_torch_distributed(monkeypatch):
  monkeypatch.setattr(torch.distributed, 'is_available', lambda: True)
  monkeypatch.setattr(torch.distributed, 'is_initialized', lambda: True)
  _refused(_driver(BOTH), NotImplementedError, match='under torch.distributed')


@pytest.mark.parametrize('images', [
    [np.zeros((8, 8, 3), np.float32)],
    [np.zeros((8, 8, 3), np.uint8), np.zeros((8, 8, 3), np.int16)],
    [np.zeros((8, 8), np.uint8)],
    [np.zeros((8, 8, 4), np.uint8)],
    torch.zeros(2, 8, 8, 3, dtype=torch.float32),
    torch.zeros(2, 8, 8, 3, dtype=torch.uint8)[..., :2],
    [],
], ids=['float32', 'int16', 'gray', 'rgba', 'float_tensor', 'two_channel_tensor', 'empty_request'])
def test_invalid_images_raise(images):
  _refused(_driver(BOTH, batch_size=None), ValueError, images=images)


def test_count_other_than_batch_size_raises():
  _refused(_driver(BOTH, batch_size=2), ValueError, images=IMAGE * 3, match='expected 2 images')
