"""EfficientDetModel's refusals, without a GPU: each bad call raises before any device work.

The engine factory and both pre-process entry points are replaced by a stub that raises
DeviceWork, so a refusal that came after the first of them would surface as DeviceWork instead."""
import numpy as np
import pytest
import torch

from automl_b200 import efficientdet_arch
from automl_b200 import hparams_config
from automl_b200 import ops
from automl_b200.efficientdet_keras import EfficientDetModel

SIZE = 128


class DeviceWork(Exception):
  pass


@pytest.fixture(autouse=True)
def no_device(monkeypatch):
  def stub(*args, **kwargs):
    raise DeviceWork()
  monkeypatch.setattr(efficientdet_arch, 'get_engine', stub)
  monkeypatch.setattr(ops, 'preprocess', stub)
  monkeypatch.setattr(ops, 'preprocess_float', stub)
  monkeypatch.setattr(torch.Tensor, 'to', stub)


def _model(**over):
  c = hparams_config.get_efficientdet_config('efficientdet-d0')
  c.override(dict(image_size=SIZE, **over))
  return EfficientDetModel(config=c)


def _u8(shape=(2, 48, 64, 3)):
  return np.zeros(shape, np.uint8)


@pytest.mark.parametrize('pre_mode', ['train', 'eval', 'INFER'])
def test_unknown_pre_mode(pre_mode):
  with pytest.raises(ValueError, match='preprocessing must be infer or empty'):
    _model()(_u8(), pre_mode=pre_mode)


@pytest.mark.parametrize('post_mode', ['per_class', 'combined', 'tflite'])
def test_unbuilt_post_modes(post_mode):
  with pytest.raises(NotImplementedError):
    _model()(_u8(), post_mode=post_mode)


@pytest.mark.parametrize('post_mode', ['nms', 'Global', 'per-class'])
def test_unknown_post_mode(post_mode):
  with pytest.raises(ValueError, match='Unsupported postprocess mode'):
    _model()(_u8(), post_mode=post_mode)


def test_post_mode_is_read_only_with_the_detection_head():
  """Like the reference (:997-1001): without 'object_detection' the post mode is never used."""
  m = _model(heads=['segmentation'])
  with pytest.raises(DeviceWork):
    m(_u8(), post_mode='per_class')


def test_training():
  with pytest.raises(NotImplementedError):
    _model()(_u8(), training=True)


@pytest.mark.parametrize('dtype', [np.float64, np.float16, np.int32, np.uint16, np.int8, np.bool_])
def test_wrong_dtype(dtype):
  m = _model()
  with pytest.raises(ValueError, match='uint8 or float32'):
    m(np.zeros((1, 48, 64, 3), dtype))
  with pytest.raises(ValueError, match='uint8 or float32'):
    m(torch.from_numpy(np.zeros((1, 48, 64, 3), dtype)))


@pytest.mark.parametrize('shape', [(48, 64, 3), (1, 1, 48, 64, 3), (64, 3), (1, 48, 64, 1),
                                   (1, 48, 64, 4), (1, 3, 48, 64), (0, 48, 64, 3), (1, 0, 64, 3)])
def test_wrong_shape(shape):
  m = _model()
  for dtype, tdtype in ((np.uint8, torch.uint8), (np.float32, torch.float32)):
    with pytest.raises(ValueError, match='channels-last'):
      m(np.zeros(shape, dtype))
    with pytest.raises(ValueError, match='channels-last'):
      m(torch.zeros(shape, dtype=tdtype))


def test_image_that_collapses():
  """1 x 1000 into 128 x 128 scales to 0 rows: edet_preprocess would refuse it on the device."""
  with pytest.raises(ValueError, match='collapses'):
    _model()(_u8((1, 1, 1000, 3)))


def test_pre_mode_none_takes_the_float_network_input():
  m = _model()
  with pytest.raises(ValueError, match='pre_mode=None'):
    m(_u8((1, SIZE, SIZE, 3)), pre_mode=None)
  with pytest.raises(ValueError, match='pre_mode=None'):
    m(np.zeros((1, SIZE, SIZE + 1, 3), np.float32), pre_mode=None)
  with pytest.raises(DeviceWork):       # the right input reaches the device
    m(np.zeros((1, SIZE, SIZE, 3), np.float32), pre_mode=None)


@pytest.mark.parametrize('dtype', [np.uint8, np.float32])
def test_valid_inputs_reach_the_device(dtype):
  """The stub is what stops a valid call: any size for pre_mode='infer', both post modes."""
  m = _model()
  for post_mode in ('global', None):
    with pytest.raises(DeviceWork):
      m(np.zeros((3, 37, 211, 3), dtype), post_mode=post_mode)
