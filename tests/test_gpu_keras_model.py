"""EfficientDetModel (tf2/efficientdet_keras.py:918-1003) and the float32 pre-process under it.

The kernel: edet_preprocess_float against the oracle's image_preprocess on float images, bit for bit
(as the uint8 kernel is checked), against edet_preprocess on integral images, and on an output past
2^31 elements.  The model, D0 at 128 px: post_mode='global' against the oracle's postprocess_global
and against ServingDriver, pre_mode=None, both heads, channels_first, batch sizes, ownership of the
results and stream order of a device input."""
import numpy as np
import pytest
import torch

from automl_b200 import hparams_config
from automl_b200._lib import EdetError
from oracle import postprocess_oracle as po
from test_gpu_memory_bound_kernels import Buf
from test_gpu_persistent_kernels import DEV, SENTINEL

pytestmark = pytest.mark.gpu

PREP_MEAN, PREP_STD = [100.5, 120.25, 90.75], [50.0, 60.5, 70.125]
SIZE = 128


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _float_images(n, hw, seed):
  """Fractional values, negative ones and ones above 255."""
  rng = np.random.default_rng(seed)
  return (rng.normal(120.0, 150.0, size=(n,) + tuple(hw) + (3,)) + 0.37).astype(np.float32)


def _scaled_hw(src, size):
  (h, w), (oh, ow) = src, size
  s = min(np.float32(oh) / np.float32(h), np.float32(ow) / np.float32(w))
  return int(np.float32(h) * s), int(np.float32(w) * s)


def _run_float(imgs, size, mean=PREP_MEAN, std=PREP_STD):
  """edet_preprocess_float of `imgs` into a sentinel-guarded output, read past the input's end as
  NaN: (output, scale)."""
  raw = Buf(torch.from_numpy(imgs), float('nan'))
  out = Buf(torch.full((len(imgs),) + tuple(size) + (3,), SENTINEL), SENTINEL)
  scale = _ops().preprocess_float(raw.t, out.t, mean, std)
  return out.result().numpy(), scale


# ---------------------------------------------------------------------------------------------
# edet_preprocess_float
@pytest.mark.parametrize('src', [(480, 640), (37, 53), (1, 1), (301, 97), (128, 128)],
                         ids=lambda s: 'src%dx%d' % s)
@pytest.mark.parametrize('size', [(128, 128), (127, 129), (384, 640)], ids=lambda s: '%dx%d' % s)
def test_preprocess_float_matches_oracle(size, src):
  """Down- and up-scaled, odd and non-square sources and a 1 x 1 image: the oracle's float32
  operations in its order, zero padding included, and nothing written past the output."""
  imgs = _float_images(3, src, size[0] * 31 + src[0])
  got, scale = _run_float(imgs, size)
  sh, sw = _scaled_hw(src, size)
  for i in range(len(imgs)):
    ref, ref_scale = po.image_preprocess(imgs[i], size, PREP_MEAN, PREP_STD)
    np.testing.assert_array_equal(got[i], ref, err_msg='image %d' % i)
    assert np.float32(scale) == ref_scale
    assert not got[i, sh:].any() and not got[i, :, sw:].any(), 'padding is not zero'


def test_preprocess_float_passes_nan_and_inf():
  """NaN and +-Inf are not filtered: they reach the outputs they are interpolated into, as in the
  oracle."""
  imgs = _float_images(2, (40, 50), 7)
  imgs[0, 3, 4, 0] = np.nan
  imgs[0, 20, 30, 1] = np.inf
  imgs[1, 10, 10, 2] = -np.inf
  got, _ = _run_float(imgs, (64, 96))
  for i in range(2):
    ref, _ = po.image_preprocess(imgs[i], (64, 96), PREP_MEAN, PREP_STD)
    np.testing.assert_array_equal(got[i], ref)
  assert np.isnan(got[0, ..., 0]).any() and not np.isfinite(got[0, ..., 1]).all()
  assert not np.isfinite(got[1, ..., 2]).all()


@pytest.mark.parametrize('mean,std', [(PREP_MEAN, PREP_STD),
                                      ([0.485 * 255, 0.456 * 255, 0.406 * 255],
                                       [0.229 * 255, 0.224 * 255, 0.225 * 255]),
                                      ([127.0] * 3, [128.0] * 3)], ids=['odd', 'imagenet', 'lite'])
@pytest.mark.parametrize('src,size', [((480, 640), (128, 128)), ((37, 53), (127, 129)),
                                      ((1, 1), (64, 64))], ids=['down', 'up', '1x1'])
def test_preprocess_float_equals_uint8_kernel(src, size, mean, std):
  """A float image holding integral values 0..255 gives edet_preprocess's bits on the uint8 image:
  each tap is normalised with the operations the uint8 kernel's table is built with."""
  ops = _ops()
  rng = np.random.default_rng(src[0] + size[1])
  u8 = rng.integers(0, 256, size=(3,) + src + (3,), dtype=np.uint8)
  u8[0, 0, 0] = [0, 255, 128]
  got, scale = _run_float(u8.astype(np.float32), size, mean, std)
  want = torch.empty((3,) + size + (3,), device=DEV)
  want_scale = ops.preprocess(torch.from_numpy(u8).to(DEV), want, mean, std)
  assert np.array_equal(got.view(np.int32), want.cpu().numpy().view(np.int32))
  assert scale == want_scale


def test_preprocess_float_refusals():
  """Wrong dtype, shape, layout or device raise ValueError, an image that collapses to zero rows
  EdetError; the output is untouched."""
  ops = _ops()
  out = Buf(torch.full((2, 64, 64, 3), SENTINEL), SENTINEL)
  good = torch.rand(2, 40, 50, 3, device=DEV)
  bad = {
      'uint8': good.to(torch.uint8),
      'float64': good.double(),
      'four channels': torch.rand(2, 40, 50, 4, device=DEV),
      'rank 3': good[0],
      'batch differs': good[:1],
      'strided': good.transpose(1, 2),
      'host': good.cpu(),
  }
  for what, t in bad.items():
    with pytest.raises(ValueError):
      ops.preprocess_float(t, out.t, PREP_MEAN, PREP_STD)
    assert bool((out.t == SENTINEL).all()), what
  with pytest.raises(ValueError):
    ops.preprocess_float(good, out.t[..., :2].contiguous(), PREP_MEAN, PREP_STD)
  with pytest.raises(EdetError):
    ops.preprocess_float(torch.rand(2, 1, 1000, 3, device=DEV), out.t, PREP_MEAN, PREP_STD)
  assert bool((out.result() == SENTINEL).all())


def test_preprocess_float_past_2_31_elements():
  """One launch over 305 float32 images of 1200 x 2000 into D7x's 1536 x 1536 input: the output
  passes element 2^31 at image 303 and the input at image 298.  The harness and bar of
  test_gpu_large_tensors: every image equals its source run alone, bit for bit, the canaries after
  the output hold, and two sources alone equal the oracle bit for bit."""
  import test_gpu_large_tensors as lt
  ops = _ops()
  size = lt.case_table()['preprocess'].layer['size']
  src = (1200, 2000)
  per_in, per_out = src[0] * src[1] * 3, size * size * 3
  n = lt._batch(per_out)
  case = lt.Case('preprocess_float', dict(size=size, src=src), 'out', per_out, n,
                 lt._need(n, 4 * per_out, 4 * per_in), (('in', per_in, lt.B31),))
  assert lt.extra_images(case) == [298] and lt.boundary_image(case) == 303 and n == 305
  lt.gate(case)
  g = torch.Generator(device=DEV).manual_seed(102)
  imgs = torch.randn((lt.SOURCES,) + src + (3,), generator=g, device=DEV) * 150.0 + 120.0

  def launch(ins, outs):
    ops.preprocess_float(ins[0], outs[0], PREP_MEAN, PREP_STD)

  try:
    got, = lt.run_case(case, [imgs], [((size, size, 3), torch.float32, None)], launch)
    for s in (4, 5):
      ref, _ = po.image_preprocess(imgs[s].cpu().numpy(), size, PREP_MEAN, PREP_STD)
      np.testing.assert_array_equal(got[s].cpu().numpy(), ref, err_msg='source %d' % s)
  finally:
    del imgs
    lt.free_all()


# ---------------------------------------------------------------------------------------------
# EfficientDetModel
def _config(**over):
  c = hparams_config.get_efficientdet_config('efficientdet-d0')
  c.override(dict(image_size=SIZE, **over))
  return c


def _model(config, **kw):
  from automl_b200.efficientdet_keras import EfficientDetModel
  return EfficientDetModel(config=config, **kw)


def _u8(n, hw, seed):
  return np.random.default_rng(seed).integers(0, 256, size=(n,) + tuple(hw) + (3,), dtype=np.uint8)


def _engine(config, n, weights=None):
  """The cached engine the model ran on."""
  from automl_b200 import efficientdet_arch
  return efficientdet_arch.get_engine(config, n, weights=weights, device=DEV)


def _np(outputs):
  return [t.cpu().numpy() for t in outputs]


def _nms_half(params, pre, scales):
  """The oracle's postprocess_global with its pre_nms replaced by the given (boxes, scores,
  classes): its NMS-V5, gather, clip and scaling on those tensors."""
  saved = po.pre_nms
  po.pre_nms = lambda *args, **kwargs: pre
  try:
    return po.postprocess_global(params, [None], [None], scales)
  finally:
    po.pre_nms = saved


def _pre_nms(config, n):
  """Host copies of the (boxes, scores, classes) pre-NMS tensors of the model's latest pass."""
  ps = _engine(config, n).pre_nms_only()
  return tuple(ps[k].cpu().numpy() for k in ('boxes', 'scores', 'classes'))


def _check_global(config, got, pre, cls_l, box_l, scales):
  """`got` (the model's four outputs) against the oracle's postprocess_global: bit for bit on `pre`,
  the engine's own pre-NMS tensors of the same pass, padded rows included; from the model's logits
  through the oracle's pre_nms, at the bar of test_gpu_network (the oracle's sigmoid and box decode
  differ from the device's in the last bits)."""
  params = config.as_dict()
  m = params['nms_configs']['max_output_size']
  boxes, scores, classes, valid = _np(got)
  n = len(valid)
  assert boxes.shape == (n, m, 4) and scores.shape == classes.shape == (n, m)
  assert boxes.dtype == scores.dtype == classes.dtype == np.float32 and valid.dtype == np.int32
  ref = _nms_half(params, pre, scales)
  for name, a, b in zip(('boxes', 'scores', 'classes', 'valid_len'), (boxes, scores, classes, valid), ref):
    np.testing.assert_array_equal(a, b, err_msg=name)
  for i in range(n):        # rows past valid_len: anchor 0's box and class, score 0
    v = valid[i]
    b0 = po.clip_boxes(pre[0][i, :1], params['image_size']) * (1 if scales is None else scales[i])
    assert not scores[i, v:].any()
    assert (boxes[i, v:] == b0).all() and (classes[i, v:] == pre[2][i, 0] + 1).all()
  full = po.postprocess_global(params, [t.cpu().numpy() for t in cls_l],
                               [t.cpu().numpy() for t in box_l], scales)
  np.testing.assert_array_equal(valid, full[3])
  np.testing.assert_array_equal(classes, full[2])
  np.testing.assert_allclose(scores, full[1], rtol=1e-6, atol=1e-7)
  top = 1.0 if scales is None else float(np.max(scales))
  np.testing.assert_allclose(boxes, full[0], rtol=1e-5, atol=1e-3 * top)


def _padding_config(x):
  """A hard-NMS config whose score threshold leaves fewer than max_output_size detections in the
  first image, taken from that image's pre-NMS scores on the default config: at most 40 anchors
  (but at least the top score's) score above it, and it lies midway between two distinct scores,
  so that the oracle's sigmoid, which may differ from the device's in the last bit, puts the same
  anchors above it.  Many anchors share a score (fp16 logits)."""
  c = _config()
  _model(c)(x)
  scores = _pre_nms(c, len(x))[1][0]
  distinct = np.unique(scores)
  k = 1
  while k + 1 < len(distinct) and (scores >= distinct[-k - 1]).sum() <= 40:
    k += 1
  c = _config()
  c.nms_configs.method = 'hard'
  c.nms_configs.score_thresh = float((distinct[-k] + distinct[-k - 1]) / 2)
  return c


SOURCES = {'uint8': ((96, 160), 1.25), 'float32': ((200, 150), 1.5625)}   # size, scale back


def _source(dtype, n, seed):
  hw = SOURCES[dtype][0]
  return _u8(n, hw, seed) if dtype == 'uint8' else _float_images(n, hw, seed)


@pytest.mark.parametrize('nms', ['default', 'thresholded'])
@pytest.mark.parametrize('dtype', ['uint8', 'float32'])
def test_global_matches_oracle(dtype, nms):
  """pre_mode='infer': the four outputs of post_mode='global' are the oracle's postprocess_global of
  the model's own pass and scales; 'thresholded' leaves padded rows."""
  x = _source(dtype, 2, 1)
  c = _padding_config(x) if nms == 'thresholded' else _config()
  model = _model(c)
  got = model(x)
  pre = _pre_nms(c, 2)
  cls_l, box_l = model(x, post_mode=None)
  scales = np.full(2, SOURCES[dtype][1], np.float32)
  for i in range(2):
    assert po.image_preprocess(x[i], SIZE, c.mean_rgb, c.stddev_rgb)[1] == scales[i]
  _check_global(c, got, pre, cls_l, box_l, scales)
  if nms == 'thresholded':
    assert int(got[3][0]) < c.nms_configs.max_output_size, 'no padded rows'


def test_matches_serving_driver():
  """uint8 images: the same detections as ServingDriver.serve_images, column for column."""
  from automl_b200 import inference
  x = _source('uint8', 2, 2)
  driver = inference.ServingDriver('efficientdet-d0', '_', batch_size=2,
                                   model_params={'image_size': SIZE})
  want = driver.serve_images(list(x))
  boxes, scores, classes, _ = _np(_model(_config())(x))
  np.testing.assert_array_equal(boxes, want[..., 1:5])
  np.testing.assert_array_equal(scores, want[..., 5])
  np.testing.assert_array_equal(classes, want[..., 6])


def test_pre_mode_none():
  """The float32 network input: EfficientDetNet's logits, and boxes that are not scaled."""
  from automl_b200.efficientdet_keras import EfficientDetNet
  c = _config()
  x = np.random.default_rng(3).uniform(-2, 2, size=(2, SIZE, SIZE, 3)).astype(np.float32)
  model = _model(c)
  got = model(torch.from_numpy(x).to(DEV), pre_mode=None)
  pre = _pre_nms(c, 2)
  cls_l, box_l = model(x, pre_mode=None, post_mode=None)
  net_cls, net_box = EfficientDetNet(config=c)(x)
  for a, b in zip(cls_l + box_l, net_cls + net_box):
    assert torch.equal(a, b)
  _check_global(c, got, pre, cls_l, box_l, None)
  assert float(got[0].max()) <= SIZE


def test_both_heads():
  """'object_detection' and 'segmentation': five outputs from one pass, the segmentation logits
  EfficientDetNet's on the pre-processed input."""
  from automl_b200.efficientdet_keras import EfficientDetNet
  c = _config(heads=['object_detection', 'segmentation'])
  x = _source('uint8', 2, 4)
  got = _model(c)(x)
  assert len(got) == 5
  pre = _pre_nms(c, 2)
  inp = torch.empty(2, SIZE, SIZE, 3, device=DEV)
  _ops().preprocess(torch.from_numpy(x).to(DEV), inp, c.mean_rgb, c.stddev_rgb)
  net = EfficientDetNet(config=c)(inp)
  assert len(net) == 3 and torch.equal(got[4], net[2])
  assert got[4].shape == (2, SIZE // 4, SIZE // 4, c.seg_num_classes)
  _check_global(c, got[:4], pre, net[0], net[1], np.full(2, 1.25, np.float32))
  seg_only = _model(_config(heads=['segmentation']))(x)
  assert len(seg_only) == 1 and seg_only[0].shape == got[4].shape


def test_channels_first():
  """channels_first takes the same NHWC images and gives the same detections; its logits are the
  NCHW transposes."""
  x = _source('float32', 2, 5)
  last = _model(_config())
  first = _model(_config(data_format='channels_first'))
  for a, b in zip(first(x), last(x)):
    assert torch.equal(a, b)
  for la, fa in zip(last(x, post_mode=None), first(x, post_mode=None)):
    for lv, fv in zip(la, fa):
      assert torch.equal(fv, lv.permute(0, 3, 1, 2))


@pytest.mark.parametrize('dtype', ['uint8', 'float32'])
def test_batch_sizes(dtype):
  """Batches of 1 and 3 through one model: each image's detections equal its call alone."""
  x = _source(dtype, 3, 6)
  model = _model(_config())
  alone = [_np(model(x[i:i + 1])) for i in range(3)]
  batch = _np(model(x))
  for i in range(3):
    for a, b in zip(batch, alone[i]):
      np.testing.assert_array_equal(a[i], b[0])
  again = _np(model(x[1:2]))
  for a, b in zip(again, alone[1]):
    np.testing.assert_array_equal(a, b)


def test_results_are_owned():
  """A later call, of either post mode and with other images, leaves earlier results unchanged."""
  c = _config(heads=['object_detection', 'segmentation'])
  model = _model(c)
  x, y = _source('uint8', 2, 7), _source('uint8', 2, 8)
  first = model(x)
  kept = [t.clone() for t in first]
  logits = model(x, post_mode=None)
  kept_logits = [t.clone() for t in logits[0] + logits[1]]
  second = model(y)
  model(y, post_mode=None)
  assert not torch.equal(second[1], kept[1]), 'the two requests give the same scores'
  for a, b in zip(first, kept):
    assert torch.equal(a, b)
  for a, b in zip(logits[0] + logits[1], kept_logits):
    assert torch.equal(a, b)


@pytest.mark.parametrize('dtype', ['uint8', 'float32'])
def test_device_input_is_read_after_its_write(dtype):
  """A device input written on the current (side) stream right before the call, behind a stall,
  is read after the write: the result is that of the written images, not of what the buffer held."""
  model = _model(_config())
  x, y = _source(dtype, 2, 9), _source(dtype, 2, 10)
  want = _np(model(x))
  src = torch.from_numpy(x).to(DEV)
  buf = torch.from_numpy(y).to(DEV)
  torch.cuda.synchronize()
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    torch.cuda._sleep(1 << 24)
    buf.copy_(src)
    got = model(buf)
    got = _np(got)               # .cpu() on the side stream: the results are ready there
  for a, b in zip(got, want):
    np.testing.assert_array_equal(a, b)
