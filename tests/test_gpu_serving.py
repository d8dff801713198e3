"""ServingDriver call surface (reference inference.py:340-554) and the device pre-process."""
import numpy as np
import pytest
import torch

from oracle import postprocess_oracle as po

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('hw,size', [((96, 128), 128), ((200, 150), (128, 160)), ((64, 64), 64)])
def test_preprocess_matches_oracle(hw, size):
  from automl_b200 import ops, utils
  rng = np.random.default_rng(hw[0])
  imgs = rng.integers(0, 256, size=(2,) + hw + (3,), dtype=np.uint8)
  mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
  oh, ow = utils.parse_image_size(size)
  out = torch.empty(2, oh, ow, 3, device='cuda:0')
  scale = ops.preprocess(torch.from_numpy(imgs).cuda(), out, mean, std)
  torch.cuda.synchronize()
  for i in range(2):
    ref, ref_scale = po.image_preprocess(imgs[i], size, mean, std)
    np.testing.assert_allclose(out[i].cpu().numpy(), ref, rtol=1e-5, atol=2e-6)
    assert abs(scale - ref_scale) <= 1e-6 * ref_scale


def test_serving_driver_call_surface():
  from automl_b200 import inference
  rng = np.random.default_rng(0)
  imgs = [rng.integers(0, 256, size=(96, 128, 3), dtype=np.uint8) for _ in range(2)]
  driver = inference.ServingDriver('efficientdet-d0', '_', batch_size=2,
                                   model_params={'image_size': 128})
  assert driver.params['is_training_bn'] is False and driver.params['image_size'] == 128
  pred = driver.serve_images(imgs)            # lazily builds, like the reference
  assert sorted(driver.signitures) == ['image_arrays', 'image_files', 'prediction']
  assert pred.shape == (2, 100, 7) and pred.dtype == np.float32
  np.testing.assert_array_equal(pred[:, :, 0], [[0.0] * 100, [1.0] * 100])
  assert ((pred[:, :, 6] >= 1) & (pred[:, :, 6] <= 90)).all()      # 1-based classes
  assert (np.diff(pred[:, :, 5], axis=1) <= 0).all()               # scores sorted per image
  # boxes are clipped to the network input and scaled back to the original image
  scale = 1.0 / min(128 / 96, 128 / 128)
  assert pred[:, :, 1:5].min() >= 0 and pred[:, :, 1:5].max() <= 128 * scale + 1e-3
  # the engine input is the oracle's pre-process of the raw image
  ref, _ = po.image_preprocess(imgs[1], 128, driver.params['mean_rgb'], driver.params['stddev_rgb'])
  np.testing.assert_allclose(driver.engine.input[1].cpu().numpy(), ref, rtol=1e-5, atol=2e-6)
  again = driver.serve_images(imgs)
  np.testing.assert_array_equal(pred, again)                       # deterministic
  with pytest.raises(ValueError):
    driver.serve_images(imgs[:1])
  with pytest.raises(NotImplementedError):
    driver.export('/tmp/x')
  with pytest.raises(ValueError):
    inference.ServingDriver('resnet50', '_')


def test_generate_detections_per_class_path():
  """postprocess.generate_detections (the reference's nms_configs.pyfunc branch) on an engine:
  equals the oracle's per_class_nms on the engine's own pre-NMS output wherever the candidate
  scores are distinct (NumPy leaves the order of equal scores undefined)."""
  from automl_b200 import hparams_config, postprocess, weights
  from automl_b200.arch import DetArch
  from automl_b200.engine import Engine
  c = hparams_config.get_efficientdet_config('efficientdet-d0')
  c.override(dict(image_size=128))
  c.nms_configs.method = 'hard'
  c.nms_configs.pyfunc = True
  eng = Engine(c, weights.synthetic_weights(DetArch(c), 3), 2)
  x = np.random.default_rng(5).uniform(-2, 2, size=(2, 128, 128, 3)).astype(np.float32)
  eng.forward(torch.from_numpy(x))
  params = c.as_dict()
  scales, ids = np.asarray([1.25, 2.0], np.float32), np.asarray([7, 8], np.float32)
  det = postprocess.generate_detections(params, eng, scales, ids).cpu().numpy()
  torch.cuda.synchronize()
  assert det.shape == (2, 100, 7)
  ps = eng.pre_nms_only()
  boxes, scores, classes = (ps[k].cpu().numpy() for k in ('boxes', 'scores', 'classes'))
  K = scores.shape[1]
  for i in range(2):
    assert (np.diff(det[i][:, 5]) <= 0).all()
    assert set(np.unique(det[i][:, 0])) == {ids[i]}
  # The engine's fp16 logits produce tied scores, whose order NumPy's argsort leaves undefined.
  # Bit-exact check on the engine's boxes / classes with the scores replaced by distinct values
  # of the same ranking (score descending, higher anchor index first = the device's tie rule).
  ranked = np.empty_like(scores)
  for i in range(2):
    order = np.lexsort((np.arange(K), scores[i]))[::-1]
    ranked[i, order] = (1.0 - np.arange(K) / K).astype(np.float32)
  assert all(len(np.unique(ranked[i])) == K for i in range(2))
  got, _, _ = postprocess.per_class_nms(ps['boxes'], torch.from_numpy(ranked).cuda(), ps['classes'],
                                        ids, scales, params['num_classes'], 100, params['nms_configs'])
  got = got.cpu().numpy()
  for i in range(2):
    ref = po.per_class_nms(boxes[i], ranked[i], classes[i], ids[i:i + 1], scales[i:i + 1],
                           params['num_classes'], 100, params['nms_configs'])
    np.testing.assert_array_equal(got[i], ref)
    # same keep decisions on the real scores: same boxes and classes row by row
    np.testing.assert_array_equal(det[i][:, [1, 2, 3, 4, 6]], ref[:, [1, 2, 3, 4, 6]])
  # flip mirrors x about the original image width (postprocess.py:558-571)
  flipped = postprocess.generate_detections(params, eng, scales, ids, flip=True).cpu().numpy()
  ow = scales * 128
  np.testing.assert_array_equal(flipped[..., 1], ow[:, None] - det[..., 3])
  np.testing.assert_array_equal(flipped[..., 3], ow[:, None] - det[..., 1])
  t = postprocess.transform_detections(torch.from_numpy(det)).numpy()
  np.testing.assert_array_equal(t[..., 3], det[..., 3] - det[..., 1])


def test_pipelined_submit_equals_synchronous_serving():
  """submit()/result() keeps up to three requests in flight (H2D + pre-process of request i+1, the
  head stage / NMS + D2H of request i-1 overlap the backbone of request i): results must equal the synchronous
  serve_images() of the same batches, in order, also when slots are reused."""
  from automl_b200 import inference
  rng = np.random.default_rng(2)
  batches = [[rng.integers(0, 256, size=(96, 128, 3), dtype=np.uint8) for _ in range(2)] for _ in range(5)]
  driver = inference.ServingDriver('efficientdet-d0', '_', batch_size=2,
                                   model_params={'image_size': 128})
  expect = [driver.serve_images(b) for b in batches]
  handles = []
  got = []
  for b in batches:                     # never more than two un-collected handles
    handles.append(driver.submit(b))
    if len(handles) == 2:
      got.append(handles.pop(0).result())
  got.append(handles.pop(0).result())
  for g, e in zip(got, expect):
    np.testing.assert_array_equal(g, e)
  # a submit beyond MAX_IN_FLIGHT completes the oldest request by itself; any collection order
  assert driver.MAX_IN_FLIGHT == 3
  h = [driver.submit(b) for b in batches[:4]]
  np.testing.assert_array_equal(h[0].result(), expect[0])
  np.testing.assert_array_equal(h[3].result(), expect[3])
  np.testing.assert_array_equal(h[1].result(), expect[1])
  np.testing.assert_array_equal(h[2].result(), expect[2])
  assert [r.shape for r in driver.serve_stream(batches)] == [(2, 100, 7)] * 5
  for g, e in zip(driver.serve_stream(iter(batches)), expect):
    np.testing.assert_array_equal(g, e)
  # pinned uint8 tensors are uploaded without the host staging copy
  pinned = torch.from_numpy(np.stack(batches[3])).pin_memory()
  np.testing.assert_array_equal(driver.serve_images(pinned), expect[3])
  # CUDA uint8 tensors are read in place on the current stream
  np.testing.assert_array_equal(driver.serve_images(pinned.to('cuda:0')), expect[3])


def test_dynamic_batch_and_channels_first():
  """batch_size=None (reference inference.py:68-109): any number of images per request; and a
  channels_first config through the driver (inference.py:456-457) gives the same detections."""
  from automl_b200 import inference
  rng = np.random.default_rng(4)
  imgs = [rng.integers(0, 256, size=(80, 100, 3), dtype=np.uint8) for _ in range(3)]
  fixed = inference.ServingDriver('efficientdet-d0', '_', batch_size=3, model_params={'image_size': 128})
  ref = fixed.serve_images(imgs)
  dyn = inference.ServingDriver('efficientdet-d0', '_', batch_size=None, model_params={'image_size': 128})
  np.testing.assert_array_equal(dyn.serve_images(imgs), ref)
  one = dyn.serve_images(imgs[1:2])
  assert one.shape == (1, 100, 7)
  np.testing.assert_array_equal(one[0, :, 1:], ref[1, :, 1:])     # same image, image id 0 instead of 1
  cf = inference.ServingDriver('efficientdet-d0', '_', batch_size=3,
                               model_params={'image_size': 128, 'data_format': 'channels_first'})
  np.testing.assert_array_equal(cf.serve_images(imgs), ref)
  # ragged request: images of different sizes are pre-processed one by one
  ragged = [imgs[0], rng.integers(0, 256, size=(60, 90, 3), dtype=np.uint8), imgs[2]]
  out = dyn.serve_images(ragged)
  np.testing.assert_array_equal(out[0], ref[0])
  np.testing.assert_array_equal(out[2], ref[2])
