"""The ragged serving pre-process (edet_preprocess_ragged) and ServingDriver requests whose images
differ in size.

Kernel: every image of a ragged launch equals edet_preprocess of that image alone, bit for bit,
with the same image_scale_to_original; the padding is zero and nothing past `out` is written.
Driver: a ragged request is one staged H2D and one launch; its detections equal each image served
alone, also with several requests in flight while the staging buffers grow, mixed with uniform
requests, and with batch_size=None.  The PDL chains of test_gpu_pdl_chains.py check that the launch
reads only what the copy ahead of it wrote and writes only `out`."""
import numpy as np
import pytest
import torch

import test_gpu_pdl_chains as pdl

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
GUARD = 1024
SENTINEL = 7.0


def _image(rng, h, w):
  return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def _pack(images, image_size):
  """(packed uint8 device buffer, desc int32 device table, host desc, host scales)."""
  from automl_b200 import inference
  desc, total, scales = inference.preprocess_table([im.shape[:2] for im in images], image_size)
  packed = np.zeros(total, np.uint8)
  for im, off in zip(images, desc[:, :2].copy().view(np.int64)[:, 0]):
    packed[off:off + im.size] = im.reshape(-1)
  return torch.from_numpy(packed).to(DEV), torch.from_numpy(desc).to(DEV), desc, scales


def _ragged(images, image_size):
  """One ragged launch into an output followed by GUARD sentinels: (out, host desc, scales)."""
  from automl_b200 import ops, utils
  oh, ow = utils.parse_image_size(image_size)
  n = len(images)
  packed, desc_dev, desc, scales = _pack(images, image_size)
  mem = torch.full((n * oh * ow * 3 + GUARD,), SENTINEL, device=DEV)
  out = mem[:n * oh * ow * 3].view(n, oh, ow, 3)
  ops.preprocess_ragged(packed, desc_dev, out, MEAN, STD)
  torch.cuda.synchronize()
  assert bool((mem[n * oh * ow * 3:] == SENTINEL).all()), 'written past the end of out'
  return out, desc, scales


def _alone(image, image_size):
  from automl_b200 import ops, utils
  oh, ow = utils.parse_image_size(image_size)
  out = torch.full((1, oh, ow, 3), SENTINEL, device=DEV)
  scale = ops.preprocess(torch.from_numpy(np.ascontiguousarray(image[None])).to(DEV), out, MEAN, STD)
  return out[0], scale


def _sizes(case, oh, ow):
  rng = np.random.default_rng(11)
  if case == 'mixed':       # landscape, portrait, square; up- and downscale; odd sizes
    return [(480, 640), (640, 480), (333, 333), (37, 53), (1001, 777), (64, 64), (127, 255)]
  if case == 'thin':        # a 1-pixel row and column; aspects where one scaled side is 1
    return [(1, 50), (50, 1), (1, 1), (1, ow), (oh, 1), (3, 2 * ow), (2 * oh, 3)]
  if case == 'one':
    return [(123, 77)]
  if case == 'many':        # n = 128, many distinct sizes
    return [tuple(int(v) for v in rng.integers(40, 700, size=2)) for _ in range(128)]
  raise ValueError(case)


@pytest.mark.parametrize('case,image_size', [('mixed', 128), ('mixed', '640x384'), ('thin', 64),
                                             ('thin', '640x384'), ('one', 128), ('many', 256)])
def test_ragged_equals_each_image_alone(case, image_size):
  from automl_b200 import utils
  oh, ow = utils.parse_image_size(image_size)
  rng = np.random.default_rng(len(case))
  images = [_image(rng, h, w) for h, w in _sizes(case, oh, ow)]
  out, desc, scales = _ragged(images, image_size)
  if case == 'thin':
    assert 1 in desc[:, 4] and 1 in desc[:, 5]
  for i, im in enumerate(images):
    want, scale = _alone(im, image_size)
    assert torch.equal(out[i], want), (case, im.shape)
    assert scales[i] == np.float32(scale), (im.shape, scales[i], scale)
    sh, sw = int(desc[i, 4]), int(desc[i, 5])
    assert 1 <= sh <= oh and 1 <= sw <= ow
    assert not bool(out[i, sh:].any()) and not bool(out[i, :, sw:].any()), 'padding is not zero'
    assert bool(torch.isfinite(out[i, :sh, :sw]).all())


def test_ragged_of_one_size_equals_the_uniform_launch():
  from automl_b200 import ops
  rng = np.random.default_rng(3)
  images = [_image(rng, 375, 500) for _ in range(6)]
  out, _, scales = _ragged(images, '640x384')
  want = torch.empty(6, 384, 640, 3, device=DEV)
  scale = ops.preprocess(torch.from_numpy(np.stack(images)).to(DEV), want, MEAN, STD)
  torch.cuda.synchronize()
  assert torch.equal(out, want)
  assert (scales == np.float32(scale)).all()


# ---------------------------------------------------------------------------------------------
# the driver
def _driver(batch_size):
  from automl_b200 import inference
  return inference.ServingDriver('efficientdet-d0', '_', batch_size=batch_size,
                                 model_params={'image_size': 128})


@pytest.fixture(scope='module')
def dyn():
  return _driver(None)


def _check_rows(got, images, alone):
  """Each image's rows equal that image served alone, image id aside."""
  assert got.shape == (len(images), 100, 7)
  for i, im in enumerate(images):
    np.testing.assert_array_equal(got[i, :, 1:], alone(im)[0, :, 1:])
    assert (got[i, :, 0] == i).all()


def _alone_cache(driver):
  cache = {}

  def alone(im):
    key = (im.shape, im.tobytes())
    if key not in cache:
      cache[key] = driver.serve_images([im])
    return cache[key]
  return alone


def test_driver_ragged_rows_equal_each_image_alone(dyn):
  """batch_size=None: ragged requests of different lengths, each image as if served alone."""
  rng = np.random.default_rng(21)
  alone = _alone_cache(dyn)
  for sizes in ([(96, 128), (128, 96), (60, 90)],
                [(480, 640), (33, 200), (128, 128), (200, 33), (77, 101)],
                [(1, 64), (64, 1)]):
    images = [_image(rng, h, w) for h, w in sizes]
    _check_rows(dyn.serve_images(images), images, alone)


def test_driver_stream_of_growing_ragged_requests():
  """Seven ragged requests, each about 1.7x the bytes of the one before, through serve_stream (three
  in flight): every slot's staging buffers grow while earlier requests are queued.  Equal to serving
  each request synchronously afterwards."""
  driver = _driver(3)
  rng = np.random.default_rng(5)
  batches = []
  for k in range(7):
    side = int(60 * 1.3 ** k)
    batches.append([_image(rng, side, side + 17), _image(rng, side + 31, side), _image(rng, side // 2 + 1, side)])
  got = list(driver.serve_stream(batches))
  assert max(s.staging.dev.numel() for s in driver._slots[3]) >= sum(im.size for im in batches[-1])
  for g, b in zip(got, batches):
    np.testing.assert_array_equal(g, driver.serve_images(b))


def test_driver_stream_mixing_uniform_and_ragged_requests():
  driver = _driver(2)
  rng = np.random.default_rng(9)
  uniform = [_image(rng, 96, 128) for _ in range(2)]
  requests = [uniform,
              [_image(rng, 96, 128), _image(rng, 70, 50)],
              torch.from_numpy(np.stack(uniform)).pin_memory(),
              [_image(rng, 300, 200), _image(rng, 20, 30)],
              [_image(rng, 80, 100) for _ in range(2)],
              [_image(rng, 50, 70), _image(rng, 128, 128)]]
  got = list(driver.serve_stream(requests))
  for g, r in zip(got, requests):
    np.testing.assert_array_equal(g, driver.serve_images(r))
  np.testing.assert_array_equal(got[2], got[0])


def test_driver_rejects_invalid_images_before_enqueueing(dyn):
  rng = np.random.default_rng(13)
  good = _image(rng, 96, 128)
  bad = [rng.integers(0, 256, size=(60, 80, 3)).astype(np.float32),    # not uint8
         _image(rng, 60, 80)[:, :, :2],                                 # two channels
         rng.integers(0, 256, size=(60, 80), dtype=np.uint8),           # no channel axis
         _image(rng, 1, 2000)]                                          # collapses to 0 x 128
  alone = _alone_cache(dyn)
  for b in bad:
    with pytest.raises(ValueError):
      dyn.serve_images([good, b])
    images = [good, _image(rng, 40, 90)]
    _check_rows(dyn.serve_images(images), images, alone)


# ---------------------------------------------------------------------------------------------
# PDL chains (test_gpu_pdl_chains.py): a slow copy writes the packed images and the table, or
# reads what the launch will overwrite
def _pdl_case():
  from automl_b200 import inference
  sizes = [(200, 150), (37, 91), (128, 128)]
  desc, total, _ = inference.preprocess_table(sizes, (96, 160))

  def launch(ops, t):
    ops.preprocess_ragged(t['packed'], t['desc'], t['out'], MEAN, STD)
  # bytes below 64: every 16-bit half the identity copy moves is a finite fp16
  packed = lambda g: torch.randint(0, 64, (total,), generator=g, dtype=torch.uint8)
  return pdl.Case('preprocess_ragged',
                  [pdl.buf('packed', (total,), torch.uint8, make=packed),
                   pdl.buf('desc', desc.shape, torch.int32, make=lambda g: torch.from_numpy(desc)),
                   pdl.buf('out', (len(sizes), 96, 160, 3), torch.float32, 'out')], launch)


@pytest.fixture(scope='module')
def region():
  return pdl.Region()


def test_pdl_reads_only_what_the_copy_wrote(region):
  raw = pdl.Raw(_pdl_case(), region)
  want = pdl._raw_want(raw)
  raw.prepare()
  pdl._sleep()
  raw.chain()
  torch.cuda.synchronize()
  got = raw.result()
  for k in want:
    assert torch.equal(got[k], want[k]), '%s differs from the launch alone on NEW' % k


def test_pdl_writes_only_out_after_the_copy(region):
  war = pdl.War(_pdl_case(), region)
  try:
    war.case.run(war.t)
  finally:
    pdl._reset_all(pdl._ops())
  war.prepare()
  pdl._sleep()
  war.chain()
  war.check()
