"""Flip test-time augmentation on the GPU: edet_wbf bit for bit against the numpy oracle
(tests/wbf_oracle.py) on the reference goldens and on seeded batches, its fused un-mirror against
postprocess.generate_detections(flip=True), its programmatic-dependent-launch read of the rows,
edet_preprocess_mirrored against edet_preprocess_ragged (also past 2^31 output elements), and
ServingDriver.serve_images_tta / serve_stream_tta end to end."""
import os

import numpy as np
import pytest
import torch

import plan_settings as ps
import wbf_oracle as wo
from automl_b200 import utils

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GUARD = 64                      # sentinel rows / counts after each output
SENTINEL = np.float32(-7.5e33)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wbf.npz')
PAD = np.array([0, 0, 0, 0, 0, 0, -1], np.float32)


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _launch(blocks, num_models, num_classes, mask=0, scales=None, width=1):
  """edet_wbf on float32 blocks [num_models * n, rows, 7] into guarded outputs; checks the
  sentinels and the padding rows, returns the list of [k_i, 7] clusters."""
  ops = _ops()
  det = torch.from_numpy(np.ascontiguousarray(blocks, np.float32)).to(DEV)
  n, rows = det.shape[0] // num_models, det.shape[1]
  cap = num_models * rows
  out = torch.full((n * cap + GUARD, 7), float(SENTINEL), device=DEV)
  cnt = torch.full((n + GUARD,), -5, dtype=torch.int32, device=DEV)
  sc = None if scales is None else torch.from_numpy(np.asarray(scales, np.float32)).to(DEV)
  ops.wbf(det, num_models, num_classes, out[:n * cap].view(n, cap, 7), cnt[:n], mask, sc, width)
  host, counts = out.cpu().numpy(), cnt.cpu().numpy()
  assert (host[n * cap:] == SENTINEL).all() and (counts[n:] == -5).all(), 'written past the outputs'
  clusters = host[:n * cap].reshape(n, cap, 7)
  res = []
  for i in range(n):
    assert 0 <= counts[i] <= cap
    assert (clusters[i, counts[i]:] == PAD).all(), 'padding rows of image %d' % i
    res.append(clusters[i, :counts[i]])
  return res


def _golden():
  data = np.load(GOLDEN)
  names = sorted({k.split('/')[0] for k in data.files})
  return {n: (data[n + '/det'], data[n + '/meta'], data[n + '/scale'], data[n + '/out']) for n in names}


def test_kernel_matches_reference_goldens():
  cases = _golden()
  assert len(cases) >= 20
  for name, (det, (num_models, mask, num_classes, width), scale, want) in cases.items():
    got = _launch(det, int(num_models), int(num_classes), int(mask), [scale], int(width))[0]
    assert wo.same_bits(got, want), name


def _nms_like(rng, n, num_models, rows, num_classes, width=512.0):
  """Seeded per-class-NMS-like rows: jittered copies of a few boxes per image and model, 1-based
  classes up to num_classes (the last one is dropped by WBF), quantised scores (ties), and the
  dummy rows [id, 0, 0, 0, 0, -1e5, 0] at the end of each block."""
  out = np.zeros((num_models, n, rows, 7), np.float32)
  scales = rng.uniform(0.5, 4, n).astype(np.float32)
  for i in range(n):
    real = int(rng.integers(0, rows + 1))
    base = rng.uniform(0, width - 64, (max(real // 3, 1), 2))
    size = rng.uniform(4, 64, (len(base), 2))
    pick = rng.integers(0, len(base), real)
    cls = rng.integers(1, num_classes + 1, len(base))[pick]
    for m in range(num_models):
      b = out[m, i]
      xy = base[pick] + rng.normal(0, 2, (real, 2))
      b[:real, 0] = 100 + i
      b[:real, 1:3] = xy
      b[:real, 3:5] = xy + size[pick] + rng.normal(0, 2, (real, 2))
      b[:real, 5] = np.round(rng.uniform(0, 1, real) * 64) / 64
      b[:real, 6] = cls
      b[real:, 0] = 100 + i
      b[real:, 5] = -1e5
  return out.reshape(num_models * n, rows, 7), scales


@pytest.mark.parametrize('num_models', [1, 2, 3])
def test_kernel_random_against_oracle(num_models):
  rng = np.random.default_rng(10 + num_models)
  mask = 0b10 if num_models > 1 else 0b1
  for rows, n, check in ((7, 9, range(9)), (100, 40, range(40)),
                         (1024 // num_models, 3, range(3)), (100, 4000, (0, 1, 1999, 3998, 3999))):
    det, scales = _nms_like(rng, n, num_models, rows, 8)
    got = _launch(det, num_models, 8, mask, scales, 512)
    blocks = det.reshape(num_models, n, rows, 7)
    for i in check:
      want = wo.ensemble(wo.stack_models(list(blocks[:, i]), mask, scales[i], 512), 8, num_models)
      assert wo.same_bits(got[i], want), (rows, n, i)


def test_refuses_bad_launches():
  ops = _ops()
  from automl_b200._lib import EdetError
  det = torch.zeros(2, 513, 7, device=DEV)
  out = torch.empty(1, 1026, 7, device=DEV)
  cnt = torch.empty(1, dtype=torch.int32, device=DEV)
  with pytest.raises(EdetError, match='exceeds'):
    ops.wbf(det, 2, 8, out, cnt)
  det = torch.zeros(2, 10, 7, device=DEV)
  with pytest.raises(EdetError, match='image_scales'):
    ops.wbf(det, 2, 8, out[:, :20], cnt, mirrored_mask=2)


class _Pre(object):
  """An engine stand-in whose pre-NMS buffers postprocess.generate_detections reads."""

  def __init__(self, boxes, scores, classes):
    self.ps = {'boxes': boxes, 'scores': scores, 'classes': classes}

  def pre_nms_only(self):
    return self.ps


def test_fused_unmirror_equals_generate_detections_flip():
  from automl_b200 import hparams_config
  from automl_b200 import postprocess
  params = hparams_config.get_detection_config('efficientdet-d0').as_dict()
  params['image_size'] = 640
  rng = np.random.default_rng(3)
  n, k = 6, 2000
  yx = rng.uniform(0, 600, (n, k, 2))
  hw = rng.uniform(4, 90, (n, k, 2))
  boxes = torch.from_numpy(np.concatenate([yx, yx + hw], -1).astype(np.float32)).to(DEV)
  scores = torch.from_numpy(rng.uniform(0, 1, (n, k)).astype(np.float32)).to(DEV)
  classes = torch.from_numpy(rng.integers(0, 90, (n, k)).astype(np.int32)).to(DEV)
  scales = rng.uniform(0.5, 3, n).astype(np.float32)
  ids = np.arange(n, dtype=np.float32)
  eng = _Pre(boxes, scores, classes)
  plain = postprocess.generate_detections(params, eng, scales, ids).cpu().numpy()
  flipped = postprocess.generate_detections(params, eng, scales, ids, flip=True).cpu().numpy()
  nc = params['num_classes']
  fused = _launch(plain, 1, nc, 0b1, scales, 640)
  torch_path = _launch(flipped, 1, nc)
  for i in range(n):
    assert wo.same_bits(fused[i], torch_path[i]), i
    assert wo.same_bits(fused[i], wo.ensemble(flipped[i], nc, 1)), i


def _exact_rows(rng, count):
  """Rows whose float32 values have at most 8 significant bits, so their low fp16 half is +0 and
  the identity fp16 GEMM copies them exactly (a -0 half would come back as +0): integer boxes
  below 256, scores in 1/128 steps."""
  r = np.zeros((count, 7), np.float32)
  r[:, 0] = 3
  xy = rng.integers(0, 120, (count, 2))
  r[:, 1:3] = xy
  r[:, 3:5] = xy + rng.integers(8, 120, (count, 2))
  r[:, 5] = rng.integers(1, 128, count) / 128.0
  r[:, 6] = rng.integers(1, 4, count)
  return r


def test_reads_rows_written_by_the_previous_kernel():
  """RAW through PDL (the pattern of tests/test_gpu_pdl_chains.py): a one-CTA identity copy writes
  the detection rows, edet_wbf is launched right behind it and must see every row the copy wrote,
  though its CTAs start while the copy is still running."""
  ops = _ops()
  rows_total, t = 1 << 17, 49                  # the last 49 fp16 rows hold 2 x 112 float32 rows
  rng = np.random.default_rng(4)
  want_rows, old_rows = _exact_rows(rng, 224), _exact_rows(rng, 224)
  g = torch.Generator().manual_seed(1)
  old = (torch.randn(rows_total, 64, generator=g) * 0.5).half()
  new = (torch.randn(rows_total, 64, generator=g) * 0.5).half()
  old[old == 0] = 0.5
  new[new == 0] = 0.5
  new[-t:] = torch.from_numpy(want_rows.reshape(-1).view(np.float16).reshape(t, 64).copy())
  old[-t:] = torch.from_numpy(old_rows.reshape(-1).view(np.float16).reshape(t, 64).copy())
  region = old.to(DEV)
  src = new.to(DEV)
  eye = torch.eye(64, dtype=torch.float16, device=DEV)
  zero = torch.zeros(64, dtype=torch.float32, device=DEV)
  det = region[rows_total - t:].view(torch.float32).view(2, 112, 7)
  out = torch.full((1, 224, 7), float(SENTINEL), device=DEV)
  cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
  assert (want_rows.view(np.uint32) & 0xffff == 0).all() and (old_rows.view(np.uint32) & 0xffff == 0).all()
  want = wo.ensemble(want_rows, 4, 2)
  assert not wo.same_bits(want, wo.ensemble(old_rows, 4, 2)), 'the chain could not fail'
  ops.pointwise_conv(src[:256], eye, zero, region[:256].clone(), utils.ACT_NONE)   # warm both
  ops.wbf(det, 2, 4, out, cnt)
  torch.cuda.synchronize()
  region.copy_(old.to(DEV))
  torch.cuda.synchronize()
  torch.cuda._sleep(1 << 22)                    # the host queues the chain meanwhile
  ops.set_option('max_ctas', 1)
  try:
    ops.pointwise_conv(src, eye, zero, region, utils.ACT_NONE)
  finally:
    ps.reset(ops)
  ops.wbf(det, 2, 4, out, cnt)
  torch.cuda.synchronize()
  k = int(cnt.item())
  assert wo.same_bits(out[0, :k].cpu().numpy(), want), 'edet_wbf read rows before its wait'
  assert torch.equal(region.cpu(), new)


# ---- mirrored pre-process ------------------------------------------------------------------------
def _mirrored_and_ragged(images, size):
  from automl_b200 import inference
  ops = _ops()
  desc, total, _ = inference.preprocess_table([im.shape[:2] for im in images], size)
  packed = np.zeros(total, np.uint8)
  for im, off in zip(images, desc[:, :2].copy().view(np.int64)[:, 0]):
    packed[off:off + im.size] = im.reshape(-1)
  pk, ds = torch.from_numpy(packed).to(DEV), torch.from_numpy(desc).to(DEV)
  n = len(images)
  mir = torch.full((2 * n, size[0], size[1], 3), 9.0, device=DEV)
  rag = torch.empty(n, size[0], size[1], 3, device=DEV)
  mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
  ops.preprocess_mirrored(pk, ds, mir, mean, std)
  ops.preprocess_ragged(pk, ds, rag, mean, std)
  return mir, rag


@pytest.mark.parametrize('shapes', [[(200, 300)] * 3, [(200, 300), (512, 100), (5, 7), (640, 640)]],
                         ids=['uniform', 'ragged'])
def test_mirrored_preprocess(shapes):
  rng = np.random.default_rng(len(shapes))
  images = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
  for size in ((256, 256), (320, 192)):
    mir, rag = _mirrored_and_ragged(images, size)
    n = len(images)
    assert torch.equal(mir[:n], rag)
    assert torch.equal(mir[n:], torch.flip(rag, dims=[2]))


def test_mirrored_preprocess_past_2_31_elements():
  """D7x at 1536^2: 152 images and their mirrors, 2.15e9 output elements; the last mirror starts
  past 2^31."""
  n, size = 152, (1536, 1536)
  assert 2 * n * size[0] * size[1] * 3 > 2 ** 31
  rng = np.random.default_rng(7)
  images = [rng.integers(0, 256, (48 + i % 5, 64 - i % 3, 3), dtype=np.uint8) for i in range(n)]
  mir, _ = _mirrored_and_ragged(images[:1], size)       # warm
  del mir
  from automl_b200 import inference
  ops = _ops()
  desc, total, _ = inference.preprocess_table([im.shape[:2] for im in images], size)
  packed = np.zeros(total, np.uint8)
  for im, off in zip(images, desc[:, :2].copy().view(np.int64)[:, 0]):
    packed[off:off + im.size] = im.reshape(-1)
  pk, ds = torch.from_numpy(packed).to(DEV), torch.from_numpy(desc).to(DEV)
  mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
  out = torch.empty(2 * n, size[0], size[1], 3, device=DEV)
  ops.preprocess_mirrored(pk, ds, out, mean, std)
  for i in (0, n - 2, n - 1):
    one = torch.empty(1, size[0], size[1], 3, device=DEV)
    ops.preprocess_ragged(pk, ds[i:i + 1].contiguous(), one, mean, std)
    assert torch.equal(out[i], one[0]), i
    assert torch.equal(out[n + i], torch.flip(one[0], dims=[1])), i
  del out
  torch.cuda.empty_cache()


# ---- ServingDriver --------------------------------------------------------------------------------
def _driver(batch_size=None, heads=None, size=256):
  from automl_b200 import inference
  mp = {'image_size': size}
  if heads is not None:
    mp['heads'] = heads
  return inference.ServingDriver('efficientdet-d0', '_', batch_size=batch_size, model_params=mp)


def _rand_images(rng, shapes):
  return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes]


RAGGED = [(200, 256), (256, 180), (37, 300), (300, 300), (5, 7)]


def test_serve_images_tta_end_to_end():
  drv = _driver()
  rng = np.random.default_rng(21)
  images = _rand_images(rng, RAGGED)
  got = drv.serve_images_tta(images)
  n = len(images)
  tta = [s.tta for s in drv._slots[2 * n] if s.tta is not None][-1]  # pylint: disable=protected-access
  torch.cuda.synchronize()
  det = tta.rows.cpu().numpy()
  scales = tta.scales.cpu().numpy()
  nc = drv.config.num_classes
  assert len(got) == n
  for i in range(n):
    assert det[i, 0, 0] == i and det[n + i, 0, 0] == i and scales[i] == scales[n + i]
    want = wo.ensemble(wo.stack_models([det[i], det[n + i]], 0b10, scales[i], 256), nc, 2)
    assert got[i].dtype == np.float32 and wo.same_bits(got[i], want), i
  # the first half is the plain per-class NMS of generate_detections on the un-mirrored input
  from automl_b200 import postprocess
  eng = drv._engines[2 * n]   # pylint: disable=protected-access
  plain = postprocess.generate_detections(drv.config.as_dict(), eng, scales, np.concatenate(
      [np.arange(n), np.arange(n)]).astype(np.float32)).cpu().numpy()
  assert wo.same_bits(plain, det)


def test_request_forms_agree():
  drv = _driver()
  rng = np.random.default_rng(31)
  same = _rand_images(rng, [(120, 160)] * 3)
  ragged = same + _rand_images(rng, [(90, 250)])
  alone = [drv.serve_images_tta([im])[0] for im in ragged]
  together = drv.serve_images_tta(ragged)
  uniform = drv.serve_images_tta(same)
  pinned = drv.serve_images_tta(torch.from_numpy(np.stack(same)).pin_memory())
  on_device = drv.serve_images_tta(torch.from_numpy(np.stack(same)).to(DEV))
  for i in range(4):
    a = alone[i].copy()
    a[:, 0] = together[i][:, 0]           # image ids follow the position in the request
    assert wo.same_bits(a, together[i]), i
  for i in range(3):
    assert wo.same_bits(uniform[i], together[i]) and wo.same_bits(pinned[i], together[i]), i
    assert wo.same_bits(on_device[i], uniform[i]), i


def test_serve_stream_tta_equals_sequential():
  drv = _driver()
  rng = np.random.default_rng(41)
  reqs = [_rand_images(rng, RAGGED), _rand_images(rng, [(256, 256)] * 2),
          _rand_images(rng, RAGGED[::-1]), _rand_images(rng, [(640, 64), (64, 640)]),
          _rand_images(rng, RAGGED), _rand_images(rng, [(400, 300)] * 5)]
  streamed = list(drv.serve_stream_tta(reqs))
  ref = _driver()
  for req, got in zip(reqs, streamed):
    want = ref.serve_images_tta(req)
    assert len(got) == len(want) and all(wo.same_bits(a, b) for a, b in zip(got, want))


def test_fixed_batch_size_driver():
  drv = _driver(batch_size=2)
  rng = np.random.default_rng(51)
  images = _rand_images(rng, [(100, 200), (300, 150)])
  got = drv.serve_images_tta(images)
  want = _driver().serve_images_tta(images)
  assert all(wo.same_bits(a, b) for a, b in zip(got, want))
  with pytest.raises(ValueError):
    drv.serve_images_tta(images[:1])


def test_detection_unchanged_by_interleaved_tta():
  drv = _driver(batch_size=2)
  rng = np.random.default_rng(61)
  det_images = _rand_images(rng, [(240, 320), (200, 256)])
  first = drv.serve_images(det_images)
  tta_first = drv.serve_images_tta(det_images)
  for _ in range(2):
    drv.serve_images_tta(_rand_images(rng, [(256, 200), (64, 96)]))
    assert np.array_equal(drv.serve_images(det_images), first)
  handles = [drv.submit(det_images), drv.submit_tta(det_images), drv.submit(det_images)]
  assert np.array_equal(handles[0].result(), first) and np.array_equal(handles[2].result(), first)
  assert all(wo.same_bits(a, b) for a, b in zip(handles[1].result(), tta_first))


def test_detection_on_the_shared_engine_unchanged_by_interleaved_tta():
  """batch_size=None: a TTA request of n images runs on the engine (and slots) of regular requests
  of 2n images.  Its pre-NMS rewrites the buffer set the previous regular request's NMS may still
  be reading, so it must wait for that NMS; regular and TTA results, interleaved in both orders,
  equal each request served alone."""
  rng = np.random.default_rng(71)
  big = [_rand_images(rng, [(240, 320), (200, 256), (256, 256), (180, 300)]) for _ in range(2)]
  small = [_rand_images(rng, [(256, 200), (64, 96)]) for _ in range(2)]
  alone = _driver()
  det_alone = [alone.serve_images(b) for b in big]
  tta_alone = [_driver().serve_images_tta(s) for s in small]
  drv = _driver()
  for _ in range(3):
    handles = [('det', 0, drv.submit(big[0])), ('tta', 0, drv.submit_tta(small[0])),
               ('det', 1, drv.submit(big[1])), ('tta', 1, drv.submit_tta(small[1])),
               ('tta', 0, drv.submit_tta(small[0])), ('det', 0, drv.submit(big[0]))]
    for kind, i, h in handles:
      if kind == 'det':
        assert np.array_equal(h.result(), det_alone[i]), (kind, i)
      else:
        got = h.result()
        assert len(got) == len(tta_alone[i]) and all(
            wo.same_bits(a, b) for a, b in zip(got, tta_alone[i])), (kind, i)
  assert drv._engines.keys() == {4}        # pylint: disable=protected-access


def test_segmentation_only_config_raises():
  drv = _driver(batch_size=1, heads=['segmentation'])
  with pytest.raises(ValueError):
    drv.serve_images_tta([np.zeros((64, 64, 3), np.uint8)])
