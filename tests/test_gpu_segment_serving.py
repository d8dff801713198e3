"""Segmentation masks on the GPU: edet_seg_masks bit for bit against the numpy oracle
(tests/seg_mask_oracle.py), a packed output past 2^31 bytes, its programmatic-dependent-launch
read of the logits, and ServingDriver.segment_images / segment_stream end to end."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import plan_settings as ps
import seg_mask_oracle as smo
import seg_oracle
from automl_b200 import utils

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GUARD = 4096             # sentinel bytes after the packed masks
SENTINEL = 0xAB
BOTH = ['object_detection', 'segmentation']
# fp32-oracle agreement: pixels whose fp32 top-two logit margin exceeds MARGIN times the RMS of the
# fp32 logits (the device logits are within 1e-3 rel-L2 of them, tests/test_gpu_segmentation.py)
MARGIN = 0.05


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _round8(x):
  return (x + 7) // 8 * 8


def _logits(rng, n, hs, ws, c, ld, ties=False, nans=0):
  """fp16 [n, hs, ws, ld]: channels >= c hold large values the kernel must never read as classes."""
  if ties:      # few distinct values: many equal maxima
    x = rng.integers(-2, 3, size=(n, hs, ws, ld)).astype(np.float16)
  else:
    x = rng.standard_normal((n, hs, ws, ld)).astype(np.float16)
  x[..., c:] = 1000
  for _ in range(nans):
    x[rng.integers(n), rng.integers(hs), rng.integers(ws), rng.integers(c)] = np.nan
  return x


def _run(logits, c, f, table, total, shapes):
  """Launches seg_masks into a buffer with GUARD sentinel bytes behind the packed masks; checks
  the sentinels and returns the masks."""
  ops = _ops()
  lg = torch.from_numpy(logits).to(DEV)
  tb = torch.from_numpy(table).to(DEV)
  out = torch.full((total + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
  max_hw = tuple(int(v) for v in np.max(np.asarray(shapes), axis=0))
  ops.seg_masks(lg, c, f, tb, max_hw, out)
  host = out.cpu().numpy()
  assert (host[total:] == SENTINEL).all(), 'written past the packed masks'
  masks, off = [], 0
  for h, w in shapes:
    masks.append(host[off:off + h * w].reshape(h, w))
    off += h * w
  return masks


def _images(table):
  return [tuple(int(v) for v in row[2:]) for row in table]


SHAPES = [(1, 1), (1, 7), (7, 1), (3, 250), (250, 3), (64, 64), (128, 96), (96, 128), (480, 640),
          (640, 480), (37, 53), (1000, 1500), (2001, 999)]


@pytest.mark.parametrize('c', [1, 3, 8, 19, 256])
@pytest.mark.parametrize('ties', [False, True])
def test_kernel_matches_oracle(c, ties):
  from automl_b200 import inference
  rng = np.random.default_rng(c * 2 + ties)
  f, hs, ws = 4, 32, 24                        # a 128 x 96 network input
  ld = _round8(c) + 8                          # ld > C: the padding channels are ignored
  table, total = inference.seg_mask_table(SHAPES, (hs * f, ws * f))
  lg = _logits(rng, len(SHAPES), hs, ws, c, ld, ties=ties, nans=0 if ties else 20)
  got = _run(lg, c, f, table, total, SHAPES)
  want = smo.masks(lg, c, f, _images(table))
  for i, (g, w) in enumerate(zip(got, want)):
    assert np.array_equal(g, w), 'image %d %s' % (i, SHAPES[i])
  if c > 1:
    assert len(np.unique(np.concatenate([m.ravel() for m in got]))) > 1


def test_kernel_hand_rows_and_grid_factors():
  """Table rows written by hand (scaled sizes that cover the whole grid, a sliver of it, or one
  cell) at f = 1, 2 and 8."""
  rng = np.random.default_rng(5)
  for f in (1, 2, 8):
    hs, ws, c = 9, 13, 5
    rows = [(50, 70, hs * f, ws * f), (3, 3, 1, 1), (1, 200, 1, ws * f), (200, 1, hs * f, 1),
            (hs * f, ws * f, hs * f, ws * f)]
    lg = _logits(rng, len(rows), hs, ws, c, 8)
    table = np.zeros((len(rows), 6), np.int32)
    areas = [h * w for h, w, _, _ in rows]
    table[:, :2] = np.concatenate([[0], np.cumsum(areas)[:-1]]).astype(np.int64).view(np.int32).reshape(-1, 2)
    table[:, 2:] = rows
    shapes = [(h, w) for h, w, _, _ in rows]
    got = _run(lg, c, f, table, sum(areas), shapes)
    for g, w in zip(got, smo.masks(lg, c, f, rows)):
      assert np.array_equal(g, w), f


def test_packed_output_past_2_31_bytes():
  """Three 30000 x 30000 masks: 2.7e9 bytes, the last mask starting past 2^31."""
  from automl_b200 import inference
  rng = np.random.default_rng(9)
  f, hs, ws, c = 4, 128, 128, 19
  shapes = [(30000, 30000)] * 3
  table, total = inference.seg_mask_table(shapes, (hs * f, ws * f))
  assert total > 2 ** 31
  lg = _logits(rng, 3, hs, ws, c, 24)
  ops = _ops()
  out = torch.full((total + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
  ops.seg_masks(torch.from_numpy(lg).to(DEV), c, f, torch.from_numpy(table).to(DEV),
                (30000, 30000), out)
  torch.cuda.synchronize()
  assert bool((out[total:] == SENTINEL).all())
  for i in range(3):
    ys = np.concatenate([[0, 1, 29998, 29999, 29999, 0], rng.integers(0, 30000, 200)])
    xs = np.concatenate([[0, 29999, 0, 29998, 29999, 15000], rng.integers(0, 30000, 200)])
    idx = torch.from_numpy(i * 9 * 10 ** 8 + ys * 30000 + xs).to(DEV)
    got = out[idx].cpu().numpy()
    want = smo.pixels(lg, c, f, _images(table)[i], i, ys, xs)
    assert np.array_equal(got, want), i
  del out
  torch.cuda.empty_cache()


def test_reads_logits_written_by_the_previous_kernel():
  """RAW through PDL (the pattern of tests/test_gpu_pdl_chains.py): a one-CTA identity copy writes
  the logits, the mask kernel is launched right behind it and must see every row the copy wrote,
  though its CTAs start while the copy is still running."""
  ops = _ops()
  rows, hs, ws, c, f = 1 << 17, 64, 32, 19, 4
  g = torch.Generator().manual_seed(1)
  old = (torch.randn(rows, 64, generator=g) * 0.5).half()
  new = (torch.randn(rows, 64, generator=g) * 0.5).half()
  old[old == 0] = 0.5
  new[new == 0] = 0.5                           # -0 would come back as +0
  region = old.to(DEV)
  src = new.to(DEV)
  eye = torch.eye(64, dtype=torch.float16, device=DEV)
  zero = torch.zeros(64, dtype=torch.float32, device=DEV)
  logits = region[rows - hs * ws:].view(1, hs, ws, 64)     # the rows the copy writes last
  shape = (hs * f, ws * f)
  images = [shape + shape]
  total = shape[0] * shape[1]
  tb = torch.zeros(1, 6, dtype=torch.int32)
  tb[0, 2:] = torch.tensor(images[0])
  tb = tb.to(DEV)
  out = torch.full((total + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)

  def masks_of(t):
    lgn = t[rows - hs * ws:].view(1, hs, ws, 64).cpu().numpy()
    return smo.masks(lgn, c, f, images)[0]

  want, before = masks_of(new), masks_of(old)
  assert not np.array_equal(want, before), 'the chain could not fail'
  ops.pointwise_conv(src[:256], eye, zero, region[:256].clone(), utils.ACT_NONE)   # warm both
  ops.seg_masks(logits, c, f, tb, shape, out)
  torch.cuda.synchronize()
  region.copy_(old.to(DEV))
  out.fill_(SENTINEL)
  torch.cuda.synchronize()
  torch.cuda._sleep(1 << 22)                    # the host queues the chain meanwhile
  ops.set_option('max_ctas', 1)
  try:
    ops.pointwise_conv(src, eye, zero, region, utils.ACT_NONE)
  finally:
    ps.reset(ops)
  ops.seg_masks(logits, c, f, tb, shape, out)
  torch.cuda.synchronize()
  host = out.cpu().numpy()
  assert (host[total:] == SENTINEL).all()
  assert np.array_equal(host[:total].reshape(shape), want), \
      'the mask kernel read logits before its grid-dependency wait'
  assert torch.equal(region.cpu(), new)


# ---- ServingDriver ------------------------------------------------------------------------------
def _driver(heads, batch_size=None, size=256):
  from automl_b200 import inference
  return inference.ServingDriver('efficientdet-d0', '_', batch_size=batch_size,
                                 model_params={'image_size': size, 'heads': heads})


def _rand_images(rng, shapes):
  return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes]


RAGGED = [(200, 256), (256, 180), (37, 300), (300, 300), (5, 7), (512, 384)]


@pytest.mark.parametrize('heads', [['segmentation'], BOTH], ids=['seg', 'both'])
def test_segment_images_end_to_end(heads):
  from automl_b200 import inference
  drv = _driver(heads)
  rng = np.random.default_rng(21)
  images = _rand_images(rng, RAGGED)
  got = drv.segment_images(images)
  eng = drv._engines[len(images)]   # pylint: disable=protected-access
  torch.cuda.synchronize()
  assert [m.shape for m in got] == RAGGED and all(m.dtype == np.uint8 for m in got)
  c = drv.config.seg_num_classes
  table, _ = inference.seg_mask_table(RAGGED, 256)
  # the device's own logits through the oracle: bit for bit
  dev_logits = eng.seg_logits.cpu().numpy()
  for i, (g, w) in enumerate(zip(got, smo.masks(dev_logits, c, 4, _images(table)))):
    assert np.array_equal(g, w), i
  # the fp32 oracle network on the device's pre-processed input: equal wherever it is decisive
  ref = seg_oracle.seg_logits(drv.config, drv._weights, eng.input.cpu().numpy(), torch.float32).numpy()  # pylint: disable=protected-access
  top2 = np.sort(ref, axis=-1)[..., -2:]
  decisive = (top2[..., 1] - top2[..., 0]) > MARGIN * float(np.sqrt((ref ** 2).mean()))
  ref_masks = smo.masks(ref, c, 4, _images(table))
  checked = 0
  for i, (h, w, sh, sw) in enumerate(_images(table)):
    cy, cx = smo.cells(h, sh, 4, 64), smo.cells(w, sw, 4, 64)
    keep = decisive[i][cy[:, None], cx[None, :]]
    assert np.array_equal(got[i][keep], ref_masks[i][keep]), i
    checked += int(keep.sum())
  assert checked >= 0.8 * sum(h * w for h, w in RAGGED)


def test_request_forms_agree():
  drv = _driver(['segmentation'])
  rng = np.random.default_rng(31)
  ragged = _rand_images(rng, [(120, 160)] * 3 + [(90, 250)])
  alone = [drv.segment_images([im])[0] for im in ragged]
  together = drv.segment_images(ragged)
  for a, b in zip(alone, together):
    assert np.array_equal(a, b)
  # a uniform batch (list and pinned tensor) equals the same images inside a ragged request
  uniform = drv.segment_images(ragged[:3])
  pinned = drv.segment_images(torch.from_numpy(np.stack(ragged[:3])).pin_memory())
  for a, b, t in zip(uniform, pinned, together[:3]):
    assert np.array_equal(a, t) and np.array_equal(b, t)


def test_segment_stream_equals_sequential():
  drv = _driver(['segmentation'])
  rng = np.random.default_rng(41)
  reqs = [_rand_images(rng, RAGGED), _rand_images(rng, [(256, 256)] * 2),
          _rand_images(rng, RAGGED[::-1]), _rand_images(rng, [(640, 64), (64, 640)]),
          _rand_images(rng, RAGGED), _rand_images(rng, [(1000, 800)] * 6)]
  streamed = list(drv.segment_stream(reqs))
  ref = _driver(['segmentation'])
  for req, got in zip(reqs, streamed):
    want = ref.segment_images(req)
    assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want))


def test_fixed_batch_size_driver():
  drv = _driver(['segmentation'], batch_size=2)
  rng = np.random.default_rng(51)
  images = _rand_images(rng, [(100, 200), (300, 150)])
  got = drv.segment_images(images)
  want = _driver(['segmentation']).segment_images(images)
  assert all(np.array_equal(a, b) for a, b in zip(got, want))
  with pytest.raises(ValueError):
    drv.segment_images(images[:1])


def test_detection_unchanged_by_interleaved_masks():
  drv = _driver(BOTH, batch_size=2)
  rng = np.random.default_rng(61)
  det_images = _rand_images(rng, [(240, 320), (200, 256)])
  first = drv.serve_images(det_images)
  for _ in range(2):
    drv.segment_images(_rand_images(rng, [(256, 200), (64, 96)]))
    assert np.array_equal(drv.serve_images(det_images), first)
  handles = [drv.submit(det_images), drv.submit_segment(_rand_images(rng, [(99, 77)] * 2)),
             drv.submit(det_images)]
  assert np.array_equal(handles[0].result(), first) and np.array_equal(handles[2].result(), first)
  assert len(handles[1].result()) == 2
  # the same detections as a detection-only driver (the seeded weights they share are equal)
  det_only = _driver(['object_detection'], batch_size=2)
  assert np.array_equal(det_only.serve_images(det_images), first)


def test_segmentation_only_driver_refuses_detection():
  drv = _driver(['segmentation'], batch_size=1)
  with pytest.raises(ValueError):
    drv.serve_images([np.zeros((64, 64, 3), np.uint8)])


def test_seg_masks_compiles_without_spills():
  from automl_b200 import build
  src = os.path.join(build.CSRC, 'seg_masks.cu')
  with tempfile.TemporaryDirectory() as tmp:
    res = subprocess.run([build.NVCC] + [f for f in build.FLAGS if f != '--shared'] +
                         ['-Xptxas', '-v', '-c', src, '-o', os.path.join(tmp, 'seg_masks.o')],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  assert res.returncode == 0, res.stdout
  assert "for 'sm_90a'" in res.stdout
  spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', res.stdout)
  assert spills and all(s == ('0', '0') for s in spills), res.stdout
