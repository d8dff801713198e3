"""Detections and segmentation masks from one pipelined pass: ServingDriver.serve_images_with_masks /
submit_with_masks / serve_stream_with_masks against serve_images and segment_images on the same
driver, bit for bit, alone, streamed, interleaved with every other request kind, with each stream
of the path stalled in turn, and on engines built with pipeline=False; and Engine.run(after_heads=)
refusing engines without the segmentation head.

The stall harness, its stall points and its helpers are those of tests/test_gpu_stream_handoffs.py.
A combined request crosses the driver's copy stream (h2d), the main stream (preprocess, bb1, bb2),
the engine's head stream (cell0, heads+pre, then seg_masks from the after_heads hook), its NMS stream
(nms, then the detection copy) and the driver's D2H stream (d2h, the mask copy)."""
import functools

import numpy as np
import pytest
import torch

import test_gpu_stream_handoffs as sh

pytestmark = pytest.mark.gpu
harness = sh.harness          # autouse: the stall points and wait controls of the handoffs file

BOTH = ['object_detection', 'segmentation']
SIZES = (128, 256)
MODES = {'pipelined': '1', 'sequential': '0'}   # EDET_PIPELINE of the driver's engines


@pytest.fixture(scope='module')
def cache():
  built = {}
  yield built
  built.clear()
  torch.cuda.synchronize()


def _driver(cache, size, batch_size, mode='pipelined'):
  """A both-heads D0 driver at `size` with seeded synthetic weights, built once per module; its
  engines are built under the mode's EDET_PIPELINE (batch_size=None: on each first use, see
  _serving)."""
  from automl_b200 import inference
  key = ('driver', size, batch_size, mode)
  if key not in cache:
    with pytest.MonkeyPatch.context() as m:
      m.setenv('EDET_PIPELINE', MODES[mode])
      drv = inference.ServingDriver('efficientdet-d0', '_', batch_size=batch_size,
                                    model_params={'image_size': size, 'heads': BOTH})
      drv.build()
    drv.mode = mode
    cache[key] = drv
  return cache[key]


def _serving(drv, fn):
  """fn() with engines built on first use getting the driver's EDET_PIPELINE."""
  with pytest.MonkeyPatch.context() as m:
    m.setenv('EDET_PIPELINE', MODES[drv.mode])
    out = fn()
  torch.cuda.synchronize()
  for eng in drv._engines.values():                                # pylint: disable=protected-access
    assert eng.pipeline == (drv.mode == 'pipelined')
  return out


def _two_passes(drv, request):
  return drv.serve_images(request), drv.segment_images(request)


def _assert_same(got, want):
  assert len(got) == len(want)
  bad = [i for i, (g, w) in enumerate(zip(got, want)) if not sh._same(g, w)]
  assert bad == [], 'results that differ: %s' % bad


def _check_result(result, request_shapes, max_output_size):
  det, masks = result
  assert det.dtype == np.float32 and det.shape == (len(request_shapes), max_output_size, 7)
  assert [m.shape for m in masks] == [tuple(s) for s in request_shapes]
  assert all(m.dtype == np.uint8 for m in masks)


def _shapes(request):
  if isinstance(request, torch.Tensor):
    return [tuple(request.shape[1:3])] * request.shape[0]
  return [im.shape[:2] for im in request]


# ---- one request, against the two passes on the same driver --------------------------------------
def _case(rng, case):
  """(batch_size, requests) of a case."""
  if case == 'uniform':
    return 4, [sh._images(rng, [(96, 128)] * 4), sh._pinned(rng, (150, 100), 4),
               sh._on_device(rng, (128, 128), 4)]
  if case == 'ragged':        # with a 1 x N and an N x 1 image
    return 4, [sh._images(rng, [(1, 100), (100, 1), (200, 150), (64, 90)]),
               sh._images(rng, [(300, 240), (37, 53), (128, 128), (90, 300)])]
  if case == 'single':
    return 1, [sh._images(rng, [(120, 160)]), sh._images(rng, [(1, 77)]),
               sh._on_device(rng, (200, 90), 1)]
  # batch_size=None: three request sizes, so three engines and three slot rings
  return None, [sh._images(rng, [(96, 128)] * 3), sh._images(rng, [(180, 120)]),
                sh._images(rng, [(64, 200), (100, 1)]), sh._pinned(rng, (128, 96), 3),
                sh._images(rng, [(1, 100), (150, 150)]), sh._on_device(rng, (80, 80), 1)]


@pytest.mark.parametrize('case,mode', [('uniform', 'pipelined'), ('ragged', 'pipelined'),
                                       ('single', 'pipelined'), ('dynamic', 'pipelined'),
                                       ('uniform', 'sequential'), ('ragged', 'sequential')])
@pytest.mark.parametrize('size', SIZES)
def test_one_pass_equals_two_passes(cache, size, case, mode):
  """Each request of the case on the same driver; engines built with pipeline=False must also give
  the bits of the pipelined engines."""
  batch_size, reqs = _case(np.random.default_rng(SIZES.index(size) * 10 + len(case)), case)
  drv = _driver(cache, size, batch_size, mode)
  got = _serving(drv, lambda: [drv.serve_images_with_masks(r) for r in reqs])
  want = _serving(drv, lambda: [_two_passes(drv, r) for r in reqs])
  max_out = next(iter(drv._engines.values())).max_output_size     # pylint: disable=protected-access
  for r, g in zip(reqs, got):
    _check_result(g, _shapes(r), max_out)
  _assert_same(got, want)
  if case == 'dynamic':
    assert {1, 2, 3} <= set(drv._engines)                          # pylint: disable=protected-access
  key = ('result', size, case)
  if key in cache:       # the other mode's engines give the same bits (pipelined runs first)
    _assert_same(got, cache[key])
  else:
    cache[key] = got


# ---- streamed, and interleaved with the other request kinds --------------------------------------
def _stream_requests(rng):
  """Seven requests of different sizes and counts, every staging form."""
  return [sh._images(rng, [(96, 128)] * 2), sh._images(rng, [(200, 150), (64, 90), (1, 60)]),
          sh._pinned(rng, (100, 160), 1), sh._images(rng, [(300, 240), (128, 128)]),
          sh._on_device(rng, (80, 200), 3), sh._images(rng, [(192, 144)] * 2),
          sh._images(rng, [(60, 1)])]


@pytest.mark.parametrize('size', SIZES)
def test_stream_equals_each_request_alone(cache, size):
  drv = _driver(cache, size, None)
  reqs = _stream_requests(np.random.default_rng(size))
  want = _serving(drv, lambda: [drv.serve_images_with_masks(r) for r in reqs])
  got = _serving(drv, lambda: list(drv.serve_stream_with_masks(reqs)))
  _assert_same(got, want)


def _submitters(drv):
  return {'both': drv.submit_with_masks, 'det': drv.submit, 'seg': drv.submit_segment,
          'tta': drv.submit_tta}


def _alone(drv, kind, request):
  return _submitters(drv)[kind](request).result()


def _mixed_plan(rng):
  """Combined, detection, mask and TTA requests on a batch_size=None driver; requests of four images
  and TTA requests of two share the engine of four."""
  return [('both', sh._images(rng, [(240, 320), (200, 256), (1, 90), (180, 300)])),
          ('det', sh._images(rng, [(256, 200)] * 4)),
          ('tta', sh._images(rng, [(256, 200), (64, 96)])),
          ('both', sh._pinned(rng, (200, 240), 4)),
          ('seg', sh._images(rng, [(99, 77), (256, 256), (200, 100), (64, 64)])),
          ('both', sh._images(rng, [(120, 160)] * 2)),
          ('tta', sh._pinned(rng, (180, 256), 2)),
          ('both', sh._on_device(rng, (160, 240), 4)),
          ('det', sh._images(rng, [(64, 96), (300, 200)])),
          ('both', sh._images(rng, [(90, 1), (256, 256), (200, 100), (64, 64)]))]


def _mixed(cache, size):
  key = ('mixed', size)
  if key not in cache:
    drv = _driver(cache, size, None)
    plan = _mixed_plan(np.random.default_rng(100 + size))
    cache[key] = (drv, plan, _serving(drv, lambda: [_alone(drv, k, r) for k, r in plan]))
  return cache[key]


def _run_plan(drv, plan):
  from automl_b200 import staging
  submit = _submitters(drv)
  return list(staging.pipelined(lambda kr: submit[kr[0]](kr[1]), sh._indexed(plan),
                                drv.MAX_IN_FLIGHT))


@pytest.mark.parametrize('size', SIZES)
def test_interleaved_with_every_request_kind(cache, size):
  drv, plan, want = _mixed(cache, size)
  _assert_same(_serving(drv, lambda: _run_plan(drv, plan)), want)
  assert {2, 4} <= set(drv._engines)                               # pylint: disable=protected-access


# ---- every stream stalled in turn -----------------------------------------------------------------
STALL_POINTS = {
    'pipelined': ('h2d', 'preprocess', 'bb1', 'bb2', 'cell0', 'heads+pre', 'seg_masks', 'nms', 'd2h'),
    'sequential': ('h2d', 'preprocess', 'net+pre', 'seg_masks', 'nms', 'd2h'),
}


def _combined_stream(cache, mode):
  key = ('combined', mode)
  if key not in cache:
    drv = _driver(cache, 128, 2, mode)
    rng = np.random.default_rng(211)
    reqs = [sh._images(rng, [(96, 128)] * 2), sh._images(rng, [(200, 150), (1, 90)]),
            sh._pinned(rng, (100, 160), 2), sh._images(rng, [(300, 240), (128, 128)]),
            sh._on_device(rng, (80, 200), 2), sh._images(rng, [(192, 144), (90, 1)])]
    cache[key] = (drv, reqs, _serving(drv, lambda: [drv.serve_images_with_masks(r) for r in reqs]))
  return cache[key]


def _run_combined(drv, reqs, want, points, target):
  sh._watch_driver(drv)
  got = sh._stalled(points, target, lambda: list(drv.serve_stream_with_masks(sh._indexed(reqs))))
  return sh._mismatches(got, want)


@pytest.mark.parametrize('which', sh.WHICH)
@pytest.mark.parametrize('mode,point', [(m, p) for m, ps in STALL_POINTS.items() for p in ps])
def test_combined_stream_stalled(cache, mode, point, which):
  """Combined requests of two images through serve_stream_with_masks, `point` stalled: a stalled
  mask kernel also holds back the staging release and the next request's head stage, which
  rewrites seg_out."""
  drv, reqs, want = _combined_stream(cache, mode)
  assert _run_combined(drv, reqs, want, [point], sh._target(which, len(reqs))) == []


@pytest.mark.parametrize('which', sh.WHICH)
@pytest.mark.parametrize('point', STALL_POINTS['pipelined'])
def test_interleaved_kinds_stalled(cache, point, which):
  drv, plan, want = _mixed(cache, 256)
  both = [i for i, (kind, _) in enumerate(plan) if kind == 'both']
  target = None if which == 'all' else both[len(both) // 2]
  sh._watch_driver(drv)
  got = sh._stalled([point], target, lambda: _run_plan(drv, plan))
  assert sh._mismatches(got, want) == []


def test_control_result_waits_for_the_detection_copy(cache):
  """The mask copy waits for slot.ev_out, recorded on the NMS stream after the detection copy; with
  that wait skipped, ev_done no longer follows the detections of a stalled NMS stage."""
  drv, reqs, want = _combined_stream(cache, 'pipelined')
  drop = [(drv._d2h_stream, s.ev_out) for s in drv._slots[2]]      # pylint: disable=protected-access
  sh._expect_caught(lambda: _run_combined(drv, reqs, want, ['nms'], None), drop)


# ---- Engine.run(after_heads=) -------------------------------------------------------------------
@pytest.mark.parametrize('heads,postprocess', [(['object_detection'], True), (BOTH, False)],
                         ids=['detection_only', 'network_only'])
def test_after_heads_refused_before_anything_is_enqueued(heads, postprocess):
  from automl_b200 import hparams_config, weights
  from automl_b200.arch import DetArch
  from automl_b200.engine import Engine
  c = hparams_config.get_efficientdet_config('efficientdet-d0')
  c.override(dict(image_size=128, heads=heads))
  eng = Engine(c, weights.synthetic_weights(DetArch(c), 3), 1)
  called = []
  with pytest.raises(ValueError, match='after_heads needs the segmentation head'):
    eng.run(postprocess=postprocess, after_heads=called.append)
  assert called == [] and eng._step == 0 and eng._graph is None    # pylint: disable=protected-access
  assert not eng._logits_current                                   # pylint: disable=protected-access


def test_after_heads_sees_the_step_logits(cache):
  """The hook receives seg_out after the step's head stage: the logits it copies on the head stream
  equal those of forward() on the same input."""
  drv = _driver(cache, 128, 2)
  eng = drv._engines[2]                                            # pylint: disable=protected-access
  rng = np.random.default_rng(5)
  xs = [torch.from_numpy(rng.uniform(-2, 2, size=(2, 128, 128, 3)).astype(np.float32)).to(sh.DEV)
        for _ in range(3)]
  outs = [torch.empty_like(eng.seg_out) for _ in xs]
  for x, out in zip(xs, outs):
    eng.input.copy_(x)
    eng.run(postprocess=True, after_heads=functools.partial(lambda o, seg: o.copy_(seg), out))
  eng.wait_detections()
  for x, out in zip(xs, outs):
    eng.forward(x)
    assert torch.equal(out, eng.seg_out)
