"""Every cross-stream hand-off of the pipelined engine, ServingDriver and EffNetV2Model, with each
stage stalled in turn.

A detection request crosses up to six streams: the driver's copy stream (H2D), the main stream
(pre-process, bb1, bb2), the engine's head stream (cell0, heads+pre), its NMS stream
(NMS, then the after_nms D2H), the driver's D2H stream (masks, TTA) and, in eager mode, the branch
streams of Engine._run_ops; EffNetV2Model adds copy and D2H streams of its own.  At test sizes every
stage finishes long before the next request reaches it, so comparing pipelined with sequential
results under natural timing passes with a wait missing.  Here one named stall point is stalled: a
torch.cuda._sleep is enqueued on its stream after its own waits, so the stage's reads and writes
move STALL_CYCLES later while the host keeps enqueueing requests.  Stalling stage X checks that
every reader of X's outputs waits for X (read after write) and that every writer of X's inputs waits
until X has read them (write after read).

The stall points are patched in from this file; the product code has no hooks for them:
  h2d            the copy streams (driver, classifier, serve_stream), after their wait_event
  preprocess     ops.preprocess, preprocess_ragged, preprocess_mirrored and cls_preprocess
  bb1, bb2, cell0, heads+pre   Engine._replay, before the stage runs
  net, net+pre   the graphs Engine._graph_for returns, before replay
  nms            the engine's NMS stream, after its wait_event
  after_nms      parallel.gather_detections, the first call of the driver's after_nms hook
  d2h            the D2H streams (driver, classifier, serve_stream), after their wait_event
  seg_masks, per_class_nms, wbf, softmax_topk   the ops of those names
  branch         the side streams of Engine._run_ops (eager engine), after their fork
  run            EffNetV2Model.run
  out copy       serve_stream's main stream, after it waits for the D2H of result k-2
Each point counts how often it fires, and a case fails if a point it declares never fires.  A case
stalls its point on every request in one run and on one middle request in another.  Consecutive
requests have different images and scales, so a stale read changes the result; each result must
equal the same request served alone and synchronously on the same driver or model, bit for bit.

Controls: for each wait whose removal cannot fault (it guards fixed-size, warmed buffers, where any
mix of earlier valid contents is in bounds for the reader), one test skips that single wait -- a
Stream.wait_event or Event.synchronize wrapper that ignores one event object on one stream -- and
must see the matching stall case mismatch.  HANDOFFS lists every wait_event, wait_stream and
synchronize() of engine.py, inference.py, staging.py and effnetv2_model.py with the case that
exercises it and its control or the reason it has none; tests/test_stream_handoff_pins.py checks
the list against the sources.  Every case and every control runs once."""
import collections
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# ~8.5 ms at the H100's 1.98 GHz: the host enqueues the next requests of these small configurations
# well inside it (every control below catches its dropped wait on an H100 SXM at 700 W; a control
# that stops catching it means the stall has become too short)
STALL_CYCLES = 1 << 24
WHICH = ('all', 'middle')

# (module, function, call, the case that exercises it, its control or why it has none)
_EAGER_JOIN = ('no control: the wait is on an event recorded on the spot, which a wrapper cannot '
               'single out from the other forks and joins of the pass; graph replays turn it into '
               'a graph edge')
_IMPLIED_SLOT = ('no control: implied -- ServingDriver._acquire completes the slot\'s previous '
                 'request (a host wait with a control of its own) before the slot is restaged')
HANDOFFS = [
    ('engine.py', 'Engine._run_ops', 'main.wait_stream(open_branches.pop(name))',
     'test_detection_stream', _EAGER_JOIN),
    ('engine.py', 'Engine._run_ops', 'st.wait_stream(main)', 'test_detection_stream', _EAGER_JOIN),
    ('engine.py', 'Engine._run_ops', 'main.wait_stream(st)', 'test_detection_stream', _EAGER_JOIN),
    ('engine.py', 'Engine._graph_for', 'torch.cuda.synchronize(self.device)', 'test_detection_stream',
     'no control: a host synchronisation before a graph capture, not a hand-off of serving work'),
    ('engine.py', 'Engine.run', 'torch.cuda.current_stream(self.device).wait_event(self._ev_pre[self._cur])',
     'test_engine_call_behind_a_stalled_step',
     'no control: dropping it puts the pending head stage and forward()\'s network in flight at once '
     'on the same launches, and so on the same tile-scheduler slots (LaunchList._bound)'),
    ('engine.py', 'Engine.run', 'main.wait_event(self._ev_nms[sidx])', 'test_detection_stream',
     'test_control_sequential_step_waits_for_nms'),
    ('engine.py', 'Engine._enqueue_nms', 'self._nms_stream.wait_event(self._ev_pre[sidx])',
     'test_detection_stream', 'test_control_nms_waits_for_pre_nms'),
    ('engine.py', 'Engine._run_pipelined', 'main.wait_event(self._ev_head)', 'test_detection_stream',
     'test_control_backbone_waits_for_cell0'),
    ('engine.py', 'Engine._enqueue_heads', 'hs.wait_event(self._ev_bb)', 'test_detection_stream',
     'test_control_heads_wait_for_backbone'),
    ('engine.py', 'Engine._enqueue_heads', 'hs.wait_event(self._ev_nms[sidx])', 'test_detection_stream',
     'test_control_heads_wait_for_nms'),
    ('engine.py', 'Engine.wait_detections',
     'torch.cuda.current_stream(self.device).wait_event(self._ev_nms[self._cur])',
     'test_engine_call_behind_a_stalled_step', 'test_control_detect_waits_for_nms'),
    ('engine.py', 'Engine.pre_nms_only', 'main.wait_event(self._ev_nms[self._cur])',
     'test_engine_call_behind_a_stalled_step', 'test_control_pre_nms_after_forward_waits_for_nms'),
    ('engine.py', 'Engine.pre_nms_only', 'main.wait_event(self._ev_pre[self._cur])',
     'test_engine_call_behind_a_stalled_step', 'test_control_pre_nms_waits_for_head_stage'),
    ('inference.py', '_Request.result', 'self._slot.ev_done.synchronize()', 'test_detection_stream',
     'test_control_result_waits_for_the_download'),
    ('inference.py', 'ServingDriver._download', 'self._d2h_stream.wait_event(slot.ev_out)',
     'test_mixed_request_kinds', 'test_control_downloads_wait_for_mask_and_tta_kernels'),
    ('staging.py', 'StagingSlot.stage', 'self.ev_h2d.synchronize()', 'test_growing_requests',
     _IMPLIED_SLOT),
    ('staging.py', 'StagingSlot.stage', 'main.synchronize()', 'test_growing_requests',
     'no control: it guards a staging buffer that is about to be freed'),
    ('staging.py', 'StagingSlot.stage', 'copy_stream.wait_event(self.ev_raw_free)', 'test_detection_stream',
     _IMPLIED_SLOT + '; the classifier collects a slot\'s results before reusing it, and its '
     'preprocess() alone stages a descriptor table that this wait guards'),
    ('staging.py', 'StagingSlot.stage', 'main.wait_event(self.ev_h2d)', 'test_detection_stream',
     'test_control_preprocess_waits_for_h2d'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.run', 'torch.cuda.synchronize()',
     'test_serve_stream',
     'no control: a host synchronisation before a graph capture, not a hand-off of serving work'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.serve_stream',
     "p['h2d'].wait_event(p['ev_in_free'][s])", 'test_serve_stream',
     'no control: implied -- before batch k+2 is staged the host has waited for the D2H of result k, '
     'which follows the main stream\'s copy out of the staging buffer'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.serve_stream', "main.wait_event(p['ev_h2d'][s])",
     'test_serve_stream', 'test_control_serve_stream_copy_waits_for_h2d'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.serve_stream',
     "main.wait_event(p['ev_d2h'][(k - 2) % 3])", 'test_serve_stream',
     'no control: implied -- the host waited for the D2H of result k-2 before it yielded that result'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.serve_stream', "p['d2h'].wait_event(p['ev_out'][s])",
     'test_serve_stream', 'test_control_serve_stream_download_waits_for_out_copy'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.serve_stream', "p['ev_d2h'][prev].synchronize()",
     'test_serve_stream', 'test_control_serve_stream_yields_after_the_download'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model.serve_stream', "p['ev_d2h'][prev].synchronize()",
     'test_serve_stream', 'test_control_serve_stream_yields_after_the_download'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model._classify_enqueue', 'main.wait_event(slot.ev_d2h)',
     'test_classify_stream',
     'no control: implied -- classify and classify_stream collect a slot\'s results (a host wait with '
     'a control of its own) before the slot is reused'),
    ('efficientnetv2/effnetv2_model.py', 'EffNetV2Model._classify_enqueue', 'd2h.wait_event(slot.ev_out)',
     'test_classify_stream', 'test_control_classify_download_waits_for_top_k'),
    ('efficientnetv2/effnetv2_model.py', '_ClassifySlot.result', 'self.ev_d2h.synchronize()',
     'test_classify_stream', 'test_control_classify_result_waits_for_the_download'),
]


# ---- the harness ------------------------------------------------------------------------------
class _Harness(object):
  """Which stall points are active, on which request, and the waits a control skips."""

  def __init__(self):
    self.points = set()
    self.target = None           # None: every request; else the index of the one request stalled
    self.req = None              # index of the request being enqueued
    self.fired = collections.Counter()
    self.streams = {}            # cuda_stream -> point stalled after every wait_event of the stream
    self.events = {}             # (cuda_stream, id(event)) -> point stalled after that wait
    self.drop = set()            # (cuda_stream, id(event)) waits a control skips
    self.drop_sync = set()       # id(event) host waits a control skips
    self.dropped = 0

  def stall(self, point, stream=None):
    if point not in self.points or torch.cuda.is_current_stream_capturing():
      return
    if self.target is not None and self.req != self.target:
      return
    self.fired[point] += 1
    with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
      torch.cuda._sleep(STALL_CYCLES)


H = _Harness()
_wait_event = torch.cuda.Stream.wait_event
_event_sync = torch.cuda.Event.synchronize


def _wait_event_stalled(stream, event):
  key = (stream.cuda_stream, id(event))
  if key in H.drop:
    H.dropped += 1
    return None
  _wait_event(stream, event)
  point = H.streams.get(stream.cuda_stream) or H.events.get(key)
  if point:
    H.stall(point, stream)
  return None


def _event_sync_dropped(event):
  if id(event) in H.drop_sync:
    H.dropped += 1
    return
  _event_sync(event)


def _stalling(point, fn):
  @functools.wraps(fn)
  def wrapper(*args, **kwargs):
    H.stall(point)
    return fn(*args, **kwargs)
  return wrapper


class _StalledGraph(object):
  def __init__(self, graph, point):
    self._graph, self._point = graph, point

  def replay(self):
    H.stall(self._point)
    self._graph.replay()


@pytest.fixture(autouse=True)
def harness(monkeypatch):
  from automl_b200 import ops, parallel
  from automl_b200.engine import Engine
  from automl_b200.efficientnetv2.effnetv2_model import EffNetV2Model
  H.__init__()
  monkeypatch.setattr(torch.cuda.Stream, 'wait_event', _wait_event_stalled)
  monkeypatch.setattr(torch.cuda.Event, 'synchronize', _event_sync_dropped)
  for name in ('preprocess', 'preprocess_ragged', 'preprocess_mirrored', 'cls_preprocess'):
    monkeypatch.setattr(ops, name, _stalling('preprocess', getattr(ops, name)))
  for name in ('seg_masks', 'per_class_nms', 'wbf', 'softmax_topk'):
    monkeypatch.setattr(ops, name, _stalling(name, getattr(ops, name)))
  monkeypatch.setattr(parallel, 'gather_detections', _stalling('after_nms', parallel.gather_detections))
  replay, graph_for, run = Engine._replay, Engine._graph_for, EffNetV2Model.run

  def stalled_replay(self, key, fn, capture_stream=None):
    H.stall(key if isinstance(key, str) else key[0])
    return replay(self, key, fn, capture_stream)

  def stalled_graph_for(self, key, fn, capture_stream=None, warm=True):
    g = graph_for(self, key, fn, capture_stream, warm)
    name = key if isinstance(key, str) else key[0]
    return _StalledGraph(g, name) if name in ('net', 'net+pre') else g

  def stalled_run(self):
    H.stall('run')
    return run(self)
  monkeypatch.setattr(Engine, '_replay', stalled_replay)
  monkeypatch.setattr(Engine, '_graph_for', stalled_graph_for)
  monkeypatch.setattr(EffNetV2Model, 'run', stalled_run)
  yield H
  torch.cuda.synchronize()
  H.__init__()


def _main():
  return torch.cuda.current_stream().cuda_stream


def _watch_engine(eng):
  """torch hands out streams from a fixed pool, round robin, so a branch stream can be the very
  CUDA stream of another role: branch streams are watched only where they run work (eager
  engines; replayed graphs fork inside the graph), and before the named streams, which win."""
  if not eng.use_cuda_graph:
    for st in eng._branch_streams.values():                        # pylint: disable=protected-access
      H.streams[st.cuda_stream] = 'branch'
  H.streams[eng._nms_stream.cuda_stream] = 'nms'                   # pylint: disable=protected-access


def _watch_driver(drv):
  for eng in drv._engines.values():                                # pylint: disable=protected-access
    _watch_engine(eng)
  H.streams[drv._copy_stream.cuda_stream] = 'h2d'                  # pylint: disable=protected-access
  H.streams[drv._d2h_stream.cuda_stream] = 'd2h'                   # pylint: disable=protected-access


def _indexed(requests):
  """Yields the requests, recording the index of the one being enqueued for the stall points."""
  for i, r in enumerate(requests):
    H.req = i
    yield r


def _stalled(points, target, run):
  """run() with `points` stalled on request `target` (None: every request); every point must fire."""
  H.points, H.target = set(points), target
  H.fired.clear()
  try:
    out = run()
    torch.cuda.synchronize()
  finally:
    H.points, H.target = set(), None
  missing = [p for p in points if not H.fired[p]]
  assert not missing, 'stall points that never fired: %s (fired: %s)' % (missing, dict(H.fired))
  return out


def _same(a, b):
  """Bit-for-bit equality of results: arrays, tensors and (nested) lists or tuples of them."""
  if isinstance(a, (list, tuple)) or isinstance(b, (list, tuple)):
    return (isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)) and len(a) == len(b)
            and all(_same(x, y) for x, y in zip(a, b)))
  a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
  b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
  return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _mismatches(got, want):
  assert len(got) == len(want)
  return [i for i, (g, w) in enumerate(zip(got, want)) if not _same(g, w)]


def _expect_caught(run, drop=(), drop_sync=()):
  """A control: `run` (a stall case returning its mismatches) with the waits `drop` [(stream,
  event)] and the host waits `drop_sync` [event] skipped must report a mismatch."""
  H.drop = {(s.cuda_stream, id(e)) for s, e in drop}
  H.drop_sync = {id(e) for e in drop_sync}
  try:
    bad = run()
  finally:
    torch.cuda.synchronize()
    H.drop, H.drop_sync = set(), set()
  assert H.dropped, 'the wait the control drops was never reached'
  assert bad, ('dropping the wait went unnoticed: the stall is too short or the workload does not '
               'reach the hand-off')


def _images(rng, shapes):
  return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes]


def _pinned(rng, shape, n):
  return torch.from_numpy(np.stack(_images(rng, [shape] * n))).pin_memory()


def _on_device(rng, shape, n):
  return torch.from_numpy(np.stack(_images(rng, [shape] * n))).to(DEV)


@pytest.fixture(scope='module')
def cache():
  """Drivers and models of this file, each built and served alone once (graphs captured)."""
  built = {}
  yield built
  built.clear()
  torch.cuda.synchronize()


def _cached(cache, key, build):
  if key not in cache:
    cache[key] = build()
  return cache[key]


# ---- detection: ServingDriver.serve_stream / submit -----------------------------------------------
MODES = {   # EDET_* settings the engines are built with, and whether they replay graphs
    'pipelined': ({'EDET_PIPELINE': '1'}, True),
    'sequential': ({'EDET_PIPELINE': '0'}, True),
    'eager': ({'EDET_PIPELINE': '1'}, False),
}
PIPELINED = ('h2d', 'preprocess', 'bb1', 'bb2', 'cell0', 'heads+pre', 'nms', 'after_nms')
DETECTION_POINTS = {
    'pipelined': PIPELINED,
    'sequential': ('h2d', 'preprocess', 'net+pre', 'nms', 'after_nms'),
    'eager': PIPELINED + ('branch',),
}


def _build_driver(mode, batch_size=2, size=128, heads=None):
  from automl_b200 import inference
  env, graphs = MODES[mode]
  mp = {'image_size': size}
  if heads is not None:
    mp['heads'] = heads
  with pytest.MonkeyPatch.context() as m:
    for k, v in env.items():
      m.setenv(k, v)
    if not graphs:
      m.setattr(inference, 'Engine', functools.partial(inference.Engine, use_cuda_graph=False))
    drv = inference.ServingDriver('efficientdet-d0', '_', batch_size=batch_size, model_params=mp)
    drv.build()
  return drv, env, graphs


def _serve_alone(drv, env, graphs, requests, serve=None):
  """Each request served alone and synchronously (engines built on first use get the mode's
  settings); returns the results."""
  from automl_b200 import inference
  with pytest.MonkeyPatch.context() as m:
    for k, v in env.items():
      m.setenv(k, v)
    if not graphs:
      m.setattr(inference, 'Engine', functools.partial(inference.Engine, use_cuda_graph=False))
    out = [(serve or drv.serve_images)(r) for r in requests]
  torch.cuda.synchronize()
  return out


def _detection_requests(rng):
  """Six requests of two images: uniform, ragged, pinned, ragged, on the device, uniform; every one
  at a different scale."""
  return [_images(rng, [(96, 128)] * 2),
          _images(rng, [(200, 150), (64, 90)]),
          _pinned(rng, (100, 160), 2),
          _images(rng, [(300, 240), (128, 128)]),
          _on_device(rng, (80, 200), 2),
          _images(rng, [(192, 144)] * 2)]


def _detection(cache, mode):
  def build():
    drv, env, graphs = _build_driver(mode)
    rng = np.random.default_rng(7)
    reqs = _detection_requests(rng)
    uniform = [_images(rng, [(112, 144)] * 2) for _ in range(6)]
    return drv, reqs, _serve_alone(drv, env, graphs, reqs), uniform, _serve_alone(drv, env, graphs, uniform)
  return _cached(cache, ('detection', mode), build)


def _target(which, n):
  return None if which == 'all' else n // 2


def _run_stream(drv, reqs, want, points, target):
  _watch_driver(drv)
  got = _stalled(points, target, lambda: list(drv.serve_stream(_indexed(reqs))))
  return _mismatches(got, want)


@pytest.mark.parametrize('which', WHICH)
@pytest.mark.parametrize('mode,point', [(m, p) for m, ps in DETECTION_POINTS.items() for p in ps])
def test_detection_stream(cache, mode, point, which):
  """Uniform, ragged, pinned and on-device requests through serve_stream, `point` stalled."""
  drv, reqs, want, _, _ = _detection(cache, mode)
  engines = dict(drv._engines)                                     # pylint: disable=protected-access
  assert _run_stream(drv, reqs, want, [point], _target(which, len(reqs))) == []
  assert drv._engines == engines                                   # pylint: disable=protected-access


@pytest.mark.parametrize('point', ('h2d', 'preprocess', 'bb1', 'nms'))
def test_growing_requests(cache, point):
  """Requests that outgrow every slot's staging buffers, from empty, with `point` stalled."""
  drv, _, _, _, _ = _detection(cache, 'pipelined')
  key = ('growing',)
  if key not in cache:
    rng = np.random.default_rng(17)
    reqs = [_images(rng, [(64, 64)] * 2), _images(rng, [(128, 96), (90, 200)]),
            _pinned(rng, (200, 200), 2), _images(rng, [(300, 400), (256, 256)]),
            _on_device(rng, (400, 300), 2), _images(rng, [(512, 480)] * 2)]
    cache[key] = (reqs, _serve_alone(drv, *MODES['pipelined'], reqs))
  reqs, want = cache[key]
  torch.cuda.synchronize()
  for slots in drv._slots.values():                                # pylint: disable=protected-access
    for slot in slots:
      slot.staging.host = slot.staging.dev = None
  assert _run_stream(drv, reqs, want, [point], None) == []


def _dynamic(cache):
  def build():
    drv, env, graphs = _build_driver('pipelined', batch_size=None)
    rng = np.random.default_rng(27)
    reqs = [_images(rng, [(96, 128)] * 2), _images(rng, [(200, 150), (64, 90), (128, 128)]),
            _pinned(rng, (100, 160), 2), _images(rng, [(300, 240)] * 3),
            _images(rng, [(80, 200), (150, 60)]), _on_device(rng, (192, 144), 3)]
    return drv, reqs, _serve_alone(drv, env, graphs, reqs)
  return _cached(cache, ('dynamic',), build)


@pytest.mark.parametrize('which', WHICH)
@pytest.mark.parametrize('point', PIPELINED)
def test_two_engines_in_flight(cache, point, which):
  """batch_size=None with requests of two and three images alternating: two engines and two slot
  rings in flight at once."""
  drv, reqs, want = _dynamic(cache)
  assert sorted(drv._engines) == [2, 3]                            # pylint: disable=protected-access
  assert _run_stream(drv, reqs, want, [point], _target(which, len(reqs))) == []


# ---- detection, masks and TTA interleaved on one engine -------------------------------------------
BOTH = ['object_detection', 'segmentation']
POINT_KINDS = {   # the request kinds that reach each point
    'h2d': ('det', 'seg', 'tta'), 'preprocess': ('det', 'seg', 'tta'),
    'bb1': ('det',), 'bb2': ('det',), 'cell0': ('det',), 'heads+pre': ('det',), 'nms': ('det',),
    'after_nms': ('det',), 'net': ('seg', 'tta'), 'seg_masks': ('seg',), 'per_class_nms': ('tta',),
    'wbf': ('tta',), 'd2h': ('seg', 'tta'),
}


def _mixed(cache):
  def build():
    drv, env, graphs = _build_driver('pipelined', batch_size=None, size=256, heads=BOTH)
    rng = np.random.default_rng(37)
    det = [_images(rng, [(240, 320), (200, 256), (256, 256), (180, 300)]),
           _pinned(rng, (200, 240), 4),
           _images(rng, [(256, 200)] * 4),
           _images(rng, [(64, 96), (300, 200), (256, 256), (128, 512)])]
    seg = [_images(rng, [(200, 256), (256, 180), (37, 300), (300, 300)]),
           _images(rng, [(120, 160)] * 4),
           _on_device(rng, (160, 240), 4),
           _images(rng, [(99, 77), (256, 256), (200, 100), (64, 64)])]
    tta = [_images(rng, [(256, 200), (64, 96)]), _images(rng, [(240, 320)] * 2),
           _pinned(rng, (180, 256), 2), _images(rng, [(300, 150), (90, 250)])]
    plans = {
        'det-seg-tta': [('det', det[0]), ('seg', seg[0]), ('tta', tta[0]),
                        ('det', det[1]), ('seg', seg[1]), ('tta', tta[1])],
        'tta-seg-det': [('tta', tta[2]), ('seg', seg[2]), ('det', det[2]),
                        ('tta', tta[3]), ('seg', seg[3]), ('det', det[3])],
    }
    serve = {'det': drv.serve_images, 'seg': drv.segment_images, 'tta': drv.serve_images_tta}
    want = {name: _serve_alone(drv, env, graphs, plan, lambda kr: serve[kr[0]](kr[1]))
            for name, plan in plans.items()}
    return drv, plans, want
  return _cached(cache, ('mixed',), build)


def _run_mixed(drv, plan, want, points, target):
  from automl_b200 import staging
  submit = {'det': drv.submit, 'seg': drv.submit_segment, 'tta': drv.submit_tta}
  _watch_driver(drv)
  got = _stalled(points, target, lambda: list(staging.pipelined(
      lambda kr: submit[kr[0]](kr[1]), _indexed(plan), drv.MAX_IN_FLIGHT)))
  return _mismatches(got, want)


@pytest.mark.parametrize('which', WHICH)
@pytest.mark.parametrize('point', sorted(POINT_KINDS))
@pytest.mark.parametrize('order', ('det-seg-tta', 'tta-seg-det'))
def test_mixed_request_kinds(cache, order, point, which):
  """submit, submit_segment and submit_tta interleaved on a both-heads driver under batch_size=None:
  detection requests of four images and TTA requests of two share one engine and its slots."""
  drv, plans, want = _mixed(cache)
  plan = plans[order]
  reach = [i for i, (kind, _) in enumerate(plan) if kind in POINT_KINDS[point]]
  target = None if which == 'all' else reach[len(reach) // 2]
  assert _run_mixed(drv, plan, want[order], [point], target) == []
  assert list(drv._engines) == [4]                                 # pylint: disable=protected-access


# ---- Engine used directly -------------------------------------------------------------------------
PRE = ('boxes', 'scores', 'classes')
ENGINE_POINTS = ('bb1', 'bb2', 'cell0', 'heads+pre', 'nms')
BEHIND = ('forward', 'detect', 'pre_nms_only', 'forward+pre_nms_only')


def _engine(cache):
  def build():
    from automl_b200 import hparams_config, weights
    from automl_b200.arch import DetArch
    from automl_b200.engine import Engine
    c = hparams_config.get_efficientdet_config('efficientdet-d0')
    c.override(dict(image_size=128))
    with pytest.MonkeyPatch.context() as m:
      for k, v in MODES['pipelined'][0].items():
        m.setenv(k, v)
      eng = Engine(c, weights.synthetic_weights(DetArch(c), 3), 2)
    rng = np.random.default_rng(47)
    xs = [torch.from_numpy(rng.uniform(-2, 2, size=(2, 128, 128, 3)).astype(np.float32)).to(DEV)
          for _ in range(8)]
    scales = [torch.tensor([1.0 + 0.25 * k, 0.5 + 0.125 * k], device=DEV) for k in range(8)]
    want = {'steps': [eng.detect(x, s).clone() for x, s in zip(xs, scales)]}
    eng.detect(xs[1], scales[1])
    want['detect'] = eng.detections.clone()
    eng.input.copy_(xs[0])
    eng.image_scales.copy_(scales[0])
    eng.run(postprocess=True)
    want['pre_nms_only'] = [eng.pre_nms_only()[k].clone() for k in PRE]
    cls, box = eng.forward(xs[1])
    want['forward'] = [t.clone() for l in sorted(cls) for t in (cls[l], box[l])]
    eng.forward(xs[1])
    want['forward+pre_nms_only'] = [eng.pre_nms_only()[k].clone() for k in PRE]
    torch.cuda.synchronize()
    return eng, xs, scales, want
  return _cached(cache, ('engine',), build)


def _run_steps(eng, xs, scales, want, points, target):
  """Eight image_scales.copy_() + run(postprocess=True) steps without a host synchronisation, each
  step's detections copied out by its after_nms hook on the NMS stream."""
  _watch_engine(eng)
  outs = [torch.empty_like(eng.detections) for _ in xs]

  def run():
    for k, (x, s) in enumerate(zip(xs, scales)):
      H.req = k
      eng.input.copy_(x)
      eng.image_scales.copy_(s)
      eng.run(postprocess=True, after_nms=lambda det, o=outs[k]: o.copy_(det))
    eng.wait_detections()
    return outs
  return _mismatches(_stalled(points, target, run), want['steps'])


@pytest.mark.parametrize('which', WHICH)
@pytest.mark.parametrize('point', ENGINE_POINTS)
def test_engine_steps(cache, point, which):
  eng, xs, scales, want = _engine(cache)
  assert _run_steps(eng, xs, scales, want, [point], _target(which, len(xs))) == []


def _run_behind(eng, xs, scales, want, call, points):
  """One pipelined step of xs[0], then `call` on xs[1] without a host synchronisation: both must
  equal what they give alone."""
  _watch_engine(eng)
  out = torch.empty_like(eng.detections)

  def run():
    H.req = 0
    eng.input.copy_(xs[0])
    eng.image_scales.copy_(scales[0])
    eng.run(postprocess=True, after_nms=lambda det: out.copy_(det))
    H.req = 1
    if call == 'forward':
      cls, box = eng.forward(xs[1])
      got = [t.clone() for l in sorted(cls) for t in (cls[l], box[l])]
    elif call == 'detect':
      got = eng.detect(xs[1], scales[1]).clone()
    else:
      if call == 'forward+pre_nms_only':
        eng.forward(xs[1])
      ps = eng.pre_nms_only()
      got = [ps[k].clone() for k in PRE]
    eng.wait_detections()
    return [out, got]
  return _mismatches(_stalled(points, None, run), [want['steps'][0], want[call]])


@pytest.mark.parametrize('point', ('cell0', 'heads+pre', 'nms'))
@pytest.mark.parametrize('call', BEHIND)
def test_engine_call_behind_a_stalled_step(cache, call, point):
  """forward(), detect() and pre_nms_only() (of that step, and after a forward()) right behind a
  pipelined step whose stage `point` is stalled."""
  eng, xs, scales, want = _engine(cache)
  assert _run_behind(eng, xs, scales, want, call, [point]) == []


# ---- EffNetV2Model.classify_stream and serve_stream ---------------------------------------------
CLASSIFY_POINTS = ('h2d', 'preprocess', 'run', 'softmax_topk', 'd2h')
SERVE_POINTS = ('h2d', 'run', 'out copy', 'd2h')


def _classifier(cache):
  def build():
    from automl_b200.efficientnetv2 import effnetv2_model
    arch = effnetv2_model.EffNetV2Arch('efficientnet-b0')
    w = effnetv2_model.synthetic_weights(arch, 11, include_top=True)
    model = effnetv2_model.get_model('efficientnet-b0', include_top=True, weights=w, batch_size=2,
                                     image_size=64)
    rng = np.random.default_rng(57)
    reqs = [_images(rng, [(90, 120), (200, 150)]), _pinned(rng, (100, 130), 2),
            _images(rng, [(300, 301), (33, 40)]), _on_device(rng, (140, 100), 2),
            _images(rng, [(90, 90)] * 2), _images(rng, [(64, 200), (120, 64)])]
    want = [model.classify(r, top_k=5) for r in reqs]
    return model, reqs, want
  return _cached(cache, ('classifier',), build)


def _run_classify(model, reqs, want, points, target):
  c = model._cls                                                   # pylint: disable=protected-access
  H.streams[c['copy'].cuda_stream] = 'h2d'
  H.streams[c['d2h'].cuda_stream] = 'd2h'
  got = _stalled(points, target, lambda: list(model.classify_stream(_indexed(reqs), top_k=5)))
  return _mismatches(got, want)


@pytest.mark.parametrize('which', WHICH)
@pytest.mark.parametrize('point', CLASSIFY_POINTS)
def test_classify_stream(cache, point, which):
  model, reqs, want = _classifier(cache)
  assert _run_classify(model, reqs, want, [point], _target(which, len(reqs))) == []


def _pipe_model(cache):
  def build():
    from automl_b200.efficientnetv2 import effnetv2_model
    arch = effnetv2_model.EffNetV2Arch('efficientnetv2-b0')
    w = effnetv2_model.synthetic_weights(arch, 5)
    model = effnetv2_model.get_model('efficientnetv2-b0', weights=w, batch_size=2, image_size=64)
    rng = np.random.default_rng(67)
    batches = [torch.from_numpy(rng.uniform(-1, 1, size=(2, 64, 64, 3)).astype(np.float32)).pin_memory()
               for _ in range(6)]
    want = [model(b).cpu().clone() for b in batches]
    assert len(list(model.serve_stream(batches[:1]))) == 1        # builds the streams and buffers
    torch.cuda.synchronize()
    return model, batches, want
  return _cached(cache, ('serve_stream',), build)


def _watch_pipe(model):
  p = model._pipe                                                  # pylint: disable=protected-access
  H.streams[p['h2d'].cuda_stream] = 'h2d'
  H.streams[p['d2h'].cuda_stream] = 'd2h'
  for ev in p['ev_d2h']:
    H.events[(_main(), id(ev))] = 'out copy'
  return p


def _run_serve(model, batches, want, points, target):
  _watch_pipe(model)
  got = _stalled(points, target, lambda: [r.clone() for r in model.serve_stream(_indexed(batches))])
  return _mismatches(got, want)


@pytest.mark.parametrize('which', WHICH)
@pytest.mark.parametrize('point', SERVE_POINTS)
def test_serve_stream(cache, point, which):
  model, batches, want = _pipe_model(cache)
  assert _run_serve(model, batches, want, [point], _target(which, len(batches))) == []


@pytest.mark.parametrize('point', (None, 'd2h'))
def test_serve_stream_result_held_while_the_next_is_taken(cache, point):
  """serve_stream's results stay valid until two further results have been yielded: a caller that
  keeps result k without copying it, and takes result k+1, still reads result k."""
  model, batches, want = _pipe_model(cache)
  _watch_pipe(model)

  def run():
    held = []
    results = model.serve_stream(_indexed(batches))
    prev = next(results)
    for r in results:
      torch.cuda.synchronize()
      held.append(prev.clone())    # result k, read after result k+1 has been taken
      prev = r
    held.append(prev.clone())
    return held
  got = _stalled([point] if point else [], None, run)
  assert _mismatches(got, want) == []


# ---- controls: each wait dropped once must be seen --------------------------------------------
def _uniform_stream(cache, mode):
  drv, _, _, uniform, want = _detection(cache, mode)
  return drv, drv._engines[2], uniform, want                       # pylint: disable=protected-access


def test_control_preprocess_waits_for_h2d(cache):
  """The pre-process would read the staging buffer before the H2D copy has written it (uniform
  requests: no table rides in the buffer)."""
  drv, _, reqs, want = _uniform_stream(cache, 'pipelined')
  main = torch.cuda.current_stream()
  drop = [(main, s.staging.ev_h2d) for s in drv._slots[2]]         # pylint: disable=protected-access
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['h2d'], None), drop)


def test_control_heads_wait_for_backbone(cache):
  drv, eng, reqs, want = _uniform_stream(cache, 'pipelined')
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['bb2'], None),
                 [(eng._head_stream, eng._ev_bb)])                 # pylint: disable=protected-access


def test_control_heads_wait_for_nms(cache):
  drv, eng, reqs, want = _uniform_stream(cache, 'pipelined')
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['nms'], None),
                 [(eng._head_stream, e) for e in eng._ev_nms])     # pylint: disable=protected-access


def test_control_nms_waits_for_pre_nms(cache):
  drv, eng, reqs, want = _uniform_stream(cache, 'pipelined')
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['heads+pre'], None),
                 [(eng._nms_stream, e) for e in eng._ev_pre])      # pylint: disable=protected-access


def test_control_backbone_waits_for_cell0(cache):
  drv, eng, reqs, want = _uniform_stream(cache, 'pipelined')
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['cell0'], None),
                 [(torch.cuda.current_stream(), eng._ev_head)])    # pylint: disable=protected-access


def test_control_sequential_step_waits_for_nms(cache):
  drv, eng, reqs, want = _uniform_stream(cache, 'sequential')
  main = torch.cuda.current_stream()
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['nms'], None),
                 [(main, e) for e in eng._ev_nms])                 # pylint: disable=protected-access


def test_control_result_waits_for_the_download(cache):
  drv, _, reqs, want = _uniform_stream(cache, 'pipelined')
  _expect_caught(lambda: _run_stream(drv, reqs, want, ['after_nms'], None),
                 drop_sync=[s.ev_done for s in drv._slots[2]])     # pylint: disable=protected-access


def test_control_downloads_wait_for_mask_and_tta_kernels(cache):
  drv, plans, want = _mixed(cache)
  plan = plans['det-seg-tta']
  drop = [(drv._d2h_stream, s.ev_out) for s in drv._slots[4]]      # pylint: disable=protected-access
  _expect_caught(lambda: _run_mixed(drv, plan, want['det-seg-tta'], ['seg_masks', 'wbf'], None), drop)


def test_control_detect_waits_for_nms(cache):
  eng, xs, scales, want = _engine(cache)
  main = torch.cuda.current_stream()
  _expect_caught(lambda: _run_behind(eng, xs, scales, want, 'detect', ['nms']),
                 [(main, e) for e in eng._ev_nms])                 # pylint: disable=protected-access


def test_control_pre_nms_after_forward_waits_for_nms(cache):
  """pre_nms_only() after forward() would rewrite the buffer set the stalled NMS still reads."""
  eng, xs, scales, want = _engine(cache)
  main = torch.cuda.current_stream()
  _expect_caught(lambda: _run_behind(eng, xs, scales, want, 'forward+pre_nms_only', ['nms']),
                 [(main, e) for e in eng._ev_nms])                 # pylint: disable=protected-access


def test_control_pre_nms_waits_for_head_stage(cache):
  eng, xs, scales, want = _engine(cache)
  main = torch.cuda.current_stream()
  _expect_caught(lambda: _run_behind(eng, xs, scales, want, 'pre_nms_only', ['heads+pre']),
                 [(main, e) for e in eng._ev_pre])                 # pylint: disable=protected-access


def test_control_classify_download_waits_for_top_k(cache):
  model, reqs, want = _classifier(cache)
  c = model._cls                                                   # pylint: disable=protected-access
  _expect_caught(lambda: _run_classify(model, reqs, want, ['softmax_topk'], None),
                 [(c['d2h'], s.ev_out) for s in c['slots']])


def test_control_classify_result_waits_for_the_download(cache):
  model, reqs, want = _classifier(cache)
  c = model._cls                                                   # pylint: disable=protected-access
  _expect_caught(lambda: _run_classify(model, reqs, want, ['d2h'], None),
                 drop_sync=[s.ev_d2h for s in c['slots']])


def test_control_serve_stream_copy_waits_for_h2d(cache):
  model, batches, want = _pipe_model(cache)
  p = model._pipe                                                  # pylint: disable=protected-access
  main = torch.cuda.current_stream()
  _expect_caught(lambda: _run_serve(model, batches, want, ['h2d'], None),
                 [(main, e) for e in p['ev_h2d']])


def test_control_serve_stream_download_waits_for_out_copy(cache):
  model, batches, want = _pipe_model(cache)
  p = model._pipe                                                  # pylint: disable=protected-access
  _expect_caught(lambda: _run_serve(model, batches, want, ['out copy'], None),
                 [(p['d2h'], e) for e in p['ev_out']])


def test_control_serve_stream_yields_after_the_download(cache):
  model, batches, want = _pipe_model(cache)
  p = model._pipe                                                  # pylint: disable=protected-access
  _expect_caught(lambda: _run_serve(model, batches, want, ['d2h'], None), drop_sync=p['ev_d2h'])
