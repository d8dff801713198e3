"""Tile-scheduler slots: launches that can be in flight together never share one.

The persistent kernels with a dynamic tile scheduler (pointwise conv and class arg-max, sepconv,
the tiled depthwise kernel, the tensor-core stem, mbconv_expand_dw) claim work units from a device
counter pair, the launch's slot (tc_common.cuh).  Two launches that share a slot while they run
both skip work units and leave stale output tiles, and can leave the slot dirty for every later
launch on it; nothing faults.  A captured graph keeps its slots for as long as it lives, and the
global pool hands a slot out again 4096 launches later, so every launch list (Engine,
EffNetV2Model) owns a pool with one slot per op (LaunchList._bound).

  a. kernel level: edet_last_sched_slot reports the slot of each slot-using family, unbound launches
     walk the global pool, bound launches take exactly the bound slots and the one beyond the count
     is refused without launching, other kernels take none, and a binding is per thread;
  b. inside one launch list: every op keeps one slot of its own list's pool in the eager passes and
     in every graph, no two ops share one, none escapes to the global pool, and every slot is reset
     after each synchronised run;
  c. engines and a classifier built 4096+ standalone launches apart share no slot with each other or
     with those launches (with the global pool alone they would);
  d. end to end, bit-exact: a dynamic-batch ServingDriver with requests of three sizes in flight, and
     a pipelined Engine next to an EffNetV2Model on another stream, give the results of running
     each request / step alone, and still do afterwards.

Out of scope: graphs captured by hand from standalone ops.* calls.  Those launches are unbound and
take global-pool slots, so such a graph shares its slots with the launches 4096 further on."""
import collections
import threading

import numpy as np
import pytest
import torch

import plan_settings as ps
from automl_b200 import hparams_config, utils, weights
from automl_b200._lib import EdetError
from automl_b200.arch import DetArch

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
POOL = 4096                  # slots of the global pool (kSchedSlots)
SLOT_BYTES = 8               # two uint32 counters
SENTINEL = 7.0
SWISH, NONE = utils.ACT_SWISH, utils.ACT_NONE
# op kinds (op_info) whose launch always takes a slot; depthwise ops take one where the tiled kernel
# is eligible for the shape (the register-tiled kernel takes none)
SLOT_KINDS = ('stem', 'pointwise_tc', 'sepconv_tc', 'mbconv_expand_dw')
SLOT_FAMILIES = ['pointwise', 'class_argmax', 'sepconv', 'depthwise_tile', 'stem', 'mbconv']


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _dev(t):
  return t.to(DEV)


def _slot_launchers():
  """name -> (launch, output tensor) for one small launch of each slot-using family (the shapes of
  test_gpu_persistent_kernels._grid_launchers)."""
  ops = _ops()
  g = torch.Generator().manual_seed(11)
  h16 = lambda *s: _dev((torch.randn(*s, generator=g) * 0.5).half())
  f32 = lambda *s: _dev(torch.randn(*s, generator=g) * 0.5)
  x = h16(2, 40, 64, 64)
  sep_out = torch.empty(2, 40, 64, 64, dtype=torch.float16, device=DEV)
  dw, pw, b = f32(9, 64), h16(64, 64), f32(64)
  img = f32(2, 80, 128, 3)
  stem_out = torch.empty(2, 40, 64, 32, dtype=torch.float16, device=DEV)
  stem_w, stem_b = h16(27, 32), f32(32)
  a = h16(8192, 64)
  a_out = torch.empty(8192, 64, dtype=torch.float16, device=DEV)
  dx = h16(1, 80, 80, 128)
  dx_out = torch.empty(1, 80, 80, 128, dtype=torch.float16, device=DEV)
  dw25, b128 = f32(25, 128), f32(128)
  mx = h16(2, 56, 56, 16)
  mx_out = torch.empty(2, 56, 56, 64, dtype=torch.float16, device=DEV)
  we, wd9 = h16(64, 16), f32(9, 64)
  am = h16(2, 8, 8, 64)
  am_w = h16(ops.CLASS_ARGMAX_COLS, 64)
  am_b = f32(ops.CLASS_ARGMAX_COLS)
  am_scores = torch.empty(2, 64, device=DEV)
  am_classes = torch.empty(2, 64, dtype=torch.int32, device=DEV)
  return {
      'pointwise': (lambda: ops.pointwise_conv(a, pw, b, a_out, SWISH), a_out),
      'class_argmax': (lambda: ops.class_argmax(am, am_w, am_b, am_scores, am_classes, 0, 1),
                       am_scores),
      'sepconv': (lambda: ops.sepconv([(x, ops.RS_SAME, None, 1.0)], NONE, dw, pw, b, sep_out, SWISH),
                  sep_out),
      'depthwise_tile': (lambda: ops.depthwise_conv(dx, dx_out, dw25, b128, SWISH, 5, 1), dx_out),
      'stem': (lambda: ops.stem_conv(img, stem_out, stem_w, stem_b, SWISH), stem_out),
      'mbconv': (lambda: ops.mbconv_expand_dw(mx, we, b, wd9, b, mx_out, SWISH, 3, 1), mx_out),
  }


def _no_slot_launchers():
  """name -> launch, one small launch of each kernel that takes no scheduler slot."""
  ops = _ops()
  g = torch.Generator().manual_seed(12)
  h16 = lambda *s: _dev((torch.randn(*s, generator=g) * 0.5).half())
  f32 = lambda *s: _dev(torch.randn(*s, generator=g) * 0.5)
  x = h16(1, 8, 20, 64)
  y = torch.empty(1, 8, 20, 64, dtype=torch.float16, device=DEV)
  wt9, b, dw = h16(9, 64, 64), f32(64), f32(9, 64)
  a, pw = h16(256, 64), h16(64, 64)
  a_out = torch.empty(256, 64, dtype=torch.float16, device=DEV)
  ct_w = h16(4, 4 * 16, 64)
  ct_out = torch.empty(1, 16, 40, 16, dtype=torch.float16, device=DEV)
  rx = h16(1, 16, 16, 32)                  # 32 channels: below the tiled kernel's 64-channel slice
  ry = torch.empty(1, 16, 16, 32, dtype=torch.float16, device=DEV)
  se_sum = torch.zeros(2, 64, dtype=torch.int64, device=DEV)
  w1, b1, w2 = f32(8, 64), f32(8), f32(8, 64)
  gate = torch.empty(2, 64, device=DEV)
  cls, box = h16(2, 4, 4, 8), h16(2, 4, 4, 8)
  anchors = _dev(torch.rand(16, 4, generator=g) * 32)
  boxes = torch.empty(2, 16, 4, device=DEV)
  scores = torch.empty(2, 16, device=DEV)
  classes = torch.empty(2, 16, dtype=torch.int32, device=DEV)
  det = torch.empty(2, 10, 7, device=DEV)
  sel = torch.empty(2, 10, dtype=torch.int32, device=DEV)
  valid = torch.empty(2, dtype=torch.int32, device=DEV)
  work = torch.empty(ops.nms_work_bytes(2, 16), dtype=torch.uint8, device=DEV)
  return {
      'conv2d': lambda: ops.conv2d(x, wt9, b, y, SWISH, 3, 1),
      'conv2d_transpose': lambda: ops.conv2d_transpose(x, ct_w, b[:16], ct_out, SWISH, 16),
      'pointwise_simt': lambda: ops.pointwise_conv(a, pw, b, a_out, SWISH, impl=ops.PW_SIMT),
      'fuse_dw': lambda: ops.fuse_dw([(x, ops.RS_SAME, None, 1.0)], dw, y, SWISH),
      'depthwise_register': lambda: ops.depthwise_conv(rx, ry, dw[:, :32].contiguous(), None, NONE, 3, 1),
      'se_fc': lambda: ops.se_fc(se_sum, 1.0 / 64, w1, b1, w2, b, gate, SWISH),
      'pre_nms': lambda: ops.pre_nms([cls], [box], [(4, 4)], 1, 8, anchors, boxes, scores, classes),
      'nms_v5': lambda: ops.nms_v5(boxes, scores, classes, None, 0, 10, 0.5, float('-inf'), 0.0,
                                   (32.0, 32.0), det, sel, valid, work),
  }


class Standalone(object):
  """Unbound stem launches (global-pool slots) whose output is checked every time: each one must
  cover its whole output even while graphs replay on other streams."""

  def __init__(self):
    ops = _ops()
    g = torch.Generator().manual_seed(8)
    self.x = _dev(torch.randn(1, 16, 40, 3, generator=g))            # 2 stem tiles
    self.w = _dev((torch.randn(27, 32, generator=g) * 0.3).half())
    self.b = _dev(torch.randn(32, generator=g))
    self.out = torch.empty(1, 8, 20, 32, dtype=torch.float16, device=DEV)
    ops.stem_conv(self.x, self.out, self.w, self.b, SWISH)
    self.want = self.out.clone()
    self.bad = torch.zeros((), dtype=torch.bool, device=DEV)
    self.slots = set()

  def launch(self, count):
    ops = _ops()
    for _ in range(count):
      self.out.fill_(SENTINEL)
      ops.stem_conv(self.x, self.out, self.w, self.b, SWISH)
      self.slots.add(ops.last_sched_slot())
      self.bad |= (self.out != self.want).any()

  def check(self):
    torch.cuda.synchronize()
    assert not bool(self.bad), 'a standalone launch skipped tiles'


@pytest.fixture(scope='module')
def global_slots():
  """Every slot of the global pool: POOL consecutive unbound launches."""
  s = Standalone()
  s.launch(POOL)
  s.check()
  assert len(s.slots) == POOL
  return s.slots


@pytest.fixture
def pinned_grid():
  """max_ctas = 8 from before the first launch of a test's lists (the grids are baked into the
  graphs): every persistent kernel walks many tiles per CTA and runs long."""
  ops = _ops()
  ops.set_option('max_ctas', 8)
  try:
    yield
  finally:
    ps.reset(ops)


class Recorder(object):
  """Wraps every stored op of a launch list so that it reads the slot hook after its call: the
  slots each op takes in eager passes and while being captured into a graph."""

  def __init__(self, model):
    self.model = model
    self.seen = collections.defaultdict(set)     # op index -> slots (None: no slot-using launch)
    for i, (name, fn) in enumerate(model._ops):
      model._ops[i] = (name, self._wrap(i, fn))

  def _wrap(self, i, fn):
    ops = _ops()

    def run():
      before = ops.last_sched_slot()
      fn()
      after = ops.last_sched_slot()
      self.seen[i].add(after if after != before else None)
    return run

  def slots(self):
    return {s for v in self.seen.values() for s in v if s is not None}

  def check(self, global_slots=()):
    """Each op: one slot for its whole life, slot i of the list's own pool if its kind takes one;
    no two ops share a slot; no op took a global-pool slot."""
    m = self.model
    pool = m._sched_slots
    assert pool is not None and tuple(pool.shape) == (len(m._ops), 2)
    base = pool.data_ptr()
    owner = {}
    for i, info in enumerate(m.op_info):
      seen = self.seen[i]
      kind = info['kind']
      if not seen:      # the stored pre-NMS / NMS ops run only under profile_ops()
        assert kind not in SLOT_KINDS, 'op %s never ran' % info['name']
        continue
      assert len(seen) == 1, (info['name'], kind, sorted(map(str, seen)))
      slot = next(iter(seen))
      if kind in SLOT_KINDS:
        assert slot is not None, '%s (%s) took no slot or the previous op\'s' % (info['name'], kind)
      elif not kind.startswith('depthwise_'):
        assert slot is None, '%s (%s) took a slot' % (info['name'], kind)
      if slot is None:
        continue
      assert slot == base + SLOT_BYTES * i, (info['name'], hex(slot), hex(base))
      assert slot not in owner, (info['name'], owner.get(slot))
      assert slot not in global_slots, info['name']
      owner[slot] = info['name']
    assert owner

  def check_pool_clean(self):
    torch.cuda.synchronize()
    pool = self.model._sched_slots.cpu()
    assert not bool(pool.any()), 'slots left dirty: %s' % (
        [self.model.op_info[i]['name'] for i in torch.nonzero(pool.any(dim=1)).flatten().tolist()])


def _det_config(image_size=128, heads=None):
  c = hparams_config.get_efficientdet_config('efficientdet-d0')
  c.override(dict(image_size=image_size) if heads is None else dict(image_size=image_size, heads=heads))
  return c


def _images(seed, n, hw=(128, 128)):
  x = np.random.default_rng(seed).uniform(-2.0, 2.0, size=(n,) + tuple(hw) + (3,))
  return torch.from_numpy(x.astype(np.float32)).to(DEV)


def _effnet(batch, image_size=64):
  from automl_b200.efficientnetv2 import effnetv2_model
  return effnetv2_model.get_model('efficientnetv2-b0', include_top=True, batch_size=batch,
                                  image_size=image_size)


# ---- a. kernel level --------------------------------------------------------------------------
def test_unbound_launches_walk_the_global_pool(global_slots):
  ops = _ops()
  for name, (fn, _) in _slot_launchers().items():
    fn()
    first = ops.last_sched_slot()
    assert first in global_slots, name
    got = [first]
    for _ in range(3):
      fn()
      got.append(ops.last_sched_slot())
    for a, b in zip(got, got[1:]):
      assert (b - a) % (POOL * SLOT_BYTES) == SLOT_BYTES, (name, [hex(s) for s in got])
  torch.cuda.synchronize()


@pytest.mark.parametrize('name', SLOT_FAMILIES)
def test_bound_launch_takes_the_bound_slot_and_the_next_is_refused(name, global_slots):
  ops = _ops()
  fn, out = _slot_launchers()[name]
  fn()
  want = out.clone()
  pool = torch.zeros(4, 2, dtype=torch.int32, device=DEV)
  torch.cuda.synchronize()
  slot = pool.data_ptr() + SLOT_BYTES
  try:
    out.fill_(SENTINEL)
    ops.sched_bind(slot, 1)
    fn()
    assert ops.last_sched_slot() == slot
    torch.cuda.synchronize()
    assert torch.equal(out, want), 'bound launch differs from the unbound one'
    out.fill_(SENTINEL)
    with pytest.raises(EdetError, match='slot'):
      fn()
    assert ops.last_sched_slot() == slot
  finally:
    ops.sched_bind(None)
  torch.cuda.synchronize()
  assert bool((out == SENTINEL).all()), 'the refused launch wrote its output'
  assert not bool(pool.any()), 'the bound slot was not reset'
  fn()                                                         # unbound again: the global pool
  assert ops.last_sched_slot() in global_slots


def test_bind_arguments():
  ops = _ops()
  pool = torch.zeros(2, dtype=torch.int32, device=DEV)
  with pytest.raises(EdetError):
    ops.sched_bind(pool.data_ptr(), 0)
  with pytest.raises(EdetError):
    ops.sched_bind(pool.data_ptr() + 4, 1)
  ops.sched_bind(None)


def test_kernels_without_a_scheduler_take_no_slot():
  ops = _ops()
  stem, _ = _slot_launchers()['stem']
  for name, fn in _no_slot_launchers().items():
    stem()
    before = ops.last_sched_slot()
    assert before
    fn()
    assert ops.last_sched_slot() == before, name
  ops.set_option('stem_impl', 1)             # the CUDA-core stem
  try:
    before = ops.last_sched_slot()
    stem()
    assert ops.last_sched_slot() == before
  finally:
    ops.set_option('stem_impl', 0)
  torch.cuda.synchronize()


def test_binding_is_per_thread(global_slots):
  ops = _ops()
  fn, out = _slot_launchers()['stem']
  fn()
  want = out.clone()
  pool = torch.zeros(1, 2, dtype=torch.int32, device=DEV)
  torch.cuda.synchronize()
  seen = {}

  def other():
    seen['before'] = ops.last_sched_slot()
    fn()
    seen['after'] = ops.last_sched_slot()
    torch.cuda.synchronize()

  try:
    ops.sched_bind(pool.data_ptr(), 1)
    t = threading.Thread(target=other)
    t.start()
    t.join()
    fn()                                     # the binding of this thread is still unused
    assert ops.last_sched_slot() == pool.data_ptr()
  finally:
    ops.sched_bind(None)
  assert seen['before'] == 0                 # the hook is per thread too
  assert seen['after'] in global_slots
  torch.cuda.synchronize()
  assert torch.equal(out, want)
  assert not bool(pool.any())


# ---- b. one launch list -------------------------------------------------------------------------
@pytest.mark.parametrize('pipeline', [False, True], ids=['single_graph', 'pipelined'])
def test_engine_ops_keep_their_own_slots(pipeline, global_slots):
  from automl_b200.engine import Engine
  c = _det_config()
  eng = Engine(c, weights.synthetic_weights(DetArch(c), 0), 2, pipeline=pipeline)
  rec = Recorder(eng)
  x = _images(1, 2)
  eng.forward(x)
  rec.check_pool_clean()
  for _ in range(3):                         # both post-processing buffer sets, then a replay
    eng.detect(x)
    rec.check_pool_clean()
  eng.profile_ops(iters=1)
  rec.check_pool_clean()
  if pipeline:
    want = {'net', 'bb1', 'bb2', 'cell0', ('heads+pre', 0), ('heads+pre', 1)}
  else:
    want = {'net', ('net+pre', 0), ('net+pre', 1)}
  assert want <= set(eng._graph), sorted(map(str, eng._graph))
  rec.check(global_slots)


def test_segmentation_twin_ops_keep_their_own_slots(global_slots):
  from automl_b200.engine import Engine
  c = _det_config(heads=['object_detection', 'segmentation'])
  eng = Engine(c, weights.synthetic_weights(DetArch(c), 0), 2)
  rec = Recorder(eng)
  x = _images(2, 2)
  eng.forward(x)
  rec.check_pool_clean()
  for _ in range(2):
    eng.detect(x)
    rec.check_pool_clean()
  assert any(i['kind'] == 'conv_transpose_tc' for i in eng.op_info)
  rec.check(global_slots)


def test_effnetv2_ops_keep_their_own_slots(global_slots):
  model = _effnet(2)
  rec = Recorder(model)
  x = _images(3, 2, (64, 64))
  for _ in range(3):                         # eager + capture, then replays
    model(x)
    rec.check_pool_clean()
  rec.check(global_slots)


# ---- c. lists built apart, no concurrency ------------------------------------------------------
def test_lists_built_thousands_of_launches_apart_share_no_slot():
  from automl_b200.engine import Engine
  c = _det_config()
  w = weights.synthetic_weights(DetArch(c), 0)
  standalone = Standalone()
  recs = {}
  for name, n in (('engine_1', 1), ('engine_2', 2)):
    eng = Engine(c, w, n)
    recs[name] = Recorder(eng)
    eng.forward(_images(4, n))
    eng.detect(_images(5, n))
    torch.cuda.synchronize()
    standalone.launch(POOL + 1)
  model = _effnet(2)
  recs['effnetv2'] = Recorder(model)
  model(_images(6, 2, (64, 64)))
  torch.cuda.synchronize()
  standalone.check()
  sets = {k: r.slots() for k, r in recs.items()}
  sets['standalone'] = standalone.slots
  names = sorted(sets)
  for i, a in enumerate(names):
    assert sets[a], a
    for b in names[i + 1:]:
      shared = sets[a] & sets[b]
      assert not shared, '%s and %s share %d slot(s)' % (a, b, len(shared))


# ---- d. concurrency, end to end ----------------------------------------------------------------
def test_dynamic_batch_serving_with_requests_in_flight(pinned_grid):
  """Requests of 1, 2 and 3 images through one ServingDriver(batch_size=None), three in flight,
  4096+ standalone launches before each engine build: every result equals the request served
  alone, and serving each alone again afterwards still does."""
  from automl_b200 import inference
  rng = np.random.default_rng(7)
  sizes = [1, 2, 3, 2, 1, 3, 3, 1, 2]
  reqs = [[rng.integers(0, 256, size=(96, 128, 3), dtype=np.uint8) for _ in range(n)] for n in sizes]
  params = {'image_size': 128}
  ref_drv = inference.ServingDriver('efficientdet-d0', '_', batch_size=None, model_params=params)
  want = [ref_drv.serve_images(r) for r in reqs]
  drv = inference.ServingDriver('efficientdet-d0', '_', batch_size=None, model_params=params)
  standalone = Standalone()
  handles, built = [], set()
  for r in reqs:
    if built and len(r) not in built:
      standalone.launch(POOL + 1)          # while the earlier requests are in flight
    built.add(len(r))
    handles.append(drv.submit(r))
  got = [h.result() for h in handles]
  standalone.check()
  for i, (g, w_) in enumerate(zip(got, want)):
    np.testing.assert_array_equal(g, w_, err_msg='request %d (%d images) in flight' % (i, sizes[i]))
  for i, r in enumerate(reqs):
    np.testing.assert_array_equal(drv.serve_images(r), want[i],
                                  err_msg='request %d served alone afterwards' % i)


def test_engine_and_classifier_on_two_streams(pinned_grid):
  """A pipelined detection Engine and an EffNetV2Model replay several steps each on their own
  stream with no synchronisation between them (the classifier's graph captured 4096+ standalone
  launches after the engine's): every step equals the sequential run, and so does each alone
  afterwards."""
  from automl_b200.engine import Engine
  c = _det_config()
  eng = Engine(c, weights.synthetic_weights(DetArch(c), 0), 2)
  model = _effnet(4, 128)
  steps = 4
  xe = [_images(20 + k, 2) for k in range(steps)]
  xm = [_images(40 + k, 4) for k in range(steps)]

  def alone():
    dets = [eng.detect(x).cpu().clone() for x in xe]
    standalone.launch(POOL + 1)
    outs = [model(x).cpu().clone() for x in xm]
    return dets, outs

  standalone = Standalone()
  want_det, want_out = alone()              # also builds every graph
  s_e, s_m = torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)
  got_det = [torch.empty_like(eng.detections) for _ in range(steps)]
  got_out = [torch.empty_like(model.output) for _ in range(steps)]
  torch.cuda.synchronize()
  for k in range(steps):
    with torch.cuda.stream(s_e):
      eng.set_input(xe[k])
      eng.run(postprocess=True, after_nms=lambda det, k=k: got_det[k].copy_(det))
    with torch.cuda.stream(s_m):
      model.input.copy_(xm[k])
      model.run()
      got_out[k].copy_(model.output)
  with torch.cuda.stream(s_e):
    eng.wait_detections()
  torch.cuda.synchronize()
  for k in range(steps):
    assert torch.equal(got_det[k].cpu(), want_det[k]), 'engine step %d' % k
    assert torch.equal(got_out[k].cpu(), want_out[k]), 'classifier step %d' % k
  again_det, again_out = alone()
  standalone.check()
  for k in range(steps):
    assert torch.equal(again_det[k], want_det[k]), 'engine step %d alone afterwards' % k
    assert torch.equal(again_out[k], want_out[k]), 'classifier step %d alone afterwards' % k
