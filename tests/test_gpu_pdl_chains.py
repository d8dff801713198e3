"""Programmatic dependent launch (PDL) on real kernel chains: before its griddepcontrol.wait a kernel
reads nothing an upstream kernel writes and writes no global memory (common.cuh, DESIGN.md
section 4).

Every PDL kernel lets the next kernel on the stream start as its first instruction, so the next
kernel's CTAs run their prologue while it is still running.  Kernel tests that fill their inputs
with torch ops never overlap a producer (torch kernels do not trigger early), and the engine tests
re-run identical inputs, so a load or store moved above the wait would pass them.  Here the
neighbour is the library's own pointwise GEMM as an identity copy ([R, 64] fp16, W = I, bias 0, no
activation) pinned to one CTA (max_ctas 1): it walks its rows in increasing order, so it reads and
writes the last rows of its operands at the end of a long run while the other SMs are free for the
next kernel's CTAs.  A torch sleep kernel ahead of the chain keeps the host out of the timing: both
launches are queued before the copy starts.

REGION is one [R, 64] fp16 allocation.  The buffers of the kernel under test (B) are carved from its
tail as typed views, 128-byte aligned.  Each has two seeded contents, OLD (what the view holds before
the chain) and NEW (what the copy writes), both valid inputs of B.  The copy reproduces every 16-bit
half that is a finite fp16 other than -0 (0 + a * 1 is exact and no column meets 0 * NaN), so fp32
payloads have bits 14-15 of their low half cleared and int64 / int32 payloads are non-negative with
0x3FFF3FFF masks.

  - control: the copy writes NEW into a pointwise B's bias, a constant that B reads before its wait;
    B's output must differ from B alone on NEW, or no overlap was observed and the file proves
    nothing;
  - RAW (copy -> B): every upstream-written input of B lives in REGION; B's outputs (guarded by
    sentinels) and the whole of REGION must equal B alone on NEW, bit for bit;
  - WAR (B -> copy): the copy reads REGION, whose tail holds every output and in-out buffer of B
    pre-filled with OLD; B starts right after it; the copy must see OLD;
  - transitive (copy -> M -> reader): M, with buffers of its own, must finish only after the copy
    has (the BiFPN reads backbone outputs many launches later); an unpinned identity copy of REGION's
    tail after M must see NEW;
  - graphs: one RAW, one WAR and one transitive chain per family captured with torch.cuda.graph
    (PDL becomes a programmatic edge), replayed once.
Each RAW and WAR case also checks that it could fail: B on OLD differs from B on NEW, and B changes
every buffer the copy reads back.  Every case runs once."""
import collections

import numpy as np
import pytest
import torch

import plan_settings as ps
from automl_b200 import utils

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
R = 1 << 17                  # REGION rows of 64 halves (128 bytes)
TAIL = 4096                  # rows the transitive reader copies back
SLEEP_CYCLES = 1 << 22       # ~2.5 ms at H100 clocks: the host queues the chain meanwhile
GUARD = 256                  # sentinel elements after every separate output
NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6
B_OPTIONS = ('dw_impl', 'stem_impl', 'sepconv_impl')


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _reset_all(ops):
  ps.reset(ops)
  for opt in B_OPTIONS:
    ops.set_option(opt, 0)


# ---------------------------------------------------------------------------------------------
# payloads whose every 16-bit half the identity copy reproduces
def half16(g, shape, scale=0.5):
  t = (torch.randn(*shape, generator=g) * scale).half()
  t[t == 0] = 0.5                       # -0 would come back as +0
  return t


def float32(g, shape, scale=0.5):
  t = torch.randn(*shape, generator=g) * scale
  return (t.view(torch.int32) & ~0xC000).view(torch.float32)   # low half finite and >= +0


def masked_ints(g, shape, dtype):
  return (torch.randint(0, 1 << 30, shape, generator=g, dtype=torch.int64) & 0x3FFF3FFF).to(dtype)


def sums(g, shape):
  return masked_ints(g, shape, torch.int64)


def payload(g, shape, dtype):
  if dtype == torch.float16:
    return half16(g, shape)
  if dtype == torch.float32:
    return float32(g, shape)
  return masked_ints(g, shape, dtype)


def _bytes(t):
  return t.contiguous().view(-1).view(torch.uint8)


def _nbytes(shape, dtype):
  return int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()


# ---------------------------------------------------------------------------------------------
# cases: buffers and one launch of the kernel under test
Buf = collections.namedtuple('Buf', 'name shape dtype role make')
# role: 'const' (host-written, never in REGION), 'in' (upstream-written input), 'out', 'inout'


def buf(name, shape, dtype=torch.float16, role='in', make=None):
  return Buf(name, tuple(shape), dtype, role, make)


class Case(object):

  def __init__(self, name, bufs, launch, options=None, slot=False):
    self.name, self.bufs, self.launch = name, bufs, launch
    self.options = options or {}
    self.slot = slot             # launches a slot-using kernel (the tiled depthwise check)

  def contents(self, seed):
    """name -> CPU tensor, one seeded content per buffer."""
    g = torch.Generator().manual_seed(seed)
    return {b.name: (b.make(g) if b.make else payload(g, b.shape, b.dtype)) for b in self.bufs}

  def run(self, t):
    """Launches B on the current stream under its options; the caller resets them."""
    ops = _ops()
    for k, v in self.options.items():
      ops.set_option(k, v)
    self.launch(ops, t)


def _pointwise(name, batch, rows, k, nout, act, res=False, per_image=False, w_in_region=False,
               options=None):
  def launch(ops, t):
    ops.pointwise_conv(t['a'], t['w'], t['bias'], t['out'], act, residual=t.get('res'), rows=rows,
                       batch=batch)
  wshape = (batch, nout, k) if per_image else (1, nout, k) if w_in_region else (nout, k)
  wscale = lambda g: half16(g, wshape, 1.0 / k ** 0.5)
  bufs = [buf('a', (batch, rows, k)),
          buf('w', wshape, role='in' if per_image or w_in_region else 'const', make=wscale),
          buf('bias', (nout,), torch.float32, 'const'),
          buf('out', (batch, rows, nout), role='out')]
  if res:
    bufs.append(buf('res', (batch, rows, nout)))
  return Case('pointwise_' + name, bufs, launch, options)


def _fuse(sig, modes, hw, in_hws, channel):
  ops = _ops()
  code = {'same': ops.RS_SAME, 'up': ops.RS_UP, 'down': ops.RS_DOWN}
  n, f = 2, 64
  wts = [0.3 + 0.2 * i for i in range(len(modes))]

  def launch(ops, t):
    specs = [(t['in%d' % i], code[m], (3, 3, 2, 2) if m == 'down' else None, wt)
             for i, (m, wt) in enumerate(zip(modes, wts))]
    ops.fuse_dw(specs, t['taps'], t['out'], SWISH, channel_weights=t.get('cw'))
  bufs = [buf('in%d' % i, (n,) + ih + (f,)) for i, ih in enumerate(in_hws)]
  bufs += [buf('taps', (9, f), torch.float32, 'const'), buf('out', (n,) + hw + (f,), role='out')]
  if channel:
    bufs.append(buf('cw', (len(modes), f), torch.float32, 'const',
                    make=lambda g: torch.rand(len(modes), f, generator=g) / len(modes)))
  return Case('%s_%s' % ('fuse_dw_channel' if channel else 'fuse_dw', sig), bufs, launch)


def _cases():
  """Every PDL entry point and the variants that change its prologue (shapes of the kernel tests,
  which pin the plan each selects)."""
  ops = _ops()
  cases = []
  # stem: tensor-core (stem_tc_kernel) and CUDA-core (stem_kernel)
  for impl in (0, 1):
    cases.append(Case(
        'stem_impl%d' % impl,
        [buf('img', (2, 80, 128, 3), torch.float32), buf('w', (27, 32), role='const'),
         buf('b', (32,), torch.float32, 'const'), buf('out', (2, 40, 64, 32), role='out')],
        lambda ops, t: ops.stem_conv(t['img'], t['out'], t['w'], t['b'], SWISH),
        {'stem_impl': impl}))
  # conv2d k3, stride 1 and 2, with residual
  for s in (1, 2):
    ho, wo = 8 // s, 20 // s
    cases.append(Case(
        'conv2d_k3s%d_res' % s,
        [buf('x', (1, 8, 20, 64)), buf('res', (1, ho, wo, 64)),
         buf('w', (9, 64, 64), make=lambda g: half16(g, (9, 64, 64), 1 / 24.), role='const'),
         buf('b', (64,), torch.float32, 'const'), buf('out', (1, ho, wo, 64), role='out')],
        lambda ops, t, s=s: ops.conv2d(t['x'], t['w'], t['b'], t['out'], SWISH, 3, s,
                                       residual=t['res'])))
  # transposed conv with the skip source
  cases.append(Case(
      'conv2d_transpose_skip',
      [buf('a0', (1, 8, 20, 32)), buf('a1', (1, 8, 20, 32)),
       buf('w', (4, 64, 64), make=lambda g: half16(g, (4, 64, 64), 1 / 16.), role='const'),
       buf('b', (16,), torch.float32, 'const'), buf('out', (1, 16, 40, 16), role='out')],
      lambda ops, t: ops.conv2d_transpose(t['a0'], t['w'], t['b'], t['out'], SWISH, 16, a1=t['a1'])))
  # depthwise: tiled kernel (eligible shape) and register kernel, k 3 and 5, with the SE sum
  for impl, shape in ((0, (1, 80, 80, 128)), (1, (2, 20, 20, 64))):
    for k in (3, 5):
      c = shape[-1]
      cases.append(Case(
          'depthwise_%s_k%d_se' % ('tile' if impl == 0 else 'register', k),
          [buf('x', shape), buf('se', (shape[0], c), torch.int64, 'inout'),
           buf('w', (k * k, c), torch.float32, 'const'), buf('b', (c,), torch.float32, 'const'),
           buf('out', shape, role='out')],
          lambda ops, t, k=k: ops.depthwise_conv(t['x'], t['out'], t['w'], t['b'], SWISH, k, 1,
                                                 se_sum=t['se']),
          {'dw_impl': impl}, slot=impl == 0))
  cases.append(Case(
      'mbconv_expand_dw_se',
      [buf('x', (2, 56, 56, 16)), buf('se', (2, 64), torch.int64, 'inout'),
       buf('we', (64, 16), role='const'), buf('be', (64,), torch.float32, 'const'),
       buf('wd', (9, 64), torch.float32, 'const'), buf('bd', (64,), torch.float32, 'const'),
       buf('out', (2, 56, 56, 64), role='out')],
      lambda ops, t: ops.mbconv_expand_dw(t['x'], t['we'], t['be'], t['wd'], t['bd'], t['out'],
                                          SWISH, 3, 1, se_sum=t['se'])))
  n, c, se, nout = 2, 256, 16, 64
  cases.append(Case(
      'se_fc_wt_zero',
      [buf('sum', (n, c), torch.int64, make=lambda g: sums(g, (n, c))),
       buf('w1', (se, c), torch.float32, 'const', lambda g: torch.randn(se, c, generator=g) / 8),
       buf('b1', (se,), torch.float32, 'const'),
       buf('w2', (se, c), torch.float32, 'const', lambda g: torch.randn(se, c, generator=g) / 2),
       buf('b2', (c,), torch.float32, 'const'), buf('wt', (nout, c), role='const'),
       buf('hidden', (n, se), torch.float32, 'out'), buf('gate', (n, c), torch.float32, 'out'),
       buf('ws', (n, nout, c), role='out'),
       buf('zero', (n, c + 8), torch.int64, 'out', lambda g: sums(g, (n, c + 8)) | 1)],
      lambda ops, t: ops.se_fc(t['sum'], 1.0 / 391, t['w1'], t['b1'], t['w2'], t['b2'], t['gate'],
                               SWISH, t['wt'], t['ws'], t['zero'], hidden=t['hidden'])))
  # pointwise GEMM plans (test_gpu_pointwise_plans / _shared_w)
  cases += [
      _pointwise('resident', 1, 2000, 64, 96, RELU6),
      _pointwise('streamed_res', 1, 700, 672, 192, SWISH, res=True),
      _pointwise('shared_w_res', 1, 700, 672, 192, SWISH, res=True, options={'max_ctas': 3}),
      _pointwise('teams3', 1, 2000, 64, 96, RELU6, options={'pw_teams': 3}),
      _pointwise('resident_res', 1, 1500, 128, 128, NONE, res=True),
      _pointwise('per_image_w', 5, 1000, 136, 200, RELU6, per_image=True),
      _pointwise('se_scaled_w_batch1', 1, 1200, 480, 80, NONE, res=True, w_in_region=True),
  ]
  cols = ops.CLASS_ARGMAX_COLS
  cases.append(Case(
      'class_argmax',
      [buf('a', (2, 8, 8, 64)), buf('w', (cols, 64), role='const'),
       buf('b', (cols,), torch.float32, 'const'), buf('scores', (2, 64), torch.float32, 'out'),
       buf('classes', (2, 64), torch.int32, 'out')],
      lambda ops, t: ops.class_argmax(t['a'], t['w'], t['b'], t['scores'], t['classes'], 0, 1)))
  # BiFPN nodes: every compiled signature, scalar and per-channel fusion weights
  hw, up, down = (13, 9), (7, 5), (25, 17)
  sigs = [('same_up', ('same', 'up'), (hw, up)),
          ('same_same_down', ('same', 'same', 'down'), (hw, hw, down)),
          ('same_down', ('same', 'down'), (hw, down)),
          ('same_same', ('same', 'same'), (hw, hw)),
          ('same_same_up', ('same', 'same', 'up'), (hw, hw, up)),
          ('generic_up_same_down', ('up', 'same', 'down'), (up, hw, down))]
  for channel in (False, True):
    cases += [_fuse(sig, modes, hw, in_hws, channel) for sig, modes, in_hws in sigs]
  for impl in (0, 1, 2):
    cases.append(Case(
        'sepconv_impl%d' % impl,
        [buf('x', (1, 8, 20, 64)), buf('dw', (9, 64), torch.float32, 'const'),
         buf('pw', (64, 64), role='const', make=lambda g: half16(g, (64, 64), 1 / 8.)),
         buf('b', (64,), torch.float32, 'const'), buf('out', (1, 8, 20, 64), role='out')],
        lambda ops, t: ops.sepconv([(t['x'], ops.RS_SAME, None, 1.0)], NONE, t['dw'], t['pw'],
                                   t['b'], t['out'], SWISH),
        {'sepconv_impl': impl}))
  cases.append(Case(
      'max_pool',
      [buf('x', (2, 13, 9, 64)), buf('out', (2, 7, 5, 64), role='out')],
      lambda ops, t: ops.max_pool(t['x'], t['out'], (3, 3), (2, 2))))
  cases.append(Case(
      'global_avg_pool',
      [buf('x', (2, 7, 7, 256)), buf('out', (2, 256), torch.float32, 'out')],
      lambda ops, t: ops.global_avg_pool(t['x'], t['out'])))
  cases.append(Case(
      'dense',
      [buf('x', (2, 256), torch.float32), buf('w', (100, 256), role='const'),
       buf('b', (100,), torch.float32, 'const'), buf('out', (2, 100), torch.float32, 'out')],
      lambda ops, t: ops.dense(t['x'], t['w'], t['b'], t['out'])))
  na, nc = 9, 4
  cases.append(Case(
      'pre_nms_two_levels',
      [buf('c0', (2, 4, 4, 40)), buf('b0', (2, 4, 4, 36)), buf('c1', (2, 2, 2, 40)),
       buf('b1', (2, 2, 2, 36)),
       buf('anchors', (na * 20, 4), torch.float32, 'const',
           lambda g: torch.rand(na * 20, 4, generator=g) * 32),
       buf('boxes', (2, na * 20, 4), torch.float32, 'out'),
       buf('scores', (2, na * 20), torch.float32, 'out'),
       buf('classes', (2, na * 20), torch.int32, 'out')],
      lambda ops, t: ops.pre_nms([t['c0'], t['c1']], [t['b0'], t['b1']], [(4, 4), (2, 2)], na, nc,
                                 t['anchors'], t['boxes'], t['scores'], t['classes'])))
  return cases


def _case_names():
  # names only (no CUDA library needed at collection)
  names = ['stem_impl0', 'stem_impl1', 'conv2d_k3s1_res', 'conv2d_k3s2_res', 'conv2d_transpose_skip',
           'depthwise_tile_k3_se', 'depthwise_tile_k5_se', 'depthwise_register_k3_se',
           'depthwise_register_k5_se', 'mbconv_expand_dw_se', 'se_fc_wt_zero']
  names += ['pointwise_' + p for p in ('resident', 'streamed_res', 'shared_w_res', 'teams3',
                                       'resident_res', 'per_image_w', 'se_scaled_w_batch1')]
  names += ['class_argmax']
  sigs = ('same_up', 'same_same_down', 'same_down', 'same_same', 'same_same_up',
          'generic_up_same_down')
  names += ['fuse_dw_' + s for s in sigs] + ['fuse_dw_channel_' + s for s in sigs]
  names += ['sepconv_impl0', 'sepconv_impl1', 'sepconv_impl2', 'max_pool', 'global_avg_pool',
            'dense', 'pre_nms_two_levels']
  return names


CASE_NAMES = _case_names()
# one configuration of each PDL kernel family (transitive and graph chains)
FAMILY_CASES = ['stem_impl0', 'stem_impl1', 'conv2d_k3s1_res', 'conv2d_transpose_skip',
                'depthwise_tile_k3_se', 'depthwise_register_k3_se', 'mbconv_expand_dw_se',
                'se_fc_wt_zero', 'pointwise_streamed_res', 'class_argmax', 'fuse_dw_same_up',
                'fuse_dw_channel_same_up', 'sepconv_impl0', 'sepconv_impl1', 'sepconv_impl2',
                'max_pool', 'global_avg_pool', 'dense', 'pre_nms_two_levels']


# ---------------------------------------------------------------------------------------------
class Region(object):
  """REGION, its NEW image (the copy's source) and the copy's destination for the WAR chains."""

  def __init__(self):
    g = torch.Generator().manual_seed(1)
    self.t = torch.empty(R, 64, dtype=torch.float16, device=DEV)
    self.src = torch.empty_like(self.t)
    self.dst = torch.empty_like(self.t)
    self.filler = half16(g, (R, 64)).to(DEV)
    self.eye = torch.eye(64, dtype=torch.float16, device=DEV)
    self.zero = torch.zeros(64, dtype=torch.float32, device=DEV)
    # first launches of both copy plans outside any graph capture
    self.slow_copy(self.filler, self.t)
    self.reader(self.dst[:TAIL])
    torch.cuda.synchronize()

  def views(self, image, bufs):
    """name -> typed view of `image` for each of `bufs`, laid out in order, ending at its last row,
    each starting on a 128-byte row."""
    rows = [-(-_nbytes(b.shape, b.dtype) // 128) for b in bufs]
    flat = _bytes(image)
    out, row = {}, R - sum(rows)
    assert row >= R // 2, 'the views must stay in the tail the copy writes last'
    for b, r in zip(bufs, rows):
      nb = _nbytes(b.shape, b.dtype)
      out[b.name] = flat[row * 128:row * 128 + nb].view(b.dtype).view(b.shape)
      row += r
    return out

  def image(self, bufs, contents):
    """A device [R, 64] image: the filler with `bufs` holding `contents`."""
    img = self.filler.clone()
    for name, v in self.views(img, bufs).items():
      v.copy_(contents[name])
    return img

  def slow_copy(self, src, dst):
    """The pinned identity copy src -> dst (both [rows, 64] fp16), one CTA."""
    ops = _ops()
    ops.set_option('max_ctas', 1)
    try:
      ops.pointwise_conv(src, self.eye, self.zero, dst, NONE)
    finally:
      ps.reset(ops)

  def reader(self, dst):
    """An unpinned identity copy of REGION's last TAIL rows into dst."""
    _ops().pointwise_conv(self.t[R - TAIL:], self.eye, self.zero, dst, NONE)


@pytest.fixture(scope='module')
def region():
  return Region()


@pytest.fixture(scope='module')
def cases():
  return {c.name: c for c in _cases()}


def test_case_list_matches(cases):
  assert sorted(cases) == sorted(CASE_NAMES)
  assert set(FAMILY_CASES) <= set(CASE_NAMES)


class Outs(object):
  """Separate buffers, each followed by GUARD sentinel elements."""

  def __init__(self, bufs):
    self.bufs = bufs
    self.mem = {b.name: torch.empty(int(np.prod(b.shape)) + GUARD, dtype=b.dtype, device=DEV)
                for b in bufs}
    self.t = {b.name: self.mem[b.name][:int(np.prod(b.shape))].view(b.shape) for b in bufs}

  def reset(self):
    for m in self.mem.values():
      m.fill_(7)

  def result(self):
    got = {}
    for b in self.bufs:
      m = self.mem[b.name]
      assert bool((m[m.numel() - GUARD:] == 7).all()), '%s: written past its end' % b.name
      got[b.name] = _bytes(self.t[b.name]).cpu()
    return got


def _separate(bufs, contents):
  return {b.name: contents[b.name].to(DEV) for b in bufs}


def _same(a, b):
  return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def _sleep():
  torch.cuda._sleep(SLEEP_CYCLES)


class Raw(object):
  """copy -> B with every upstream-written input of B in REGION."""

  def __init__(self, case, region, upstream_roles=('in', 'inout')):
    self.case, self.region = case, region
    self.up = [b for b in case.bufs if b.role in upstream_roles]
    other = [b for b in case.bufs if b.role not in upstream_roles]
    self.consts = [b for b in other if b.role != 'out']
    self.outs = Outs([b for b in other if b.role == 'out'])
    self.old_c, self.new_c = case.contents(100), case.contents(200)
    self.old = region.image(self.up, self.old_c)
    self.new = region.image(self.up, self.new_c)
    self.t = dict(_separate(self.consts, self.new_c), **self.outs.t)
    self.t.update(region.views(region.t, self.up))

  def result(self):
    got = self.outs.result()
    got['REGION'] = _bytes(self.region.t).cpu()
    return got

  def alone(self, image):
    """B alone with REGION holding `image`."""
    ops = _ops()
    self.region.t.copy_(image)
    self.outs.reset()
    torch.cuda.synchronize()
    slot = ops.last_sched_slot()
    try:
      self.case.run(self.t)
    finally:
      _reset_all(ops)
    torch.cuda.synchronize()
    if self.case.slot:
      assert ops.last_sched_slot() != slot, 'the tiled kernel did not run'
    return self.result()

  def prepare(self):
    self.region.t.copy_(self.old)
    self.region.src.copy_(self.new)
    self.outs.reset()
    torch.cuda.synchronize()

  def chain(self):
    self.region.slow_copy(self.region.src, self.region.t)
    try:
      self.case.run(self.t)
    finally:
      _reset_all(_ops())


def _raw_want(raw):
  want = raw.alone(raw.new)
  assert not _same(raw.alone(raw.old), want), 'B gives the same result on OLD and NEW'
  return want


class War(object):
  """B -> copy: the copy reads REGION, whose tail holds B's outputs and in-out buffers (OLD)."""

  def __init__(self, case, region):
    self.case, self.region = case, region
    self.ys = [b for b in case.bufs if b.role in ('out', 'inout')]
    self.old_c = case.contents(100)
    self.old = region.image(self.ys, self.old_c)
    self.t = _separate([b for b in case.bufs if b.role in ('in', 'const')], case.contents(200))
    self.t.update(region.views(region.t, self.ys))

  def prepare(self):
    self.region.t.copy_(self.old)
    self.region.dst.fill_(7)
    torch.cuda.synchronize()

  def chain(self):
    self.region.slow_copy(self.region.t, self.region.dst)
    try:
      self.case.run(self.t)
    finally:
      _reset_all(_ops())

  def check(self):
    torch.cuda.synchronize()
    assert torch.equal(_bytes(self.region.dst), _bytes(self.old)), \
        'the copy read a value B wrote before its grid-dependency wait'
    after = self.region.views(self.region.t, self.ys)
    for b in self.ys:      # B writes every one of them, so the case can fail
      assert not torch.equal(_bytes(after[b.name]).cpu(), _bytes(self.old_c[b.name])), \
          '%s: B left it unchanged' % b.name


class Transitive(object):
  """copy -> M -> reader: M (buffers of its own) must complete only after the copy has."""

  def __init__(self, case, region):
    self.case, self.region = case, region
    g = torch.Generator().manual_seed(300)
    self.old = region.filler
    self.new = half16(g, (R, 64)).to(DEV)
    contents = case.contents(200)
    self.t = _separate([b for b in case.bufs if b.role != 'out'], contents)
    self.t.update(Outs([b for b in case.bufs if b.role == 'out']).t)
    self.got = torch.empty(TAIL, 64, dtype=torch.float16, device=DEV)

  def prepare(self):
    self.region.t.copy_(self.old)
    self.region.src.copy_(self.new)
    self.got.fill_(7)
    torch.cuda.synchronize()

  def chain(self):
    self.region.slow_copy(self.region.src, self.region.t)
    try:
      self.case.run(self.t)
    finally:
      _reset_all(_ops())
    self.region.reader(self.got)

  def check(self):
    torch.cuda.synchronize()
    assert torch.equal(_bytes(self.got), _bytes(self.new[R - TAIL:])), \
        'a kernel after M read REGION before the copy ahead of M had finished'


# ---------------------------------------------------------------------------------------------
def test_copy_is_exact(region):
  """One synchronised pinned copy reproduces every payload kind bit for bit."""
  g = torch.Generator().manual_seed(5)
  bufs = [buf('h', (300, 64)), buf('f', (700, 32), torch.float32),
          buf('s', (100, 64), torch.int64), buf('i', (100, 64), torch.int32)]
  new = region.image(bufs, {b.name: payload(g, b.shape, b.dtype) for b in bufs})
  region.t.fill_(0)
  region.slow_copy(new, region.t)
  torch.cuda.synchronize()
  assert torch.equal(_bytes(region.t), _bytes(new))


def test_control_overlap_is_observed(region):
  """The copy writes NEW into the bias of a pointwise B, which B reads before its wait (a constant
  in the engine).  B must see OLD, or B never overlapped the copy and no case here can fail.  If
  pointwise_tc ever moves its bias load after the wait, point the control at another pre-wait
  constant (the fuse_dw taps, say)."""
  case = _pointwise('bias_control', 1, 2000, 64, 96, RELU6)
  case.bufs[2] = case.bufs[2]._replace(role='in')          # the bias lives in REGION
  raw = Raw(case, region)
  want = _raw_want(raw)
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  raw.prepare()
  start.record()
  region.slow_copy(region.src, region.t)
  end.record()
  torch.cuda.synchronize()
  print('pinned copy of %d rows: %.3f ms' % (R, start.elapsed_time(end)))
  raw.prepare()
  _sleep()
  raw.chain()
  torch.cuda.synchronize()
  got = raw.result()
  assert not _same(got, want), 'no overlap was observed: B read its bias after the copy finished'
  assert torch.equal(got['REGION'], want['REGION'])


@pytest.mark.parametrize('name', CASE_NAMES)
def test_raw(name, cases, region):
  raw = Raw(cases[name], region)
  want = _raw_want(raw)
  raw.prepare()
  _sleep()
  raw.chain()
  torch.cuda.synchronize()
  got = raw.result()
  for k in want:
    assert torch.equal(got[k], want[k]), \
        '%s differs from B alone on NEW: B read an upstream buffer before its wait' % k


@pytest.mark.parametrize('name', CASE_NAMES)
def test_war(name, cases, region):
  war = War(cases[name], region)
  try:                     # B alone: warms the module and shared-memory attributes
    war.case.run(war.t)
  finally:
    _reset_all(_ops())
  war.prepare()
  _sleep()
  war.chain()
  war.check()


@pytest.mark.parametrize('name', FAMILY_CASES)
def test_transitive(name, cases, region):
  """Ordering the engine relies on whenever a kernel reads a buffer written several launches
  earlier.  On an H100 it held even with max_pool_kernel's wait removed (completion follows
  stream order), so this pins the chain rather than any one kernel's wait; RAW and WAR do that."""
  tr = Transitive(cases[name], region)
  tr.prepare()
  _sleep()
  tr.chain()
  tr.check()


def _graph(chain):
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    chain()
  return g


@pytest.mark.parametrize('name', FAMILY_CASES)
def test_graph_chains(name, cases, region):
  """The RAW, WAR and transitive chains of one family captured as graphs (options set during
  capture) and replayed once each, REGION reset outside the graph."""
  case = cases[name]
  raw = Raw(case, region)
  want = _raw_want(raw)
  g = _graph(raw.chain)
  raw.prepare()
  g.replay()
  torch.cuda.synchronize()
  got = raw.result()
  for k in want:
    assert torch.equal(got[k], want[k]), 'graph RAW: %s differs from B alone on NEW' % k
  del g

  war = War(case, region)
  g = _graph(war.chain)
  war.prepare()
  g.replay()
  war.check()
  del g

  tr = Transitive(case, region)
  g = _graph(tr.chain)
  tr.prepare()
  g.replay()
  tr.check()
