"""The memory-bound kernels of every forward pass -- depthwise convolution (edet_depthwise_conv: the
register-tiled kernel of depthwise.cu and the persistent TMA-tiled kernel of depthwise_tile.cu, both
with the fused SE squeeze), the squeeze-excite FCs (edet_se_fc) and the BiFPN node
(edet_fuse_dw, edet_fuse_dw_channel, edet_max_pool) -- against float64 references at every layer
shape of the registered models, with the harness of test_gpu_persistent_kernels.py: one fp16 ulp
plus 5e-5 (check_close), NaN / sentinel guards around every input and output, bit-identical
repeats and, for the persistent kernel, every pinned grid.

The registry functions (dw_shapes, se_shapes, fpn_shapes, pool_shapes) and the tests that the case
lists cover them need no GPU; every other test is marked gpu on its own."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from automl_b200 import arch
from automl_b200 import hparams_config
from automl_b200 import utils
from automl_b200._lib import EdetError
from automl_b200.efficientnetv2 import effnetv2_model
from oracle import efficientdet_oracle as eo
from test_gpu_persistent_kernels import (  # noqa: F401  (the shared harness)
    DEV, GUARD, SENTINEL, V1_MODELS, V2_MODELS, Out, _kernel_grids, carve, check_close, over_grids,
    span_bias)

NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6
U = 2.0**-24                  # fp32 unit roundoff
SE_UNIT = 2.0**-20            # fixed-point unit of the SE squeeze sums
INT_GUARD = 0x5A5A5A5A5A5A5A5A
SWISH_LO = float(np.float32(-20.794415))   # apply_act4 clamps the swish argument here (common.cuh)
DET_MODELS = (sorted(hparams_config.efficientdet_model_param_dict) +
              sorted(hparams_config.efficientdet_lite_param_dict))
# feature-network variants whose node signatures and pools differ from the default BiFPN
FPN_VARIANTS = ((), (('fpn_name', 'qufpn'),), (('conv_after_downsample', True),),
                (('fpn_name', 'qufpn'), ('conv_after_downsample', True)))


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _cdiv(a, b):
  return -(-a // b)


@functools.lru_cache(maxsize=None)
def _det_arch(name, image_size=None, over=()):
  c = hparams_config.get_efficientdet_config(name)
  over = dict(over)
  if image_size is not None:
    over['image_size'] = image_size
  if over:
    c.override(over)
  return arch.DetArch(c)


def _act_code(act_type):
  return {'swish': SWISH, 'silu': SWISH, 'relu6': RELU6}[act_type]


class Buf(object):
  """A device tensor holding `init`, carved from an allocation with GUARD copies of `fill` after
  it: an input read past its end brings `fill` into the result, an output written past its end
  changes one of them."""

  def __init__(self, init, fill):
    self.numel, self.fill = init.numel(), fill
    self.buf = torch.full((self.numel + GUARD,), fill, dtype=init.dtype, device=DEV)
    self.buf[:self.numel] = init.reshape(-1).to(DEV)
    self.t = self.buf[:self.numel].view(init.shape)

  def result(self):
    torch.cuda.synchronize()
    assert bool((self.buf[self.numel:] == self.fill).all()), 'written past the end of the buffer'
    return self.t.cpu()


def _equal(a, b):
  return all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(a, tuple) else torch.equal(a, b)


# ---------------------------------------------------------------------------------------------
# shape registries (no GPU)
def dw_shapes(classifiers=V1_MODELS + V2_MODELS):
  """(k, stride, c, has_se, act) of every depthwise convolution of the registered models: the
  MBConv blocks of EfficientDet D0-D7x and lite0-lite4 (relu6, no SE), the MBConv (conv_type 0)
  blocks of the EfficientNet V1 and V2 classifiers (or those named), and the bias-free 3x3
  depthwise of the head / predict layers (ACT_NONE) at every feature-network width.  Every block
  depthwise has a bias, the head ones none."""
  shapes = set()
  for name in DET_MODELS:
    a = _det_arch(name)
    act = _act_code(a.act_type)
    for b in a.blocks:
      shapes.add((b.kernel_size, b.stride, b.mid_filters, bool(b.se_filters), act))
    shapes.add((3, 1, a.fpn_filters, False, NONE))
  for name in classifiers:
    v = effnetv2_model.EffNetV2Arch(name)
    for b in v.blocks:
      if b.conv_type == 0:
        shapes.add((b.kernel_size, b.strides, b.mid_filters, bool(b.se_filters), v.act))
  return sorted(shapes)


def se_shapes(classifiers=V1_MODELS + V2_MODELS):
  """(c = mid_filters, se, nout = output_filters) of every SE block of the same models."""
  shapes = set()
  for name in DET_MODELS:
    for b in _det_arch(name).blocks:
      if b.se_filters:
        shapes.add((b.mid_filters, b.se_filters, b.output_filters))
  for name in classifiers:
    for b in effnetv2_model.EffNetV2Arch(name).blocks:
      if b.conv_type == 0 and b.se_filters:
        shapes.add((b.mid_filters, b.se_filters, b.output_filters))
  return sorted(shapes)


def _node_signature(a, node):
  """((mode, pool) per input, input sizes) of a feature-network node as the engine lowers it: a
  shrinking resample with a channel change under conv_after_downsample pools and convolves before
  the node, which then reads it as a 'same' input."""
  modes, hws = [], []
  for r in node.inputs:
    if a.conv_after_pool(r):
      modes.append(('same', None))
      hws.append(r.out_hw)
    else:
      modes.append((r.mode, r.pool))
      hws.append(r.in_hw)
  return tuple(modes), tuple(hws)


def _stable_order(registry):
  """The shapes of registry(): those of the detectors and the V2 classifiers first, in their own
  sorted order, then the ones only the V1 classifiers add.  A case's map and batch follow its
  index, so the cases of the earlier shapes stay what they were when the V1 shapes joined."""
  base = registry(V2_MODELS)
  return base + [shape for shape in registry() if shape not in base]


def _pools(a):
  """(channels, pool, input size) of every stand-alone max-pool: the extra P6.. levels (on the
  fpn width, or on the backbone width when conv_after_downsample pools before the 1x1 conv) and
  the conv_after_downsample resamples inside the cells."""
  out = []
  for r in a.extra_levels:
    if r.mode == 'down':
      out.append((r.in_channels if a.conv_after_pool(r) else a.fpn_filters, r.pool, r.in_hw))
  for cell in a.cells:
    for node in cell['nodes']:
      for r in node.inputs:
        if a.conv_after_pool(r):
          out.append((r.in_channels, r.pool, r.in_hw))
  return out


def fpn_shapes():
  """(F, ((mode, pool) per input)) of every node of every detector config at its own image size,
  default BiFPN, QuFPN and conv_after_downsample."""
  shapes = set()
  for name in DET_MODELS:
    for over in FPN_VARIANTS:
      a = _det_arch(name, None, over)
      for cell in a.cells:
        for node in cell['nodes']:
          shapes.add((a.fpn_filters, _node_signature(a, node)[0]))
  return shapes


def pool_shapes():
  """(channels, (pool_h, pool_w, stride_h, stride_w)) of every stand-alone max-pool."""
  return {(c, pool) for name in DET_MODELS for over in FPN_VARIANTS
          for c, pool, _ in _pools(_det_arch(name, None, over))}


# ---------------------------------------------------------------------------------------------
# edet_depthwise_conv
# dwt::Cfg output tile (TOH x TOW) of the TMA-tiled kernel and DwCfg ROWS of the register kernel
DW_TILE = {(3, 1): (16, 16), (3, 2): (8, 8), (5, 1): (8, 16), (5, 2): (8, 8)}
DW_ROWS = {(3, 1): 8, (3, 2): 4, (5, 1): 4, (5, 2): 4}
DW_TW = 4                     # register kernel: output columns per thread
DW_THREADS = 128              # register kernel: threads per block


def dw_tiled(h, w, c, k, s):
  """dwt::eligible restated: the TMA-tiled kernel takes c >= 64 when its fixed output tile covers
  the output map with at least 70 % of the tile's outputs inside it."""
  if c < 64:
    return False
  ho, wo = _cdiv(h, s), _cdiv(w, s)
  th, tw = DW_TILE[(k, s)]
  return ho * wo * 10 >= _cdiv(ho, th) * th * _cdiv(wo, tw) * tw * 7


def dw_partials(ho, wo, c, k, s, tiled):
  """Upper bound on the number of fp32 partial sums rounded to the 2^-20 fixed point that make up
  one (image, channel) SE sum: one per warp and work unit in the tiled kernel; one per block and
  row block in the register kernel (at most every block of a row of x tiles holds the channel)."""
  if tiled:
    th, tw = DW_TILE[(k, s)]
    return 8 * _cdiv(ho, th) * _cdiv(wo, tw)
  return _cdiv(ho, DW_ROWS[(k, s)]) * _cdiv(_cdiv(wo, DW_TW) * (c // 2), DW_THREADS)


# ragged maps the tiled kernel takes (85-91 % of the tile outputs inside the map) and maps it
# leaves to the register kernel (< 70 %), two of each per (k, stride)
TILED_MAPS = {(3, 1): [(31, 45), (47, 29)], (3, 2): [(29, 45), (45, 30)],
              (5, 1): [(15, 29), (29, 45)], (5, 2): [(30, 45), (45, 29)]}
REG_MAPS = {(3, 1): [(9, 37), (6, 61)], (3, 2): [(9, 75), (5, 61)],
            (5, 1): [(7, 37), (5, 61)], (5, 2): [(9, 75), (5, 61)]}
# every (act, bias, SE) combination the two kernels implement
DW_COMBOS = [(SWISH, True, True), (SWISH, True, False), (RELU6, True, False), (RELU6, True, True),
             (NONE, False, False), (NONE, True, False)]


def _reg_map(h, w, c, s):
  """A register-kernel map whose row of x tiles spans at least three 128-thread blocks, so the SE
  block reduction also runs in blocks that start part-way through the channel pairs."""
  return h, max(w, s * (DW_TW * _cdiv(3 * DW_THREADS, c // 2) - 3))


def _dw_cases():
  cases = []
  for i, (k, s, c, se, act) in enumerate(_stable_order(dw_shapes)):
    n = 2 if c <= 512 else 1
    th, tw = TILED_MAPS[(k, s)][i % 2]
    rh, rw = _reg_map(*REG_MAPS[(k, s)][i % 2], c, s)
    assert dw_tiled(th, tw, c, k, s) == (c >= 64) and not dw_tiled(rh, rw, c, k, s)
    cases.append((n, th, tw, c, k, s, act, act != NONE, se))
    cases.append((n, rh, rw, c, k, s, act, act != NONE, se))
  # 1 x 1, 1 x W, H x 1 and maps smaller than one register tile (ROWS x 4 outputs) at both
  # strides, c = 8 (the narrowest legal width) to 264, batch 3 (the image stride)
  widths = (8, 24, 40, 72, 136, 200, 264)
  maps = [(1, 1), (1, 37), (37, 1), (2, 3), (3, 2), (5, 7), (7, 5)]
  i = 0
  for k in (3, 5):
    for s in (1, 2):
      for h, w in maps:
        act, b, se = DW_COMBOS[i % len(DW_COMBOS)]
        cases.append((3 if i % 4 == 3 else 1, h, w, widths[(i // 7 + i) % 7], k, s, act, b, se))
        i += 1
  # every implemented (act, bias, SE) combination on the tiled kernel at batch 3
  for j, ks in enumerate(sorted(TILED_MAPS)):
    for t, (act, b, se) in enumerate(DW_COMBOS):
      h, w = TILED_MAPS[ks][t % 2]
      cases.append((3, h, w, (72, 136, 200, 264)[(j + t) % 4], ks[0], ks[1], act, b, se))
  return cases


DW_CASES = _dw_cases()


def _dw_id(case):
  n, h, w, c, k, s, act, b, se = case
  return 'n%d_%dx%d_c%d_k%ds%d_a%d%s%s_%s' % (n, h, w, c, k, s, act, '_b' if b else '',
                                              '_se' if se else '',
                                              'tile' if dw_tiled(h, w, c, k, s) else 'reg')


def _dw_inputs(case):
  n, h, w, c, k, s, act, has_bias, _ = case
  g = torch.Generator().manual_seed(1000 + 7 * h + 3 * w + c + 11 * k + s + act)
  x = torch.randn(n, h, w, c, generator=g).half()
  taps = torch.randn(k * k, c, generator=g) / k          # genuine fp32 taps [k*k][c]
  assert bool((taps.half().float() != taps).float().mean() > 0.99)
  bias = span_bias(c, g, act != NONE) if has_bias else None
  return x, taps, bias


def depthwise_f64(x, taps, k, s):
  """float64 'SAME' depthwise convolution of NHWC x with taps [k*k][c]: the sum over the taps of
  shifted, strided views of the zero-padded input.  The same values as eo.depthwise_conv2d_same
  (test_depthwise_f64_is_the_oracle), without torch's CPU float64 convolution, which takes
  seconds to minutes per call on some hosts."""
  n, h, w, c = x.shape
  ho, wo = _cdiv(h, s), _cdiv(w, s)
  pt, pb = eo.same_pad_amounts(h, k, s)
  pl, pr = eo.same_pad_amounts(w, k, s)
  xp = torch.nn.functional.pad(x.double(), (0, 0, pl, pr, pt, pb))
  taps = taps.double()
  out = torch.zeros(n, ho, wo, c, dtype=torch.float64)
  for ky in range(k):
    for kx in range(k):
      out += xp[:, ky:ky + (ho - 1) * s + 1:s, kx:kx + (wo - 1) * s + 1:s] * taps[ky * k + kx]
  return out


def _dw_reference(x, taps, bias, act, k, s):
  """float64 NHWC: the activations y (swish with the kernels' argument clamp, which moves values
  below -20.79 by < 2e-8), the pre-activations z and the magnitude m = sum_taps |x w| + |b| of the
  sum behind each output."""
  z = depthwise_f64(x, taps, k, s)
  m = depthwise_f64(x.double().abs(), taps.abs(), k, s)
  if bias is not None:
    z = z + bias.double()
    m = m + bias.double().abs()
  if act == SWISH:
    t = z.clamp(min=SWISH_LO)
    y = t * torch.sigmoid(t)
  elif act == RELU6:
    y = z.clamp(0, 6)
  else:
    y = z
  return y, z, m


def _act_slope(z, act, dz):
  """Bound on |act'| over [z - dz, z + dz] (|swish''| <= 0.5, so dz < 2e-3 moves swish' by less
  than 1e-3)."""
  if act == SWISH:
    sg = torch.sigmoid(z)
    return (sg * (1 + z * (1 - sg))).abs() + 1e-3
  if act == RELU6:
    return ((z > -dz) & (z < 6 + dz)).double()
  return torch.ones_like(z)


def _check_se_sums(sums, y, z, m, act, k, parts, what):
  """sums (int64, 2^-20 fixed point) against the float64 sum of the float64 activations.  Per
  output, to first order: the fp32 depthwise (k*k FMAs from zero, then + bias) is off by
  <= (k*k + 1) u m, scaled by the activation's slope; the approximate swish (ex2 / rcp.approx,
  argument rounded by the log2(e) scaling) adds <= (12 + |z|) u |y|.  Each partial sum then
  takes <= 32 fp32 additions in a thread and <= 32 more in the register kernel's block reduction
  (<= 63 u sum |y|), and is rounded to the fixed point once (half a unit per partial)."""
  dz = (k * k + 1) * U * m
  per_out = _act_slope(z, act, dz) * dz + (63 + (12 + z.abs() if act == SWISH else 0)) * U * y.abs()
  bound = per_out.sum((1, 2)) + parts * SE_UNIT / 2
  err = (sums.double() * SE_UNIT - y.sum((1, 2))).abs()
  bad = ~(err <= bound)
  assert not bool(bad.any()), '%s: SE sum off by %g (bound %g), %d sums outside, first at %s' % (
      what, float(err.max()), float(bound.flatten()[int((err - bound).argmax())]), int(bad.sum()),
      tuple(bad.nonzero()[0].tolist()))


@pytest.mark.gpu
@pytest.mark.parametrize('case', DW_CASES, ids=_dw_id)
def test_depthwise(case):
  """Output within one fp16 ulp of float64 with fp32 taps; the SE sums within the bound of
  _check_se_sums; the tiled kernel gives the same bits under every grid, the register kernel (not
  persistent) on a second run; from a non-zero start the SE sums come out exactly start + the sums
  from zero (they are added to, as the engine's alternating accumulators rely on)."""
  ops = _ops()
  n, h, w, c, k, s, act, _, has_se = case
  x, taps, bias = _dw_inputs(case)
  dx, dt, db = carve(x), carve(taps), carve(bias)
  ho, wo = _cdiv(h, s), _cdiv(w, s)
  tiled = dw_tiled(h, w, c, k, s)

  def launch(start=None):
    out = Out((n, ho, wo, c))
    se = None
    if has_se:
      se = Buf(start if start is not None else torch.zeros(n, c, dtype=torch.int64), INT_GUARD)
    ops.depthwise_conv(dx, out.t, dt, db, act, k, s, se.t if se else None)
    got = out.result()
    return (got, se.result()) if has_se else got

  if tiled:
    res = over_grids(launch)
  else:
    res = launch()
    assert _equal(launch(), res), 'two runs of the register kernel differ'
  got = res[0] if has_se else res
  y, z, m = _dw_reference(x, taps, bias, act, k, s)
  check_close(got, y, _dw_id(case))
  if has_se:
    sums = res[1]
    _check_se_sums(sums, y, z, m, act, k, dw_partials(ho, wo, c, k, s, tiled), _dw_id(case))
    start = torch.randint(-2**40, 2**40, (n, c), generator=torch.Generator().manual_seed(c + h),
                          dtype=torch.int64)
    assert torch.equal(launch(start)[1], start + sums), 'SE sums not added to a non-zero start'


@pytest.mark.gpu
@pytest.mark.parametrize('case', [c for c in DW_CASES if dw_tiled(*c[1:6])], ids=_dw_id)
def test_depthwise_tiled_equals_register_kernel(case):
  """dw_impl = 1 runs the register kernel on a map the tiled kernel takes: the same fp32 arithmetic
  in the same order, so bit-identical fp16 outputs; the SE sums differ only in how the fp32
  partial sums are formed and rounded to 2^-20 (at most one unit per output)."""
  ops = _ops()
  n, h, w, c, k, s, act, _, has_se = case
  x, taps, bias = _dw_inputs(case)
  dx, dt, db = carve(x), carve(taps), carve(bias)
  ho, wo = _cdiv(h, s), _cdiv(w, s)
  res = []
  try:
    for impl in (0, 1):
      ops.set_option('dw_impl', impl)
      out = Out((n, ho, wo, c))
      se = Buf(torch.zeros(n, c, dtype=torch.int64), INT_GUARD) if has_se else None
      ops.depthwise_conv(dx, out.t, dt, db, act, k, s, se.t if se else None)
      res.append((out.result(), se.result() if se else None))
  finally:
    ops.set_option('dw_impl', 0)
  assert torch.equal(res[0][0], res[1][0])
  if has_se:
    assert int((res[0][1] - res[1][1]).abs().max()) <= ho * wo


DW_DISPATCH = [
    # (h, w, c, k, s): each side of the 70 % rule per (k, stride), c < 64, partly live slices
    (23, 16, 64, 3, 1), (22, 16, 64, 3, 1), (31, 45, 40, 3, 1), (31, 45, 336, 3, 1),
    (9, 37, 336, 3, 1), (29, 45, 144, 3, 2), (9, 75, 144, 3, 2), (15, 29, 1392, 5, 1),
    (7, 37, 1392, 5, 1), (30, 45, 2064, 5, 2), (9, 75, 2064, 5, 2), (12, 16, 72, 5, 2),
    (10, 16, 72, 5, 2),
]


def dispatch_mismatches():
  """[(shape, dw_impl, kernel names)] wherever a torch.profiler trace of one depthwise launch does
  not show exactly the kernel dw_tiled names (the register kernel whenever dw_impl = 1)."""
  ops = _ops()
  bad = []
  for h, w, c, k, s in DW_DISPATCH:
    x = torch.randn(1, h, w, c, device=DEV).half()
    out = torch.empty(1, _cdiv(h, s), _cdiv(w, s), c, dtype=torch.float16, device=DEV)
    taps, bias = torch.randn(k * k, c, device=DEV), torch.randn(c, device=DEV)
    fn = lambda: ops.depthwise_conv(x, out, taps, bias, SWISH, k, s)
    fn()
    for impl in (0, 1):
      ops.set_option('dw_impl', impl)
      try:
        names = [name for name, _ in _kernel_grids(fn)]
      finally:
        ops.set_option('dw_impl', 0)
      tiled = impl == 0 and dw_tiled(h, w, c, k, s)
      if not (len(names) == 1 and ('dw_tile_kernel' in names[0]) == tiled and
              ('depthwise_kernel' in names[0]) != tiled):
        bad.append(((h, w, c, k, s), impl, names))
  return bad


@pytest.mark.gpu
def test_depthwise_dispatch_matches_eligible():
  """dw_tiled (the restatement of dwt::eligible the tests rely on) names the kernel a
  torch.profiler trace shows, on both sides of each boundary; dw_impl = 1 always runs the register
  kernel.  The traces are taken in a child process: after a run of profiler sessions in this
  process the next one, test_max_ctas_pins_the_grid's, came back without its kernel records."""
  assert dw_tiled(23, 16, 64, 3, 1) and not dw_tiled(22, 16, 64, 3, 1)
  assert dw_tiled(12, 16, 72, 5, 2) and not dw_tiled(10, 16, 72, 5, 2)    # 6 / 5 of 8 tile rows
  here = os.path.dirname(os.path.abspath(__file__))
  env = dict(os.environ)
  env['PYTHONPATH'] = os.pathsep.join([os.path.dirname(here), here] +
                                      ([env['PYTHONPATH']] if env.get('PYTHONPATH') else []))
  code = ('import test_gpu_memory_bound_kernels as t\n'
          'bad = t.dispatch_mismatches()\n'
          'print(bad)\n'
          'raise SystemExit(1 if bad else 0)\n')
  res = subprocess.run([sys.executable, '-s', '-c', code], cwd=here, env=env, capture_output=True,
                       text=True, timeout=600)
  assert res.returncode == 0, res.stdout + res.stderr[-3000:]


def _dw_refusals():
  cases = []
  for act in (NONE, SWISH, RELU6, utils.ACT_RELU, utils.ACT_HSWISH, utils.ACT_SIGMOID):
    for b in (False, True):
      for se in (False, True):
        if (act, b, se) not in DW_COMBOS:
          cases.append(('act%d%s%s' % (act, '_bias' if b else '', '_se' if se else ''), act, b, se))
  return cases + [('c12', SWISH, True, True), ('k7', SWISH, True, True), ('stride3', SWISH, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize('kernel', ['tile', 'reg'])
@pytest.mark.parametrize('what,act,has_bias,has_se', _dw_refusals(), ids=[r[0] for r in _dw_refusals()])
def test_depthwise_refusals(what, act, has_bias, has_se, kernel):
  """Unimplemented (act, bias, SE) combinations, c % 8 != 0, k = 7 and stride 3 raise on either
  kernel's map; neither the output nor the SE sums nor anything after them changes."""
  ops = _ops()
  c = 12 if what == 'c12' else 136
  k = 7 if what == 'k7' else 3
  s = 3 if what == 'stride3' else 1
  h, w = (31, 45) if kernel == 'tile' else (9, 37)
  if what not in ('c12', 'k7', 'stride3'):
    assert dw_tiled(h, w, c, k, s) == (kernel == 'tile')
  g = torch.Generator().manual_seed(5)
  x = carve(torch.randn(1, h, w, c, generator=g).half())
  taps = carve(torch.randn(k * k, c, generator=g))
  bias = carve(torch.randn(c, generator=g)) if has_bias else None
  out = Out((1, _cdiv(h, s), _cdiv(w, s), c))
  start = torch.randint(-2**40, 2**40, (1, c), generator=g, dtype=torch.int64)
  se = Buf(start, INT_GUARD) if has_se else None
  with pytest.raises(EdetError):
    ops.depthwise_conv(x, out.t, taps, bias, act, k, s, se.t if se else None)
  assert bool((out.result() == SENTINEL).all())
  if se:
    assert torch.equal(se.result(), start)


# ---------------------------------------------------------------------------------------------
# edet_se_fc
SE_WARPS = 8


def se_split(n, c, se):
  """edet_se_fc's host rule restated: warps per output of se_fc1 (1, 2, 4 or 8)."""
  split = 1
  while split < SE_WARPS and n * se * split < 2048 and c // (2 * split) >= 128:
    split *= 2
  return split


def _se_cases():
  """Every registry shape at batch 1, 2, 3 or 5 (1 or 2 for the largest wt_scaled), which reaches
  every split; swish as in the registered models, relu6 on every fifth shape (se_fc1 applies the
  block's activation)."""
  cases = []
  for i, (c, se, nout) in enumerate(_stable_order(se_shapes)):
    n = (1, 2, 3, 5)[i % 4] if nout * c < 10**6 else (1, 2)[i % 2]
    cases.append((n, c, se, nout, RELU6 if i % 5 == 4 else SWISH))
  return cases


SE_CASES = _se_cases()


def _se_id(case):
  n, c, se, nout, act = case
  return 'n%d_c%d_se%d_o%d_a%d_split%d' % (n, c, se, nout, act, se_split(n, c, se))


@pytest.mark.gpu
@pytest.mark.parametrize('case', SE_CASES, ids=_se_id)
def test_se_fc(case):
  """hidden and gate against float64 from the same int64 squeeze sums, each within a bound derived
  from its fp32 dot-product length; wt_scaled within one fp16 ulp of the float64 wt x gate;
  exactly n x zc elements of zero_buf cleared; the same bits on a second run and without wt."""
  ops = _ops()
  n, c, se, nout, act = case
  g = torch.Generator().manual_seed(c * 7 + se + nout + n)
  hw = 391                                         # a 17 x 23 map
  inv_hw = float(np.float32(1.0 / hw))
  means = torch.randn(n, c, generator=g).double() * 0.5 + 0.2
  sums = torch.round(means * hw / SE_UNIT).to(torch.int64)   # realistic 2^-20 fixed-point sums
  w1 = torch.randn(se, c, generator=g) * 2.0 / c**0.5
  b1 = torch.randn(se, generator=g) * 0.5
  w2t = torch.randn(se, c, generator=g) * 2.0 / se**0.5        # [se][c], the conv2d_1 kernel
  b2 = torch.randn(c, generator=g) * 0.5
  wt = (torch.randn(nout, c, generator=g) / c**0.5).half()
  zc = c + 8 * (se % 5)                              # the next block's accumulator width
  dsum = Buf(sums, INT_GUARD)
  dw1, db1, dw2, db2, dwt = carve(w1), carve(b1), carve(w2t), carve(b2), carve(wt)

  def launch(with_wt):
    hidden = Buf(torch.full((n, se), SENTINEL), SENTINEL)
    gate = Buf(torch.full((n, c), SENTINEL), SENTINEL)
    ws = Out((n, nout, c)) if with_wt else None
    zero = Buf(torch.full((n, zc), 123, dtype=torch.int64), INT_GUARD) if with_wt else None
    ops.se_fc(dsum.t, inv_hw, dw1, db1, dw2, db2, gate.t, act, dwt if with_wt else None,
              ws.t if with_wt else None, zero.t if with_wt else None, hidden=hidden.t)
    got = (hidden.result(), gate.result())
    if with_wt:
      assert bool((zero.result() == 0).all()), 'zero_buf not cleared'
      got += (ws.result(),)
    assert dsum.result().equal(sums)
    return got

  hid, gate, ws = launch(True)
  assert _equal(launch(True), (hid, gate, ws)), 'two runs differ'
  assert _equal(launch(False), (hid, gate)), 'gate-only run differs'

  # se_fc1: mean = sum * inv_hw / 2^20, rounded to fp32 (u relative); every product then passes
  # <= ceil(c / 32) FMAs in a lane, 2 adds joining its four accumulators, 5 shuffle adds, <= 8
  # adds joining the split warps and the bias add: <= (ceil(c / 32) + 16 + 1) u sum |w1 mean|
  mean = sums.double() * (np.float64(inv_hw) * SE_UNIT)
  z1 = mean @ w1.double().t() + b1.double()
  e1 = (_cdiv(c, 32) + 17) * U * (mean.abs() @ w1.double().abs().t() + b1.double().abs())
  if act == SWISH:
    h_ref = z1 * torch.sigmoid(z1)
    # act_swish = x / (1 + __expf(-x)): ex2.approx of a rounded x log2(e), fast division
    eh = _act_slope(z1, act, e1) * e1 + (12 + 2 * z1.abs()) * U * h_ref.abs()
  else:
    h_ref = z1.clamp(0, 6)
    eh = _act_slope(z1, act, e1) * e1
  err = (hid.double() - h_ref).abs()
  assert bool((err <= eh).all()), 'hidden off by %g (bound %g)' % (
      float(err.max()), float(eh.flatten()[int((err - eh).argmax())]))
  # se_fc2: b2 starts the first of four accumulators; a product passes <= ceil(se / 4) + 3 FMAs
  # and 2 adds; the hidden errors above propagate through |w2|; sigmoid' <= 1/4; expf (2 ulp)
  # and the division add <= 8 u gate
  z2 = h_ref @ w2t.double() + b2.double()
  e2 = eh @ w2t.double().abs() + (_cdiv(se, 4) + 5) * U * (h_ref.abs() @ w2t.double().abs() + b2.double().abs())
  g_ref = torch.sigmoid(z2)
  eg = 0.25 * e2 + 8 * U * g_ref
  err = (gate.double() - g_ref).abs()
  assert bool((err <= eg).all()), 'gate off by %g (bound %g)' % (
      float(err.max()), float(eg.flatten()[int((err - eg).argmax())]))
  # wt_scaled: the fp32 product rounded to fp16 once
  check_close(ws, wt.double()[None] * g_ref[:, None, :], 'wt_scaled')


# ---------------------------------------------------------------------------------------------
# edet_fuse_dw / edet_fuse_dw_channel / edet_max_pool
# level sizes: an odd image, a non-square one, and one whose P6 and P7 (and D7x's P8) are 1 x 1,
# where BiFPN nodes read two 'same' inputs
FPN_IMAGES = (97, (96, 160), 64)


@functools.lru_cache(maxsize=None)
def _fpn_geometries():
  """(F, modes) -> [(image, node size, input sizes)] and (channels, pool) -> [(image, input
  size)], one entry per image size, from every detector config and variant."""
  nodes, pools = {}, {}
  for image in FPN_IMAGES:
    for name in DET_MODELS:
      for over in FPN_VARIANTS:
        try:
          a = _det_arch(name, image, over)
        except ValueError:    # D7x at (96, 160): P7 1 x 2 -> P8 1 x 1 resamples neither way
          continue
        for cell in a.cells:
          for node in cell['nodes']:
            modes, hws = _node_signature(a, node)
            seen = nodes.setdefault((a.fpn_filters, modes), {})
            seen.setdefault(image, (node.hw, hws))
        for c, pool, hw in _pools(a):
          pools.setdefault((c, pool), {}).setdefault(image, hw)
  return nodes, pools


def _sig_name(modes):
  return '-'.join(m if p is None or p == (3, 3, 2, 2) else '%s%d%d%d%d' % ((m,) + p) for m, p in modes)


def _fuse_cases():
  nodes, _ = _fpn_geometries()
  cases = []
  for (f, modes), per_image in sorted(nodes.items(), key=lambda kv: (kv[0][0], _sig_name(kv[0][1]))):
    for image in FPN_IMAGES:
      if image in per_image and (f, modes) + per_image[image] not in cases:
        hw, in_hws = per_image[image]
        cases.append((f, modes, hw, in_hws))
  # kSigGeneric beyond the registry: one-input nodes, an upsampled input first, non-3 x 3 pools
  s, u = ('same', None), ('up', None)
  cases += [
      (40, (s,), (13, 9), ((13, 9),)),
      (88, (u,), (13, 9), ((7, 5),)),
      (64, (('down', (3, 3, 2, 2)),), (13, 9), ((25, 17),)),
      (88, (u, s, ('down', (3, 3, 2, 2))), (20, 12), ((10, 6), (20, 12), (40, 24))),
      (40, (s, ('down', (2, 2, 2, 2))), (7, 10), ((7, 10), (13, 20))),
      (200, (s, s, ('down', (5, 5, 4, 4))), (5, 3), ((5, 3), (5, 3), (17, 12))),
      (112, (s, ('down', (3, 2, 2, 3))), (6, 5), ((6, 5), (12, 13))),
  ]
  return cases


FUSE_CASES = _fuse_cases()


def _fuse_id(case):
  f, modes, (h, w), in_hws = case
  return 'F%d_%s_%dx%d_from_%s' % (f, _sig_name(modes), h, w, '-'.join('%dx%d' % hw for hw in in_hws))


def _fastattn(raw):
  """Fusion weights as engine.py computes fastattn (scalars) and channel_fastattn (per-channel
  arrays) in float32: relu(w_i) / (sum_j relu(w_j) + 1e-4), summed in input order."""
  ew = [np.maximum(np.asarray(r, np.float32), np.float32(0)) for r in raw]
  tot = ew[0]
  for e in ew[1:]:
    tot = tot + e
  tot = tot + np.float32(0.0001)
  return [e / tot for e in ew]


def carve_inf(t):
  """carve() for inputs that are max-pooled: fmaxf drops NaN, +inf survives."""
  return Buf(t, float('inf')).t


@pytest.mark.gpu
@pytest.mark.parametrize('case', FUSE_CASES, ids=_fuse_id)
def test_fuse_dw(case):
  """One node at every registry (width, signature): scalar fastattn weights and genuine
  per-channel channel_fastattn weights, fp32 taps, swish / relu6 / none; within one fp16 ulp of the
  float64 resample -> weighted sum -> activation -> depthwise 3 x 3, the same bits on a second
  run."""
  ops = _ops()
  f, modes, (h, w), in_hws = case
  n = 2
  idx = FUSE_CASES.index(case)
  act = (SWISH, RELU6, NONE)[idx % 3]
  g = torch.Generator().manual_seed(500 + idx)
  rng = np.random.default_rng(500 + idx)
  code = {'same': ops.RS_SAME, 'up': ops.RS_UP, 'down': ops.RS_DOWN}
  tens = [torch.randn(n, ih, iw, f, generator=g).half() for ih, iw in in_hws]
  taps = torch.randn(9, f, generator=g) / 3
  scalar = _fastattn(rng.uniform(0.1, 1.5, size=len(modes)).astype(np.float32))
  channel = np.stack(_fastattn(rng.uniform(0.1, 1.5, size=(len(modes), f)).astype(np.float32)))
  devs = [carve_inf(t) if m == 'down' else carve(t) for t, (m, _) in zip(tens, modes)]
  dtaps, dch = carve(taps), carve(torch.from_numpy(channel))
  specs = [(d, code[m], pool, float(wt)) for d, (m, pool), wt in zip(devs, modes, scalar)]
  for per_channel in (False, True):
    def launch():
      out = Out((n, h, w, f))
      ops.fuse_dw(specs, dtaps, out.t, act, channel_weights=dch if per_channel else None)
      return out.result()
    got = launch()
    assert torch.equal(launch(), got), 'two runs differ'
    ref = fuse_reference(tens, modes, (h, w), taps, channel if per_channel else scalar, per_channel, act)
    check_close(got, ref, '%s channel=%d' % (_fuse_id(case), per_channel))


def fuse_reference(tens, modes, hw, taps, weights, per_channel, act):
  """float64 NHWC resample -> weighted sum (scalar weights, or [inputs, C] per-channel ones) ->
  activation -> depthwise 3 x 3 of fp16 inputs [N,h,w,F] (nearest and max select fp16 values:
  exact in fp32)."""
  h, w = hw
  res = []
  for t, (m, pool) in zip(tens, modes):
    x = t.float().permute(0, 3, 1, 2)
    x = (x if m == 'same' else eo.resize_nearest_tf1(x, h, w) if m == 'up'
         else eo.max_pool_same(x, pool[:2], pool[2:]))
    res.append(x.permute(0, 2, 3, 1).double())
  if per_channel:
    fused = sum(r * torch.from_numpy(np.asarray(cw, np.float64)) for r, cw in zip(res, weights))
  else:
    fused = sum(r * float(wt) for r, wt in zip(res, weights))
  fused = {SWISH: lambda t: t * torch.sigmoid(t), RELU6: lambda t: t.clamp(0, 6),
           NONE: lambda t: t}[act](fused)
  return depthwise_f64(fused, taps, 3, 1)


def _pool_cases():
  _, pools = _fpn_geometries()
  cases = []
  for (c, pool), per_image in sorted(pools.items()):
    for image in FPN_IMAGES:
      if image in per_image:
        cases.append((c, pool, per_image[image]))
  # other windows (the kernel takes any pool / stride)
  return cases + [(64, (2, 2, 2, 2), (13, 9)), (40, (5, 3, 4, 2), (17, 11)), (8, (3, 3, 1, 1), (5, 1))]


POOL_CASES = _pool_cases()


def _pool_id(case):
  c, pool, (h, w) = case
  return 'c%d_p%d%d%d%d_%dx%d' % ((c,) + pool + (h, w))


@pytest.mark.gpu
@pytest.mark.parametrize('case', POOL_CASES, ids=_pool_id)
def test_max_pool(case):
  """Bit-exact (the max of fp16 values is one of them), +inf after the input, sentinels after the
  output."""
  ops = _ops()
  c, pool, (h, w) = case
  n = 2
  x = torch.randn(n, h, w, c, generator=torch.Generator().manual_seed(c + h + w)).half()
  out = Out((n, _cdiv(h, pool[2]), _cdiv(w, pool[3]), c))
  ops.max_pool(carve_inf(x), out.t, pool[:2], pool[2:])
  got = out.result()
  ref = eo.max_pool_same(x.float().permute(0, 3, 1, 2), pool[:2], pool[2:]).permute(0, 2, 3, 1)
  assert torch.equal(got.float(), ref)


# ---------------------------------------------------------------------------------------------
# the float64 reference and registry coverage (no GPU)
@pytest.mark.parametrize('k,s', sorted(DW_TILE))
def test_depthwise_f64_is_the_oracle(k, s):
  """depthwise_f64 equals eo.depthwise_conv2d_same (TF 'SAME' padding, including the extra pad
  after on odd sizes at stride 2) up to float64 summation order."""
  g = torch.Generator().manual_seed(k * 10 + s)
  for n, h, w, c in [(1, 1, 1, 8), (2, 1, 7, 16), (1, 6, 1, 8), (3, 9, 12, 24), (1, 10, 13, 40)]:
    x = torch.randn(n, h, w, c, generator=g).half()
    taps = torch.randn(k * k, c, generator=g) / k
    ref = eo.depthwise_conv2d_same(x.double().permute(0, 3, 1, 2), taps.double().view(k, k, c, 1), s)
    got = depthwise_f64(x, taps, k, s)
    assert got.shape == (n, _cdiv(h, s), _cdiv(w, s), c)
    assert torch.allclose(got, ref.permute(0, 2, 3, 1), rtol=1e-14, atol=1e-14)


def test_dw_registry_shapes_are_covered():
  shapes = dw_shapes()
  # the shapes where the kernels' index arithmetic has edges: a partly live last 64-channel
  # slice, c not a multiple of 16, channel-pair counts that do not divide the 128-thread block
  assert {c % 64 for _, _, c, _, _ in shapes if c > 64} >= {16, 32, 48}
  assert {40, 56} <= {c for _, _, c, _, _ in shapes}
  assert any(128 % (c // 2) and c // 2 < 128 for _, _, c, _, _ in shapes)
  assert {(k, s) for k, s, _, _, _ in shapes} == set(DW_TILE)
  assert {F for k, s, F, se, act in shapes if act == NONE} == {64, 88, 112, 160, 200, 224, 288, 384}
  # the V1 classifiers' widest maps (efficientnet-l2, -b8)
  assert {(3, 1, 8256, True, SWISH), (5, 1, 4944, True, SWISH), (5, 2, 2880, True, SWISH)} <= set(shapes)
  covered = {}
  for n, h, w, c, k, s, act, b, se in DW_CASES:
    assert b == (act != NONE) or (act, b, se) in DW_COMBOS
    covered.setdefault((k, s, c, se, act), set()).add(dw_tiled(h, w, c, k, s))
  for shape in shapes:
    assert shape in covered, shape
    want = {True, False} if shape[2] >= 64 else {False}
    assert covered[shape] == want, (shape, covered[shape])
  for tiled in (True, False):
    assert {(a, b, se) for case in DW_CASES for (a, b, se) in [case[6:]]
            if dw_tiled(*case[1:6]) == tiled} == set(DW_COMBOS)
  # the register kernel's SE reduction in a block that starts part-way through the channel pairs
  assert any(not dw_tiled(*case[1:6]) and case[8] and 128 % (case[3] // 2) and
             _cdiv(case[2], case[5]) // DW_TW * (case[3] // 2) > 2 * DW_THREADS for case in DW_CASES)


def test_se_registry_shapes_are_covered():
  shapes = se_shapes()
  assert min(se for _, se, _ in shapes) == 4 and max(se for _, se, _ in shapes) == 344
  assert (8256, 344, 1376) in shapes                   # efficientnet-l2 blocks 83-87
  assert any(se % 4 for _, se, _ in shapes)            # se_fc2's tail loop
  assert {(c, se, nout) for _, c, se, nout, _ in SE_CASES} == set(shapes)
  assert {se_split(n, c, se) for n, c, se, _, _ in SE_CASES} == {1, 2, 4, 8}
  # se_fc1 slices that end short of a 32-channel multiple at split > 1
  assert any(se_split(n, c, se) > 1 and c % (32 * se_split(n, c, se)) for n, c, se, _, _ in SE_CASES)


def test_fpn_registry_shapes_are_covered():
  shapes = fpn_shapes()
  assert {f for f, _ in shapes} == {64, 88, 112, 160, 200, 224, 288, 384}
  covered = {(f, modes) for f, modes, _, _ in FUSE_CASES}
  assert covered >= shapes, sorted(shapes - covered)
  for f, modes, (h, w), in_hws in FUSE_CASES:     # input sizes the node accepts
    assert len(in_hws) == len(modes), (f, modes)
    for (m, pool), (ih, iw) in zip(modes, in_hws):
      want = {'same': lambda: (ih, iw) == (h, w), 'up': lambda: ih <= h and iw <= w,
              'down': lambda: (_cdiv(ih, pool[2]), _cdiv(iw, pool[3])) == (h, w)}[m]
      assert want(), (f, modes, (h, w), in_hws)
  # every width meets two 'same' inputs (1 x 1 levels), and each width runs at every image size
  nodes, _ = _fpn_geometries()
  for f in {f for f, _ in shapes}:
    assert (f, (('same', None), ('same', None))) in nodes
  for (f, modes) in shapes:
    assert sum(1 for c in FUSE_CASES if c[:2] == (f, modes)) >= 2, (f, modes)
  assert {(c, p) for c, p, _ in POOL_CASES} >= pool_shapes()
  assert {320, 448} <= {c for c, _ in pool_shapes()}
