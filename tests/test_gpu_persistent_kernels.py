"""The persistent tensor-core kernels of the default paths -- the k x k convolution of the
EfficientNetV2 fused stages (edet_conv2d), the fused separable convolution of the head towers
(edet_sepconv, TMA-staged and global-load kernels) and the stem (edet_stem_conv) -- against float64
references at the shapes where such kernels go wrong: every fused-conv layer shape of the
registered EfficientNetV2 models, k-block tails, ragged and multiple N tiles, 1-wide and 1-high
maps, maps smaller than a tile.

Shared rules:
  - one fp16 rounding of an fp32 sum: within one fp16 ulp of the float64 reference plus 5e-5 for
    values near zero (check_close);
  - every input, weight, bias and residual is carved out of a larger allocation with NaN after its
    last element, every output out of one with a 7.0 sentinel after it: no NaN may reach an output
    and no sentinel may change;
  - every case runs twice at the default grid and once under each "max_ctas" in GRIDS (1 = one CTA
    walks every tile): every run must give the same bits.  mbconv_expand_dw (off by default) gets
    the grid sweep alone."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

import plan_settings as ps
from automl_b200 import utils
from automl_b200._lib import EdetError
from automl_b200.efficientnetv2 import effnetv2_model
from oracle import efficientdet_oracle as eo

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SENTINEL = 7.0
GUARD = 4096                 # elements of NaN / sentinel after every carved tensor
GRIDS = (1, 2, 3, 8, 33)
FLOOR = 5e-5
NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6
ACTS = (SWISH, RELU6, NONE)  # what conv2d, sepconv and the stem accept
V2_MODELS = ['efficientnetv2-%s' % v for v in ('b0', 'b1', 'b2', 'b3', 's', 'm', 'l', 'xl')]
V1_MODELS = ['efficientnet-b%d' % i for i in range(9)] + ['efficientnet-l2']


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def carve(t):
  """A device copy of `t` whose allocation continues with GUARD NaNs: a read past its end brings
  NaN into the result."""
  if t is None:
    return None
  buf = torch.full((t.numel() + GUARD,), float('nan'), dtype=t.dtype, device=DEV)
  buf[:t.numel()] = t.reshape(-1).to(DEV)
  return buf[:t.numel()].view(t.shape)


class Out(object):
  """An fp16 output of `shape` filled with SENTINEL, carved from an allocation with GUARD more
  sentinels after it."""

  def __init__(self, shape):
    self.numel = int(np.prod(shape))
    self.buf = torch.full((self.numel + GUARD,), SENTINEL, dtype=torch.float16, device=DEV)
    self.t = self.buf[:self.numel].view(shape)

  def result(self):
    torch.cuda.synchronize()
    assert bool((self.buf[self.numel:] == SENTINEL).all()), 'written past the end of the output'
    got = self.t.cpu()
    assert not bool(got.isnan().any()), 'NaN in the output'
    return got


def span_bias(n, g, span):
  """Biases evenly over [-26, 10] (pre-activations cross every kink of SWISH / RELU6 and the
  swish clamp at -20.8), else N(0, 0.25)."""
  if not span:
    return torch.randn(n, generator=g) * 0.5
  return torch.linspace(-26.0, 10.0, n)[torch.randperm(n, generator=g)]


def act_ref(x, act):
  return {NONE: lambda t: t, SWISH: lambda t: t * torch.sigmoid(t),
          RELU6: lambda t: torch.clamp(t, 0, 6)}[act](x)


def check_close(got, ref, what=''):
  """Within one fp16 ulp of the float64 reference (the kernels round an fp32 sum to fp16 once),
  with an absolute floor for values near zero.  NaN fails."""
  ref = ref.double().cpu()
  ulp = torch.from_numpy(np.spacing(np.abs(ref.numpy()).astype(np.float16)).astype(np.float64))
  err = (got.double().cpu() - ref).abs()
  bad = ~(err <= ulp + FLOOR)
  assert not bool(bad.any()), '%s: max err %g (%d outside 1 ulp), first at %s' % (
      what, float(err.max()), int(bad.sum()), tuple(bad.nonzero()[0].tolist()))


def _same(a, b):
  if isinstance(a, tuple):
    return all(torch.equal(x, y) for x, y in zip(a, b))
  return torch.equal(a, b)


def over_grids(launch):
  """launch() -> output host tensor(s), written into fresh sentinel-filled buffers each call.  Two
  runs at the default grid and one under each max_ctas in GRIDS must give the same bits; returns
  them."""
  ops = _ops()
  base = launch()
  assert _same(launch(), base), 'two runs at the default grid differ'
  for g in GRIDS:
    try:
      ops.set_option('max_ctas', g)
      got = launch()
    finally:
      ops.set_option('max_ctas', 0)
    assert _same(got, base), 'max_ctas=%d differs from the default grid' % g
  return base


# ---------------------------------------------------------------------------------------------
# edet_conv2d (conv_tc.cu)
def v2_conv_shapes():
  """(cin, cout, k, stride, residual) of every k x k conv of the Fused-MBConv blocks of the
  registered EfficientNetV2 models: the expand conv (cin -> mid) of expand_ratio > 1 blocks, the
  single conv (+ skip) of expand_ratio == 1 blocks."""
  shapes = set()
  for name in V2_MODELS:
    for b in effnetv2_model.EffNetV2Arch(name).blocks:
      if b.conv_type != 1:
        continue
      if b.expand_ratio == 1:
        shapes.add((b.input_filters, b.output_filters, b.kernel_size, b.strides, b.has_skip))
      else:
        shapes.add((b.input_filters, b.mid_filters, b.kernel_size, b.strides, False))
  return sorted(shapes)


def _conv_cases():
  cases = []
  # registry shapes on small ragged maps: 11 x 19 outputs = 3 x 2 tiles of 4 x 16, the last ones
  # 3 rows / 3 columns wide
  for i, (cin, cout, k, s, res) in enumerate(v2_conv_shapes()):
    h, w = (11, 19) if s == 1 else (21, 37)
    cases.append((2, h, w, cin, cout, k, s, ACTS[i % 3], res))
  # 1-, 2- and 3-wide / high maps at both strides (the stride-2 encoder gives a 1-wide input an
  # empty odd-column sub-image), outputs narrower than 16 and lower than 4
  for s in (1, 2):
    for i, (h, w) in enumerate([(1, 1), (1, 9), (9, 1), (2, 3), (3, 2), (2, 17), (3, 33)]):
      cases.append((2, h, w, 24 if i % 2 else 40, 40 if i % 2 else 24, 3, s, ACTS[i % 3],
                    s == 1 and i % 2 == 0))
  cases += [
      (2, 13, 21, 40, 200, 3, 1, SWISH, True),     # 128 + 72: ragged second N tile, residual
      (1, 9, 18, 56, 264, 3, 1, RELU6, True),      # 128 + 128 + 8
      (2, 10, 14, 48, 96, 1, 1, SWISH, False),     # ksize 1
      (1, 13, 21, 16, 64, 1, 2, NONE, False),
      (1, 12, 20, 32, 48, 5, 1, RELU6, True),      # ksize 5
      (2, 11, 23, 24, 72, 5, 2, SWISH, False),
      (1, 5, 1, 16, 24, 5, 2, NONE, False),
      (3, 15, 33, 32, 128, 3, 2, SWISH, False),    # batch 3 at stride 2: the sub-image batch stride
  ]
  return cases


CONV_CASES = _conv_cases()


def _conv_id(c):
  n, h, w, cin, cout, k, s, act, res = c
  return 'n%d_%dx%d_c%d-%d_k%ds%d_a%d%s' % (n, h, w, cin, cout, k, s, act, '_res' if res else '')


def _conv_inputs(case, seed):
  n, h, w, cin, cout, k, s, act, has_res = case
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n, h, w, cin, generator=g).half()
  wk = (torch.randn(k, k, cin, cout, generator=g) / (k * cin**0.5)).half()      # HWIO like Keras
  bias = span_bias(cout, g, act != NONE)
  ho, wo = -(-h // s), -(-w // s)
  res = torch.randn(n, ho, wo, cout, generator=g).half() if has_res else None
  return x, wk, bias, res


def _conv_reference(x, wk, bias, res, act, s):
  ref = eo.conv2d_same(x.double().permute(0, 3, 1, 2), wk.double(), s) + bias.double().view(1, -1, 1, 1)
  ref = act_ref(ref, act).permute(0, 2, 3, 1)
  return ref + res.double() if res is not None else ref


def test_v2_registry_shapes_are_covered():
  shapes = v2_conv_shapes()
  assert {c for c, _, _, _, _ in shapes} == {16, 24, 32, 40, 48, 56, 64, 80, 96}
  assert min(o for _, o, _, _, _ in shapes) == 16 and max(o for _, o, _, _, _ in shapes) == 384
  assert {(c[3], c[4], c[5], c[6]) for c in CONV_CASES} >= {
      (cin, cout, k, s) for cin, cout, k, s, _ in shapes}


@pytest.mark.parametrize('case', CONV_CASES, ids=_conv_id)
def test_conv2d(case):
  ops = _ops()
  n, h, w, cin, cout, k, s, act, _ = case
  x, wk, bias, res = _conv_inputs(case, seed=17 + h * 7 + w + cin + cout + k)
  wt = wk.permute(0, 1, 3, 2).reshape(k * k, cout, cin).contiguous()             # [tap][cout][cin]
  dx, dwt, db, dres = carve(x), carve(wt), carve(bias), carve(res)
  ho, wo = -(-h // s), -(-w // s)

  def launch():
    out = Out((n, ho, wo, cout))
    ops.conv2d(dx, dwt, db, out.t, act, k, s, residual=dres)
    return out.result()

  got = over_grids(launch)
  check_close(got, _conv_reference(x, wk, bias, res, act, s), _conv_id(case))


@pytest.mark.parametrize('what', ['cin', 'cout', 'ksize', 'stride', 'relu', 'hswish', 'sigmoid'])
def test_conv2d_refusals(what):
  """Shapes and activations edet_conv2d does not implement raise, and the output keeps its
  sentinel."""
  ops = _ops()
  cin = 20 if what == 'cin' else 24
  cout = 36 if what == 'cout' else 32
  k = 7 if what == 'ksize' else 3
  s = 3 if what == 'stride' else 1
  act = {'relu': utils.ACT_RELU, 'hswish': utils.ACT_HSWISH, 'sigmoid': utils.ACT_SIGMOID}.get(what, SWISH)
  x = torch.randn(1, 9, 9, cin, device=DEV).half()
  wt = torch.randn(k * k, cout, cin, device=DEV).half()
  bias = torch.zeros(cout, device=DEV)
  out = Out((1, -(-9 // s), -(-9 // s), cout))
  with pytest.raises(EdetError):
    ops.conv2d(x, wt, bias, out.t, act, k, s)
  assert bool((out.result() == SENTINEL).all())


# ---------------------------------------------------------------------------------------------
# edet_sepconv (sepconv_tc.cu): c <= 64 runs the TMA-staged kernel (sepconv_impl 0 / 2), wider
# inputs and sepconv_impl 1 the global-load kernel
def _sep_cases():
  levels = [(1, 1, 1), (2, 1, 33), (2, 33, 1), (1, 8, 16), (2, 9, 17), (3, 80, 80)]
  nouts = [8, 24, 40, 64, 88, 128]
  cases = []
  for i, c in enumerate([8, 16, 40, 48, 64] + [72, 88, 112, 120, 128]):
    for j in range(3):
      cases.append(levels[(2 * i + j) % 6] + (c, nouts[(i + 2 * j) % 6], ACTS[(i + j) % 3]))
  return cases


SEP_CASES = _sep_cases()


def _sep_id(c):
  return 'n%d_%dx%d_c%d_o%d_a%d' % c


@pytest.mark.parametrize('impl', [0, 1, 2])
@pytest.mark.parametrize('case', SEP_CASES, ids=_sep_id)
def test_sepconv(case, impl):
  """Bit-identical to edet_fuse_dw + edet_pointwise_conv under every grid; the pair's depthwise
  result is within one ulp of the float64 depthwise, the output within one ulp of the float64
  pointwise of that fp16 intermediate (the kernel rounds it to fp16 in shared memory just as the
  pair does in global memory: a float64 reference that rounds its own intermediate can differ from
  the kernel's by an ulp wherever the fp32 depthwise sum lies within rounding error of an fp16
  tie, which one ulp at the output cannot absorb)."""
  ops = _ops()
  n, h, w, c, nout, act = case
  g = torch.Generator().manual_seed(31 + 5 * h + w + c + nout)
  x = torch.randn(n, h, w, c, generator=g).half()
  dw_w = (torch.randn(9, c, generator=g) / 3).float()
  pw = (torch.randn(nout, c, generator=g) / c**0.5).half()
  bias = span_bias(nout, g, act != NONE)
  ldo = nout + 16
  dx, ddw, dpw, db = carve(x), carve(dw_w), carve(pw), carve(bias)
  spec = [(dx, ops.RS_SAME, None, 1.0)]

  def launch():
    out = Out((n, h, w, ldo))
    ops.sepconv(spec, NONE, ddw, dpw, db, out.t, act, nout=nout)
    got = out.result()
    assert bool((got[..., nout:] == SENTINEL).all()), 'pad columns written'
    return got

  ops.set_option('sepconv_impl', impl)
  try:
    got = over_grids(launch)
  finally:
    ops.set_option('sepconv_impl', 0)
  check_sepconv(got, dx, ddw, dpw, db, act, nout, _sep_id(case))


def check_sepconv(got, dx, ddw, dpw, db, act, nout, what):
  """got (host, [N,h,w,ldo]) against edet_fuse_dw + edet_pointwise_conv on the device inputs, bit
  for bit, and the pair against float64 (see test_sepconv)."""
  ops = _ops()
  n, h, w, c = dx.shape
  tmp = Out((n, h, w, c))
  ops.fuse_dw([(dx, ops.RS_SAME, None, 1.0)], ddw, tmp.t, NONE)
  two = Out((n, h, w, got.shape[-1]))
  ops.pointwise_conv(tmp.t, dpw, db, two.t, act, rows=n * h * w, nout=nout)
  tmp, two = tmp.result(), two.result()
  assert torch.equal(got[..., :nout], two[..., :nout])
  x, dw_w, pw, bias = dx.cpu(), ddw.cpu(), dpw.cpu(), db.cpu()
  d = eo.depthwise_conv2d_same(x.double().permute(0, 3, 1, 2), dw_w.double().view(3, 3, c, 1))
  check_close(tmp, d.permute(0, 2, 3, 1), 'depthwise')
  ref = act_ref(tmp.double() @ pw.double().t() + bias.double(), act)
  check_close(got[..., :nout], ref, what)


@pytest.mark.parametrize('what', ['c', 'nout', 'ldo'])
def test_sepconv_refusals(what):
  ops = _ops()
  c = 136 if what == 'c' else 64
  nout = 136 if what == 'nout' else 64
  ldo = nout - 8 if what == 'ldo' else nout
  x = torch.randn(1, 8, 16, c, device=DEV).half()
  out = Out((1, 8, 16, ldo))
  with pytest.raises(EdetError):
    ops.sepconv([(x, ops.RS_SAME, None, 1.0)], NONE, torch.zeros(9, c, device=DEV),
                torch.zeros(nout, c, dtype=torch.float16, device=DEV), torch.zeros(nout, device=DEV),
                out.t, SWISH, nout=nout)
  assert bool((out.result() == SENTINEL).all())


# ---------------------------------------------------------------------------------------------
# edet_stem_conv: stem_tc.cu (float32 input split into fp16 hi + lo on the tensor cores), and the
# CUDA-core kernel of stem.cu as a second implementation
def _stem_cases():
  images = [(1, 1, 1), (1, 1, 40), (1, 40, 1), (1, 16, 32), (1, 17, 33), (16, 9, 13)]
  cases = []
  for i, cout in enumerate(range(8, 65, 8)):
    for d, dist in enumerate(('normal', 'wide')):
      cases.append(images[(i + 3 * d) % 6] + (cout, dist, ACTS[(i + d) % 3]))
  # the stems of efficientnet-b8 and -l2, wider than the tensor-core stem takes: under the default
  # stem_impl they run on the CUDA-core kernel, in 64-channel slabs (the last one partly live)
  for i, cout in enumerate((72, 136)):
    for d, dist in enumerate(('normal', 'wide')):
      cases.append(images[(2 * i + 3 * d + 1) % 6] + (cout, dist, ACTS[(i + 2 * d) % 3]))
  return cases


STEM_CASES = _stem_cases()


def _stem_id(c):
  return 'n%d_%dx%d_c%d_%s_a%d' % c


@pytest.mark.parametrize('impl', ['tensor_core', 'cuda_core'])
@pytest.mark.parametrize('case', STEM_CASES, ids=_stem_id)
def test_stem_conv(case, impl):
  """Images 1 x 1, 1 x 40, 40 x 1, one exact 8 x 16 output tile (16 x 32), one past it, and 16
  small images; inputs N(0, 1) or uniform in +-300, where dropping the lo half of the fp16 split
  costs more than an output ulp.  The two implementations agree to the bound, not bit for bit."""
  ops = _ops()
  n, h, w, cout, dist, act = case
  g = torch.Generator().manual_seed(3 + h * 3 + w + cout)
  if dist == 'normal':
    x = torch.randn(n, h, w, 3, generator=g)
  else:
    x = torch.rand(n, h, w, 3, generator=g) * 600.0 - 300.0
  k = (torch.randn(3, 3, 3, cout, generator=g) * 0.3).half()
  bias = span_bias(cout, g, act != NONE)
  dx, dk, db = carve(x), carve(k.reshape(27, cout)), carve(bias)

  def launch():
    out = Out((n, -(-h // 2), -(-w // 2), cout))
    ops.stem_conv(dx, out.t, dk, db, act)
    return out.result()

  ops.set_option('stem_impl', 0 if impl == 'tensor_core' else 1)
  try:
    got = over_grids(launch)
  finally:
    ops.set_option('stem_impl', 0)
  ref = eo.conv2d_same(x.double().permute(0, 3, 1, 2), k.double(), stride=2) + bias.double().view(1, -1, 1, 1)
  check_close(got, act_ref(ref, act).permute(0, 2, 3, 1), _stem_id(case))


# ---------------------------------------------------------------------------------------------
# edet_mbconv_expand_dw (off by default): output and SE sums do not depend on the grid
from test_gpu_kernels import MBF_CASES  # noqa: E402  (the shapes of its parity test)


@pytest.mark.parametrize('case', MBF_CASES)
def test_mbconv_expand_dw_grids(case):
  ops = _ops()
  n, h, w, cin, cmid, k, s, act, has_se = case
  g = torch.Generator().manual_seed(70 + h + cmid + k)
  x = carve(torch.randn(n, h, w, cin, generator=g).half())
  we = carve((torch.randn(cmid, cin, generator=g) / cin**0.5).half())
  be = carve(torch.randn(cmid, generator=g) * 0.2)
  wd = carve((torch.randn(k * k, cmid, generator=g) / k).float())
  bd = carve(torch.randn(cmid, generator=g) * 0.1)
  ho, wo = -(-h // s), -(-w // s)

  def launch():
    out = Out((n, ho, wo, cmid))
    se = torch.zeros(n, cmid, dtype=torch.int64, device=DEV) if has_se else None
    ops.mbconv_expand_dw(x, we, be, wd, bd, out.t, act, k, s, se)
    got = out.result()
    return (got, se.cpu()) if has_se else got

  over_grids(launch)


# ---------------------------------------------------------------------------------------------
def _kernel_grids(fn):
  """(name, grid x) of every kernel fn() launches, read from a torch.profiler trace."""
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, 'trace.json')
    prof.export_chrome_trace(path)
    with open(path) as f:
      events = json.load(f)['traceEvents']
  return [(e['name'], e['args']['grid'][0]) for e in events
          if e.get('cat') == 'kernel' and 'grid' in e.get('args', {})]


def _grid_launchers():
  """name -> (launch, number of tiles / work units) for one shape of each persistent kernel."""
  ops = _ops()
  h16 = lambda *s: torch.randn(*s, device=DEV).half()
  f32 = lambda *s: torch.randn(*s, device=DEV)
  x = h16(2, 40, 64, 64)              # conv 3x3 s1: 2 x 10 x 4 tiles; sepconv 2 x 5 x 4 tiles
  conv_out = torch.empty(2, 40, 64, 64, dtype=torch.float16, device=DEV)
  small = h16(1, 8, 20, 64)           # conv: 2 x 2 tiles; sepconv: 2 tiles
  small_out = torch.empty(1, 8, 20, 64, dtype=torch.float16, device=DEV)
  img = f32(2, 80, 128, 3)            # stem: 2 x 5 x 4 tiles of 8 x 16
  img_small = f32(1, 16, 40, 3)       # 2 tiles
  stem_out = torch.empty(2, 40, 64, 32, dtype=torch.float16, device=DEV)
  stem_small = torch.empty(1, 8, 20, 32, dtype=torch.float16, device=DEV)
  wt, b, dw, pw = h16(9, 64, 64), f32(64), f32(9, 64), h16(64, 64)
  stem_w, stem_b = h16(27, 32), f32(32)
  sep = lambda a, o: ops.sepconv([(a, ops.RS_SAME, None, 1.0)], NONE, dw, pw, b, o, SWISH)
  a = h16(8192, 64)                   # pointwise: 128 M blocks, >= 33 work units at any grid <= 33
  a_out = torch.empty(8192, 64, dtype=torch.float16, device=DEV)
  dx = h16(1, 80, 80, 128)            # tiled depthwise k5 s1: 10 x 5 tiles x 2 channel slices
  dx_out = torch.empty(1, 80, 80, 128, dtype=torch.float16, device=DEV)
  dw25, b128 = f32(25, 128), f32(128)
  mx = h16(2, 56, 56, 16)             # mbconv k3 s1: 2 x 4 x 4 tiles of 14 x 14 outputs
  mx_out = torch.empty(2, 56, 56, 64, dtype=torch.float16, device=DEV)
  we, wd9 = h16(64, 16), f32(9, 64)
  return {
      'conv2d': (lambda: ops.conv2d(x, wt, b, conv_out, SWISH, 3, 1), 80),
      'conv2d_small': (lambda: ops.conv2d(small, wt, b, small_out, SWISH, 3, 1), 4),
      'sepconv': (lambda: sep(x, conv_out), 40),
      'sepconv_small': (lambda: sep(small, small_out), 2),
      'stem': (lambda: ops.stem_conv(img, stem_out, stem_w, stem_b, SWISH), 40),
      'stem_small': (lambda: ops.stem_conv(img_small, stem_small, stem_w, stem_b, SWISH), 2),
      'pointwise': (lambda: ops.pointwise_conv(a, pw, b, a_out, SWISH), 33),
      'depthwise_tile': (lambda: ops.depthwise_conv(dx, dx_out, dw25, b128, SWISH, 5, 1), 100),
      'mbconv': (lambda: ops.mbconv_expand_dw(mx, we, b, wd9, b, mx_out, SWISH, 3, 1), 32),
  }


@pytest.mark.parametrize('max_ctas', [1, 3, 33])
def test_max_ctas_pins_the_grid(max_ctas):
  """max_ctas = G launches exactly G CTAs, or one per tile when there are fewer tiles (a CTA
  without a first tile would never retire from the dynamic scheduler, and the slot it leaves
  dirty would make a later launch skip tiles)."""
  ops = _ops()
  for name, (fn, tiles) in _grid_launchers().items():
    fn()   # module load and shared-memory opt-in outside the trace
    ops.set_option('max_ctas', max_ctas)
    try:
      grids = _kernel_grids(fn)
    finally:
      ops.set_option('max_ctas', 0)
    assert len(grids) == 1, (name, grids)
    assert grids[0][1] == min(max_ctas, tiles), (name, grids, tiles)


def test_fewer_tiles_than_max_ctas_leaves_the_scheduler_clean():
  """A launch with fewer tiles than max_ctas, then enough launches to reuse every scheduler slot
  once: each of them still covers its whole output."""
  ops = _ops()
  g = torch.Generator().manual_seed(8)
  x = carve(torch.randn(1, 16, 40, 3, generator=g))               # 2 stem tiles
  w = carve((torch.randn(27, 32, generator=g) * 0.3).half())
  b = carve(torch.randn(32, generator=g))
  out = torch.empty(1, 8, 20, 32, dtype=torch.float16, device=DEV)
  ops.stem_conv(x, out, w, b, SWISH)
  want = out.clone()
  bad = torch.zeros((), dtype=torch.bool, device=DEV)
  try:
    ops.set_option('max_ctas', 33)
    for _ in range(4097):      # the pool has 4096 self-resetting slots
      out.fill_(SENTINEL)
      ops.stem_conv(x, out, w, b, SWISH)
      bad |= (out != want).any()
    torch.cuda.synchronize()
  finally:
    ops.set_option('max_ctas', 0)
  assert not bool(bad)


def test_max_ctas_option_range():
  ops = _ops()
  assert ops.get_option('max_ctas') == 0
  for bad in (-1, 4097):
    with pytest.raises(EdetError):
      ops.set_option('max_ctas', bad)
  ops.set_option('max_ctas', 4096)
  assert ops.get_option('max_ctas') == 4096
  ps.reset(ops)
  assert ops.get_option('max_ctas') == 0
