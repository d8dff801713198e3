"""The two tensor-core kernels the earlier sweeps left out -- the sub-pixel transposed convolution of
the segmentation head (edet_conv2d_transpose, convt_tc.cu) and the fused MBConv front, expand 1x1
+ depthwise k x k (+ SE squeeze) (edet_mbconv_expand_dw, mbconv_fused.cu) -- against float64
references at every registered layer shape and at the edges of their host-side plans, with the
harness of test_gpu_persistent_kernels.py: one fp16 ulp plus 5e-5 (check_close, or a bound derived
from it), NaN / sentinel guards after every input and output, and the same bits under every
pinned grid.  Two network cases put the block_k = 16 transposed convolution (D2) and the relu6,
no-SE fused front (lite1) into a whole forward pass.

The registry functions (seg_stage_shapes, expand_block_shapes), the restatements of the two host
plans and the coverage tests need no GPU; every other test is marked gpu on its own."""
import ctypes

import numpy as np
import pytest
import torch

from automl_b200 import utils
from automl_b200._lib import EdetError
from test_gpu_conv_transpose import reference as convt_f64
from test_gpu_memory_bound_kernels import (  # noqa: F401  (the shared harness)
    DET_MODELS, INT_GUARD, SE_UNIT, SWISH_LO, Buf, _act_code, _act_slope, _check_se_sums, _det_arch,
    _dw_reference, depthwise_f64)
from test_gpu_persistent_kernels import (  # noqa: F401
    DEV, FLOOR, GUARD, SENTINEL, Out, carve, check_close, over_grids, span_bias)

NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6
U = 2.0**-24                  # fp32 unit roundoff
BOTH = ('object_detection', 'segmentation')
# lite0 (320) and lite2 (448) cannot build the segmentation head at their registered sizes (P7 is
# not half of P6 there, so the reference's concat fails): they run at the nearest smaller multiple
# of 128, every other model at its registered size
SEG_IMAGE = {'efficientdet-lite0': 256, 'efficientdet-lite2': 384}


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _cdiv(a, b):
  return -(-a // b)


def _rup(x, m):
  return _cdiv(x, m) * m


def _ulp16(t):
  """Spacing of the fp16 value of |t| (float64): the step of one fp16 rounding flip."""
  return torch.from_numpy(np.spacing(np.abs(t.double().cpu().numpy()).astype(np.float16)).astype(np.float64))


def _p(t):
  return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------
# shape registries (no GPU)
def seg_stage_shapes():
  """(in_hw, c0 = F, c1 = F or 0, cout, act) of every Conv2DTranspose stage of the segmentation
  head of every registered EfficientDet / lite model (heads = detection + segmentation): the
  first stage reads the top BiFPN level alone, the later ones the previous stage and the skip
  level, the BN stages apply the model's activation and the final one (seg_num_classes outputs)
  none, as the engine lowers them."""
  shapes = set()
  for name in DET_MODELS:
    a = _det_arch(name, SEG_IMAGE.get(name), (('heads', BOTH),))
    for st in a.seg_stages:
      c1 = st.in_channels - a.fpn_filters
      act = _act_code(a.act_type) if st.bn_scope else NONE
      shapes.add((st.in_hw, a.fpn_filters, c1, st.out_channels, act))
  return sorted(shapes)


def expand_block_shapes():
  """(cin, cmid, k, stride, has_se, act) of every MBConv block with an expand conv in the same
  models at their registered sizes."""
  shapes = set()
  for name in DET_MODELS:
    a = _det_arch(name)
    for b in a.blocks:
      if b.expand_name:
        shapes.add((b.input_filters, b.mid_filters, b.kernel_size, b.stride, bool(b.se_filters),
                    _act_code(a.act_type)))
  return sorted(shapes)


# ---------------------------------------------------------------------------------------------
# the host plans restated (no GPU)
CT_SMEM = 227 * 1024           # convttc::kSmemLimit


def convt_plan(c0, c1, cout):
  """edet_conv2d_transpose's host plan: block_k is the k-block that pads the sources' K least (the
  larger one on a tie); block_n the phase's round8(cout) channels rounded up to 32 / 64 / 96 /
  128, else tiles of 128; woff1 the weight column where source 1 starts; stages per consumer."""
  best = 0
  for bk in (64, 32, 16):
    padded = _rup(c0, bk) + (_rup(c1, bk) if c1 else 0)
    if best == 0 or padded < best:
      best, block_k = padded, bk
  c8 = _rup(cout, 8)
  block_n = _rup(c8, 32) if c8 <= 128 else 128
  n_per_phase = _cdiv(c8, block_n)
  stage = 64 * block_k * 2 + _rup(block_n * block_k * 2, 1024)
  stages = min((CT_SMEM - 1024 - (2 * 2 * 8192 + 2 * 8 * 8)) // stage, 8)
  return dict(block_k=block_k, block_n=block_n, n_per_phase=n_per_phase, woff1=_rup(c0, 8),
              partial=c8 % block_n != 0, team_stages=stages // 2,
              nkb=(_cdiv(c0, block_k), _cdiv(c1, block_k) if c1 else 0))


MBF_PATCH = 16                 # mbf::kPatch
MBF_MAX_CH = 64                # mbf::kMaxCh


def mbf_plan(cin, cmid, k, s):
  """edet_mbconv_expand_dw's host plan: cmid in num_chunks chunks of ch (a multiple of 16) channels,
  the last one holding cv = cmid - (num_chunks - 1) ch; block_k 16 / 32 / 64 by cin; an input
  patch of 16 x 16 gives otw x otw outputs."""
  num_chunks = _cdiv(cmid, MBF_MAX_CH)
  ch = _rup(_cdiv(cmid, num_chunks), 16)
  block_k = 16 if cin <= 16 else (32 if cin <= 32 else 64)
  while True:
    smem = 1024 + 256 * block_k * 2 + _rup(ch * block_k * 2, 1024) + 256 * (MBF_MAX_CH * 2 + 16) + ch * 8 + 64
    if smem <= 113 * 1024 or block_k <= 32:
      break
    block_k //= 2
  return dict(num_chunks=num_chunks, ch=ch, last_cv=cmid - (num_chunks - 1) * ch, block_k=block_k,
              num_k_blocks=_cdiv(cin, block_k), otw=(MBF_PATCH - k) // s + 1, smem=smem)


def mbf_partials(h, w, k, s):
  """Upper bound on the fp32 partial sums rounded to the 2^-20 fixed point that make up one
  (image, channel) SE sum: one per output row and tile column in the row path, one per
  column-pair work item of each tile in the k3 s2 path (4 per 7-wide tile)."""
  otw = (MBF_PATCH - k) // s + 1
  ho, wo = _cdiv(h, s), _cdiv(w, s)
  if (k, s) == (3, 2):
    return _cdiv(ho, otw) * _cdiv(wo, otw) * _cdiv(otw, 2)
  return ho * _cdiv(wo, otw)


# ---------------------------------------------------------------------------------------------
# edet_conv2d_transpose cases: (n, h, w, c0, lda0, c1, lda1, cout, ldo, act); c1 = 0: one source
def _convt_cases():
  cases = []
  shapes = seg_stage_shapes()
  # every registered stage at its real map size, batch 1, as the engine lays it out
  for (h, w), c0, c1, cout, act in shapes:
    cases.append((1, h, w, c0, c0, c1, c1, cout, _rup(cout, 8), act))
  # batch 3 on the smallest two-source stage of each width (the image stride of the maps)
  for f in sorted({s[1] for s in shapes}):
    (h, w), c0, c1, cout, act = min((s for s in shapes if s[1] == f and s[2] and s[4] != NONE),
                                    key=lambda s: s[0])
    cases.append((3, h, w, c0, c0, c1, c1, cout, cout, act))
  # synthetic edges: c0 % 8 != 0 (woff1 = round8(c0)), block_k 16, every block_n, ragged N,
  # 1 x W and H x 1 maps and maps that end inside a 4 x 16 tile, strided sources with NaN in the
  # gap, output rows wider than round8(cout)
  pairs = [(8, 0), (20, 20), (72, 88), (200, 200), (8, 88), (20, 0), (72, 8), (200, 20), (20, 200),
           (72, 0), (200, 88), (8, 20), (200, 0)]
  couts = (1, 3, 8, 21, 33, 96, 97, 128, 129, 150, 200, 288, 384)
  maps = [(1, 1), (1, 33), (33, 1), (2, 3), (3, 2), (4, 16), (5, 17), (15, 4), (16, 5), (17, 15),
          (33, 16), (1, 17), (3, 1)]
  for i, ((c0, c1), cout, (h, w)) in enumerate(zip(pairs, couts, maps)):
    lda0 = _rup(c0, 8) + (8 if i % 2 else 0)
    lda1 = _rup(c1, 8) + (16 if i % 3 == 0 else 0) if c1 else 0
    ldo = _rup(cout, 8) + (8 if i % 2 == 0 else 0)
    cases.append((2 if i % 4 == 1 else 1, h, w, c0, lda0, c1, lda1, cout, ldo, (SWISH, RELU6, NONE)[i % 3]))
  return cases


CONVT_CASES = _convt_cases()


def _convt_id(c):
  n, h, w, c0, lda0, c1, lda1, cout, ldo, act = c
  p = convt_plan(c0, c1, cout)
  return 'n%d_%dx%d_c%d.%d_c%d.%d_o%d.%d_a%d_bk%d_bn%d' % (n, h, w, c0, lda0, c1, lda1, cout, ldo, act,
                                                         p['block_k'], p['block_n'])


def test_seg_registry_shapes_are_covered():
  shapes = seg_stage_shapes()
  assert {f for _, f, _, _, _ in shapes} == {64, 88, 112, 160, 200, 224, 288, 384}
  assert {c for _, _, _, c, _ in shapes} == {3, 64, 88, 112, 160, 200, 224, 288, 384}
  # D7x: six stages, the first from a 6 x 6 map, the fifth a BN stage on a 96 x 96 map
  assert ((6, 6), 384, 0, 384, SWISH) in shapes and ((96, 96), 384, 384, 384, SWISH) in shapes
  covered = {((h, w), c0, c1, cout, act) for n, h, w, c0, lda0, c1, lda1, cout, ldo, act in CONVT_CASES
             if n == 1 and lda0 == c0 and lda1 == c1}
  assert covered >= set(shapes)
  assert {c[3] for c in CONVT_CASES if c[0] == 3} == {f for _, f, _, _, _ in shapes}


def test_convt_plan_is_reached():
  plans = [(c, convt_plan(c[3], c[5], c[7])) for c in CONVT_CASES]
  assert {p['block_k'] for _, p in plans} == {16, 32, 64}
  assert {p['block_n'] for _, p in plans} == {32, 64, 96, 128}
  assert {p['n_per_phase'] for _, p in plans} == {1, 2, 3}
  assert {p['n_per_phase'] for _, p in plans if p['partial']} >= {1, 2, 3}
  assert any(c[3] % 8 and c[5] for c, _ in plans)                     # woff1 = round8(c0) != c0
  assert any(p['block_k'] == 16 and c[5] for c, p in plans)
  assert all(p['team_stages'] >= 2 for _, p in plans)
  # the "<2 pipeline stages" refusal cannot fire: the largest stage (block_n 128, block_k 64)
  # still leaves four per consumer
  assert min(convt_plan(c0, 0, 384)['team_stages'] for c0 in (64, 96, 128)) == 4
  # the registry widths whose K pads least at block_k = 16 (D2 / lite2, lite3x), and the second
  # N block of 32 / 72 live channels (D3 / lite3, lite3x) and the partial third one (D5)
  assert convt_plan(112, 112, 112)['block_k'] == 16 and convt_plan(112, 112, 112)['nkb'] == (7, 7)
  assert convt_plan(200, 200, 200)['block_k'] == 16 and convt_plan(200, 200, 200)['nkb'] == (13, 13)
  assert convt_plan(160, 160, 160)['n_per_phase'] == 2 and convt_plan(288, 288, 288)['partial']
  # block_k is the larger on a tie: 20 + 20 pads to 64 at both 32 and 16
  assert convt_plan(20, 20, 8)['block_k'] == 32


def _convt_inputs(case, seed):
  n, h, w, c0, lda0, c1, lda1, cout, ldo, act = case
  g = torch.Generator().manual_seed(seed)
  a0 = torch.randn(n, h, w, lda0, generator=g).half()
  a0[..., c0:] = float('nan')
  a1 = None
  if c1:
    a1 = torch.randn(n, h, w, lda1, generator=g).half()
    a1[..., c1:] = float('nan')
  cin = c0 + c1
  # conv outputs of std ~3, biases over every kink
  kernel = (torch.randn(3, 3, cout, cin, generator=g) * (3.0 / (2.25 * cin)**0.5)).half()
  bias = span_bias(cout, g, act != NONE)
  return a0, a1, kernel, bias


@pytest.mark.gpu
@pytest.mark.parametrize('case', CONVT_CASES, ids=_convt_id)
def test_conv2d_transpose(case):
  """Within one fp16 ulp + 5e-5 of the float64 transposed-convolution formula; channels
  [cout, round8(cout)) exactly 0, [round8(cout), ldo) and everything after the output keep the
  sentinel; NaN after every input, weight and bias and in the sources' pixel-stride gaps; the same
  bits under every grid."""
  ops = _ops()
  n, h, w, c0, lda0, c1, lda1, cout, ldo, act = case
  a0, a1, kernel, bias = _convt_inputs(case, seed=CONVT_CASES.index(case) + 3 * cout + c0)
  wt = torch.from_numpy(ops.conv_transpose_weights(kernel.double().numpy(), c0)).half()
  da0, da1, dwt, db = carve(a0), carve(a1), carve(wt), carve(bias)
  c8 = _rup(cout, 8)

  def launch():
    out = Out((n, 2 * h, 2 * w, ldo))
    ops.conv2d_transpose(da0, dwt, db, out.t, act, cout, a1=da1, c0=c0, c1=c1 if c1 else None)
    got = out.result()
    assert bool((got[..., cout:c8] == 0).all()), 'channels cout .. round8(cout) not zero'
    assert bool((got[..., c8:] == SENTINEL).all()), 'channels past round8(cout) written'
    return got

  got = over_grids(launch)
  x = a0[..., :c0] if not c1 else torch.cat([a0[..., :c0], a1[..., :c1]], -1)
  ref = convt_f64(x.to(DEV).double(), kernel.to(DEV).double(), bias.to(DEV).double(), act)
  check_close(got[..., :cout], ref, _convt_id(case))


def _convt_refusals():
  return ['null_a0', 'null_wt', 'null_bias', 'null_out', 'empty', 'c0_over_lda0', 'lda0_mod8',
          'c1_zero', 'lda1_mod8', 'ldo_under_c8', 'ldo_mod8', 'too_many_tiles', 'act_sigmoid']


@pytest.mark.gpu
@pytest.mark.parametrize('what', _convt_refusals())
def test_conv2d_transpose_refusals(what):
  """Each argument check of edet_conv2d_transpose, and an activation it does not implement, raises;
  no input, weight, bias or output changes."""
  g = torch.Generator().manual_seed(9)
  c0, c1, cout = 24, 16, 21
  a0 = carve(torch.randn(1, 3, 5, c0, generator=g).half())
  a1 = carve(torch.randn(1, 3, 5, c1, generator=g).half())
  wt = carve(torch.randn(4, 4 * 24, 40, generator=g).half())
  bias = carve(torch.randn(cout, generator=g))
  out = Out((1, 6, 10, 24))
  before = [t.clone() for t in (a0, a1, wt, bias)]
  args = dict(a0=a0, c0=c0, lda0=c0, a1=a1, c1=c1, lda1=c1, wt=wt, bias=bias, act=SWISH, out=out.t,
              ldo=24, n=1, h=3, w=5, cout=cout)
  args.update({
      'null_a0': dict(a0=None), 'null_wt': dict(wt=None), 'null_bias': dict(bias=None),
      'null_out': dict(out=None), 'empty': dict(cout=0), 'c0_over_lda0': dict(c0=32),
      'lda0_mod8': dict(c0=20, lda0=20), 'c1_zero': dict(c1=0), 'lda1_mod8': dict(c1=12, lda1=12),
      'ldo_under_c8': dict(ldo=16), 'ldo_mod8': dict(ldo=28),
      'too_many_tiles': dict(n=1 << 24, h=64, w=64), 'act_sigmoid': dict(act=utils.ACT_SIGMOID),
  }[what])
  from automl_b200 import _lib
  with pytest.raises(EdetError):
    _lib.call('edet_conv2d_transpose', _p(args['a0']), args['c0'], args['lda0'], _p(args['a1']),
              args['c1'], args['lda1'], _p(args['wt']), _p(args['bias']), args['act'], _p(args['out']),
              args['ldo'], args['n'], args['h'], args['w'], args['cout'], _stream())
  assert bool((out.result() == SENTINEL).all())
  for t, b in zip((a0, a1, wt, bias), before):
    assert torch.equal(t, b)


# ---------------------------------------------------------------------------------------------
# edet_mbconv_expand_dw cases: (n, h, w, cin, cmid, k, s, act, has_se)
MBF_RAGGED = {1: [(37, 29)], 2: [(37, 29), (38, 30)]}   # odd / even sizes at stride 2: pad_t 1 / 0
MBF_SMALL = {1: (5, 7), 2: (6, 5)}                      # fewer outputs than one output tile


def _mbf_cases():
  cases = []
  # every registered expand block on a ragged map of 3 x 3 patches (k3 s2 alternately odd and even)
  # and on a map inside one output tile; batch 2 with SE (per-image sums)
  for i, (cin, cmid, k, s, se, act) in enumerate(expand_block_shapes()):
    n = 2 if se else 1
    h, w = MBF_RAGGED[s][i % len(MBF_RAGGED[s])]
    cases.append((n, h, w, cin, cmid, k, s, act, se))
    cases.append((n,) + MBF_SMALL[s] + (cin, cmid, k, s, act, se))
  # every (k, s) instantiation with both activations, with and without SE; partial last chunks
  # (136 = 48 + 48 + 40, 200 = 3 x 64 + 8), cmid 8 (one chunk of 8 live of 16); cin 8 / 24 / 40 /
  # 72 (block_k 16 / 32 / 64, a k-block tail); 1 x 1, 1 x 17 and 17 x 1 maps
  cmids = (136, 200, 8, 96)
  cins = (8, 24, 40, 72)
  maps = ((1, 1), (1, 17), (17, 1), (17, 17))
  i = 0
  for k, s in ((3, 1), (3, 2), (5, 1), (5, 2)):
    for act in (SWISH, RELU6):
      for se in (True, False):
        h, w = maps[(i + i // 4) % 4]
        cases.append((3 if i % 5 == 2 else 1, h, w, cins[i % 4], cmids[(i // 2) % 4], k, s, act, se))
        i += 1
  return cases


MBF2_CASES = _mbf_cases()


def _mbf_id(c):
  n, h, w, cin, cmid, k, s, act, se = c
  return 'n%d_%dx%d_c%d-%d_k%ds%d_a%d%s' % (n, h, w, cin, cmid, k, s, act, '_se' if se else '')


def test_expand_registry_shapes_are_covered():
  shapes = expand_block_shapes()
  assert len(shapes) == 103
  assert max(c[1] for c in shapes) == 3840 and max(c[0] for c in shapes) == 640
  covered = {}
  for n, h, w, cin, cmid, k, s, act, se in MBF2_CASES:
    covered.setdefault((cin, cmid, k, s, se, act), set()).add((h, w))
  for shape in shapes:
    s, otw = shape[3], mbf_plan(shape[0], shape[1], shape[2], shape[3])['otw']
    maps = covered[shape]
    assert any(_cdiv(h, s) > 2 * otw and _cdiv(w, s) > 2 * otw for h, w in maps), shape
    assert any(_cdiv(h, s) < otw and _cdiv(w, s) < otw for h, w in maps), shape
  # the k3 s2 shapes at odd and even sizes (pad_t / pad_l 1 and 0)
  assert {h % 2 for n, h, w, cin, cmid, k, s, act, se in MBF2_CASES if (k, s) == (3, 2) and h > 16} == {0, 1}
  assert all(n == 2 for n, h, w, cin, cmid, k, s, act, se in MBF2_CASES[:2 * len(shapes)] if se)


def test_mbf_plan_is_reached():
  combos = {(k, s, act, se) for _, _, _, _, _, k, s, act, se in MBF2_CASES}
  assert combos == {(k, s, a, se) for k in (3, 5) for s in (1, 2) for a in (SWISH, RELU6)
                    for se in (True, False)}
  plans = [mbf_plan(c[3], c[4], c[5], c[6]) for c in MBF2_CASES]
  assert {p['otw'] for p in plans} == {14, 7, 12, 6}
  assert {p['block_k'] for p in plans} == {16, 32, 64}
  assert any(c[3] % p['block_k'] for c, p in zip(MBF2_CASES, plans))   # a k-block tail
  assert any(p['last_cv'] < p['ch'] for p in plans)
  assert mbf_plan(24, 144, 3, 1)['num_chunks'] == 3 and mbf_plan(24, 144, 3, 1)['ch'] == 48
  assert mbf_plan(40, 136, 3, 1)['last_cv'] == 40 and mbf_plan(40, 200, 3, 1)['last_cv'] == 8
  assert mbf_plan(40, 8, 3, 1)['ch'] == 16 and mbf_plan(640, 3840, 5, 1)['num_chunks'] == 60
  assert all(p['smem'] <= 232448 for p in plans)
  assert {(h, w) for _, h, w, _, _, _, _, _, _ in MBF2_CASES} >= {(1, 1), (1, 17), (17, 1)}


def _mbf_inputs(case, seed):
  n, h, w, cin, cmid, k, s, act, _ = case
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n, h, w, cin, generator=g).half()
  we = (torch.randn(cmid, cin, generator=g) / cin**0.5).half()
  be = span_bias(cmid, g, False)
  taps = torch.randn(k * k, cmid, generator=g) / k          # genuine fp32 taps [k*k][cmid]
  bd = span_bias(cmid, g, True)
  return x, we, be, taps, bd


def _mbf_reference(x, we, be, taps, bd, act, k, s):
  """float64 NHWC (y, z, m) of _dw_reference over E = fp16(act(x we^T + be)) -- the expanded map
  as the unfused pipeline stores it -- and flip = sum_taps ulp16(E) |tap|."""
  z = x.to(DEV).double() @ we.to(DEV).double().t() + be.to(DEV).double()
  if act == SWISH:
    z = z.clamp(min=SWISH_LO)
    e = z * torch.sigmoid(z)
  else:
    e = z.clamp(0, 6)
  e = e.half().double().cpu()
  y, zd, m = _dw_reference(e, taps, bd, act, k, s)
  return y, zd, m, depthwise_f64(_ulp16(e), taps.abs(), k, s)


def check_mbf(got, y, z, m, flip, act, k, what):
  """The output bound of test_mbconv_expand_dw, from _mbf_reference's (y, z, m, flip)."""
  dz = flip + (k * k + 1) * U * m
  tol = _ulp16(y) + FLOOR + _act_slope(z, act, dz) * dz
  err = (got.double() - y).abs()
  bad = ~(err <= tol)
  assert not bool(bad.any()), '%s: max err %g, %d outside the bound, first at %s' % (
      what, float(err.max()), int(bad.sum()), tuple(bad.nonzero()[0].tolist()))


@pytest.mark.gpu
@pytest.mark.parametrize('case', MBF2_CASES, ids=_mbf_id)
def test_mbconv_expand_dw(case):
  """Output against the float64 depthwise of the fp16-rounded expanded map E.  The kernel's E is
  its fp32 expand sum + bias, activated and rounded to fp16; where the float64 value lies within
  that sum's error of an fp16 rounding boundary it rounds to the neighbouring fp16 value, one
  ulp16(E) away.  With such a flip at every tap, an output moves by at most
  flip = sum_taps ulp16(E) |tap| before its activation.  The depthwise itself (k*k fp32 FMAs from
  zero, then + bias) is off by <= (k*k + 1) u m.  So per output:
      |got - y| <= ulp16(y) + 5e-5 + act'(z) (flip + (k*k + 1) u m),
  the first two terms being check_close's single rounding, act' bounded over the window by
  _act_slope (its 1e-3 swish allowance is for windows < 2e-3; a wider window adds < 0.5 window^2,
  under 0.2 % of the window term here).  The SE sums take the same window inside _check_se_sums
  (m widened by flip / ((k*k + 1) u)), with the kernel's partial count (mbf_partials).  From a
  non-zero start they come out exactly start + the increment of a run from zero, under every
  grid; NaN after every input, sentinels after the output, INT_GUARD after the sums."""
  n, h, w, cin, cmid, k, s, act, has_se = case
  ops = _ops()
  x, we, be, taps, bd = _mbf_inputs(case, seed=MBF2_CASES.index(case) * 13 + cmid + h)
  dx, dwe, dbe, dtaps, dbd = carve(x), carve(we), carve(be), carve(taps), carve(bd)
  ho, wo = _cdiv(h, s), _cdiv(w, s)
  start = torch.full((n, cmid), INT_GUARD, dtype=torch.int64) - 977 * torch.arange(n * cmid).view(n, cmid)

  def launch(init):
    out = Out((n, ho, wo, cmid))
    se = Buf(init, INT_GUARD) if has_se else None
    ops.mbconv_expand_dw(dx, dwe, dbe, dtaps, dbd, out.t, act, k, s, se.t if se else None)
    got = out.result()
    return (got, se.result()) if has_se else got

  first = launch(torch.zeros(n, cmid, dtype=torch.int64))
  res = over_grids(lambda: launch(start))
  got = res[0] if has_se else res
  assert torch.equal(got, first[0] if has_se else first), 'output depends on the SE start'
  y, z, m, flip = _mbf_reference(x, we, be, taps, bd, act, k, s)
  check_mbf(got, y, z, m, flip, act, k, _mbf_id(case))
  if has_se:
    sums = first[1]
    _check_se_sums(sums, y, z, m + flip / ((k * k + 1) * U), act, k, mbf_partials(h, w, k, s),
                   _mbf_id(case))
    assert torch.equal(res[1], start + sums), 'SE sums not start + the increment'


def _mbf_refusals():
  return ['cin12', 'cmid20', 'k7', 'k1', 'stride3', 'act_none', 'act_relu', 'null_x', 'null_we',
          'null_bias_e', 'null_wd', 'null_bias_d', 'null_out']


@pytest.mark.gpu
@pytest.mark.parametrize('what', _mbf_refusals())
def test_mbconv_expand_dw_refusals(what):
  """cin % 8, cmid % 8, k not in {3, 5}, stride not in {1, 2}, an activation other than swish /
  relu6 and each null pointer raise; no input, output or SE sum changes."""
  g = torch.Generator().manual_seed(6)
  cin = 12 if what == 'cin12' else 16
  cmid = 20 if what == 'cmid20' else 32
  k = {'k7': 7, 'k1': 1}.get(what, 3)
  s = 3 if what == 'stride3' else 1
  act = {'act_none': NONE, 'act_relu': utils.ACT_RELU}.get(what, SWISH)
  t = dict(x=carve(torch.randn(1, 9, 9, cin, generator=g).half()),
           we=carve(torch.randn(cmid, cin, generator=g).half()),
           bias_e=carve(torch.randn(cmid, generator=g)), wd=carve(torch.randn(k * k, cmid, generator=g)),
           bias_d=carve(torch.randn(cmid, generator=g)))
  before = {name: v.clone() for name, v in t.items()}
  out = Out((1, _cdiv(9, s), _cdiv(9, s), cmid))
  start = torch.randint(-2**40, 2**40, (1, cmid), generator=g, dtype=torch.int64)
  se = Buf(start, INT_GUARD)
  ptrs = dict(t, out=out.t)
  if what.startswith('null_'):
    ptrs[what[5:]] = None
  from automl_b200 import _lib
  with pytest.raises(EdetError):
    _lib.call('edet_mbconv_expand_dw', *[_p(ptrs[a]) for a in ('x', 'we', 'bias_e', 'wd', 'bias_d', 'out')],
              _p(se.t), 1, 9, 9, cin, cmid, k, s, act, _stream())
  assert bool((out.result() == SENTINEL).all())
  assert torch.equal(se.result(), start)
  for name, v in t.items():
    assert torch.equal(v, before[name]), name


# ---------------------------------------------------------------------------------------------
# the two kernels in a whole network
@pytest.mark.gpu
def test_seg_logits_d2_match_oracle():
  """D2 (F = 112): every stage of its segmentation head runs the block_k = 16 plan (7 k-blocks per
  source), within the 1e-3 relative-L2 bar of test_seg_logits_match_oracle."""
  import seg_oracle
  from test_gpu_segmentation import REL_TOL, _engine, _setup, rel_l2
  c, a, w, x = _setup('efficientdet-d2', 256, 1, ['segmentation'])
  assert all(convt_plan(a.fpn_filters, st.in_channels - a.fpn_filters, st.out_channels)['block_k'] == 16
             for st in a.seg_stages)
  eng = _engine(c, w, 1, use_cuda_graph=False)
  eng.forward(torch.from_numpy(x))
  got = eng.seg_logits.float().cpu()
  torch.cuda.synchronize()
  ref = seg_oracle.seg_logits(c, w, x, torch.float32)
  assert tuple(got.shape) == tuple(ref.shape)
  assert rel_l2(got, ref) < REL_TOL
  assert bool((eng.seg_out[..., c.seg_num_classes:] == 0).all())


@pytest.mark.gpu
def test_fused_mbconv_front_lite1():
  """lite1 (relu6, no SE) with Engine(fuse_mbconv_front=True): every block output within 5e-4
  relative L2 of the default engine's separate expand and depthwise kernels."""
  from test_gpu_network import _engine, _setup, rel_l2
  c, a, w, x = _setup('efficientdet-lite1', 256, 2, seed=4)
  fused = _engine(c, w, 2, use_cuda_graph=False, fuse_mbconv_front=True)
  assert any(name.endswith('/expand_dw') for name in fused.op_names())
  plain = _engine(c, w, 2, use_cuda_graph=False)
  fused.forward(torch.from_numpy(x))
  plain.forward(torch.from_numpy(x))
  torch.cuda.synchronize()
  for b in a.blocks:
    got = fused.buffers[b.name + '/out'].float().cpu()
    assert rel_l2(got, plain.buffers[b.name + '/out'].float().cpu()) < 5e-4, b.name
