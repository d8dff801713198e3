"""The pointwise GEMM (edet_pointwise_conv, pointwise_tc.cu) at every 1x1 convolution the registered
models lower -- the EfficientDet D0-D7x / lite0-lite4 detectors under every feature-network
variant and the EfficientNet V1 / V2 classifiers -- against a float64 reference, with the harness
of test_gpu_persistent_kernels.py: one fp16 ulp plus 5e-5 (check_close), NaN after every input,
sentinels after every output, and the same bits under every plan setting of plan_settings.py.

pw_shapes() is the registry: (k, nout, per-image W, residual, act) of every launch.  It and the
tests that the case list and the plan classes cover it need no GPU; the drift guard checks, on the
device, that the models launch exactly the registry's shapes.  The whole file runs in under a
minute on an H100 80GB HBM3 (37 s in one run)."""
import functools

import numpy as np
import pytest
import torch

import plan_settings as ps
import test_gpu_class_argmax
from automl_b200 import arch
from automl_b200 import hparams_config
from automl_b200 import ops
from automl_b200 import utils
from automl_b200.efficientnetv2 import effnetv2_model
from test_gpu_memory_bound_kernels import DET_MODELS, FPN_VARIANTS, _act_code, _det_arch
from test_gpu_persistent_kernels import (DEV, SENTINEL, V1_MODELS, V2_MODELS, Out, act_ref, carve,
                                         check_close, span_bias)

NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6
CLS_MODELS = V1_MODELS + V2_MODELS


def _round8(x):
  return -(-x // 8) * 8


def _cdiv(a, b):
  return -(-a // b)


# ---------------------------------------------------------------------------------------------
# the registry (no GPU)
def _mbconv_pw(blocks, act):
  """Expand (shared W, act) and project (ACT_NONE; per-image W iff SE, residual iff skip) of the
  MBConv blocks (lowering.LaunchList._mbconv)."""
  out = set()
  for b in blocks:
    if b.expand_name:
      out.add((b.input_filters, b.mid_filters, False, False, act))
    out.add((b.mid_filters, b.output_filters, bool(b.se_filters), bool(b.has_skip), NONE))
  return out


@functools.lru_cache(maxsize=None)
def det_pw_shapes(name, over=()):
  """The 1x1 launches of Engine for one detector config: backbone expand / project, the resample
  convs with a channel change (P6 creation and the cell inputs), the node pointwise (F -> F, the
  activation only under conv_bn_act_pattern), the head-tower pointwise where the fused sepconv
  does not run (F > SEPCONV_MAX_C) and the stored-path predict layers F -> A*4 and F -> A*C."""
  a = _det_arch(name, None, over)
  act = _act_code(a.act_type)
  F, A, C = a.fpn_filters, a.num_anchors, a.num_classes
  out = _mbconv_pw(a.blocks, act)
  resamples = [r for r in a.extra_levels if r.has_conv]
  resamples += [r for cell in a.cells for node in cell['nodes'] for r in node.inputs if r.has_conv]
  out |= {(r.in_channels, F, False, False, NONE) for r in resamples}
  out.add((F, F, False, False, act if a.conv_bn_act_pattern else NONE))
  if F > ops.SEPCONV_MAX_C:
    out.add((F, F, False, False, act))
  out |= {(F, A * 4, False, False, NONE), (F, A * C, False, False, NONE)}
  return frozenset(out)


@functools.lru_cache(maxsize=None)
def cls_pw_shapes(name):
  """The 1x1 launches of EffNetV2Model: the MBConv blocks, the Fused-MBConv project (shared W,
  ACT_NONE, residual iff skip) and head_1x1 (act)."""
  v = effnetv2_model.EffNetV2Arch(name)
  out = _mbconv_pw([b for b in v.blocks if b.conv_type == 0], v.act)
  for b in v.blocks:
    if b.conv_type == 1 and b.expand_name:
      out.add((b.mid_filters, b.output_filters, False, bool(b.has_skip), NONE))
  out.add((v.blocks[-1].output_filters, v.head_filters, False, False, v.act))
  return frozenset(out)


def pw_shapes():
  """(k, nout, per-image W, residual, act) of every 1x1 launch of the registered models."""
  shapes = set()
  for name in DET_MODELS:
    for over in FPN_VARIANTS:
      shapes |= det_pw_shapes(name, over)
  for name in CLS_MODELS:
    shapes |= cls_pw_shapes(name)
  return sorted(shapes)


# ---------------------------------------------------------------------------------------------
# The shape-only part of the plan rule of pwtc::run() (pointwise_tc.cu), restated.  It must move
# with run(), as scripts/pw_plan_traffic.py does.
RESIDENT_W = 108 * 1024        # kResidentWBytes
SHARE_RES_MIN_KBLOCKS = 10     # kShareResMinKBlocks
SMEM_LIMIT = 227 * 1024        # kSmemLimit
# mbarriers of kMaxStages = 48 stages (full + empty), the work-unit ring (4 + 4), the resident-W
# pair and 6 residual barriers, then the 4-entry int4 tile ring
BARRIER_BYTES = (2 * 48 + 2 * 4 + 2 + 6) * 8 + 16 * 4


def plan(k, nout, per_image):
  """(block_n, block_k, number of N tiles, number of k-blocks, W bytes, resident at the default
  budget)."""
  block_n = _cdiv(nout, 32) * 32 if nout <= 128 else 128
  nnb = _cdiv(nout, block_n)

  def w_bytes(bk):
    return nnb * _cdiv(k, bk) * _cdiv(block_n * bk * 2, 1024) * 1024

  bk = 16 if k <= 16 else (32 if k <= 32 else 64)
  if bk == 64 and not per_image and w_bytes(64) > RESIDENT_W and w_bytes(32) <= RESIDENT_W:
    bk = 32
  return block_n, bk, nnb, _cdiv(k, bk), w_bytes(bk), not per_image and w_bytes(bk) <= RESIDENT_W


def plan_class(k, nout, per_image, residual):
  """(block_n, block_k, resident W, several N tiles, one k-block, residual with >= 10 k-blocks,
  per-image W): what the plan of a launch depends on besides the rows and the grid.  hold_a is
  open to resident W with several N tiles and one k-block."""
  block_n, bk, nnb, nkb, _, resident = plan(k, nout, per_image)
  return (block_n, bk, resident, nnb > 1, nkb == 1, residual and nkb >= SHARE_RES_MIN_KBLOCKS,
          per_image)


def refused(k, nout, per_image, teams, budget_kb):
  """Whether a pw_smem_kb budget (0: the default 227 KiB) refuses the launch: its fixed bytes --
  resident W (which streams instead when it would leave fewer than two A stages per consumer),
  one staging-slab set per consumer, the bias of whole N tiles, barriers -- must leave two stages
  per consumer."""
  block_n, bk, nnb, _, w_bytes, resident = plan(k, nout, per_image)
  limit = budget_kb * 1024 if budget_kb else SMEM_LIMIT
  a_stage = 64 * bk * 2
  fixed = teams * _cdiv(block_n, 64) * 64 * 64 * 2 + nnb * block_n * 4 + BARRIER_BYTES
  if resident and limit - 1024 - fixed - w_bytes >= 2 * teams * a_stage:
    return False
  return limit - 1024 - fixed < 2 * teams * (a_stage + _cdiv(block_n * bk * 2, 1024) * 1024)


def _setting_refuses(case, setting):
  _, _, k, nout, _, _, per_image, _ = case
  name, value = setting
  teams = value if name == 'pw_teams' else 2
  return refused(k, nout, per_image, teams, value if name == 'pw_smem_kb' else 0)


# ---------------------------------------------------------------------------------------------
def _cases():
  """One case per distinct registry (k, nout, per-image W, residual).  Rows small and ragged: the
  last 128-row tile alternately holds at most 64 rows (one consumer of the shared-W plan idle) and
  more.  Shared W at batch 1 (the whole batch as rows, as the models launch it), per-image W at
  batch 2 or 3.  The activations cycle through the registry's for the shape, so every activation
  meets each weight kind.  Every seventh case reads A with a pixel stride of k + 8."""
  acts = {}
  for k, nout, per_image, res, act in pw_shapes():
    acts.setdefault((k, nout, per_image, res), []).append(act)
  cases = []
  for i, (key, a) in enumerate(sorted(acts.items())):
    k, nout, per_image, res = key
    tail = 20 + (7 * i) % 45 if i % 2 == 0 else 70 + (11 * i) % 58
    rows = 128 * (i % 3) + tail
    batch = (2 + i % 2 if k * nout < 4 * 10**6 else 2) if per_image else 1
    lda = k + 8 if i % 7 == 3 else k
    cases.append((batch, rows, k, nout, a[(i // 2) % len(a)], res, per_image, lda))
  return cases


PW_CASES = _cases()


def _case_id(c):
  batch, rows, k, nout, act, res, per_image, lda = c
  return 'b%d_r%d_k%d_n%d_a%d%s%s%s' % (
      batch, rows, k, nout, act, '_res' if res else '', '_piw' if per_image else '',
      '_lda%d' % lda if lda != k else '')


def test_registry_shapes():
  """The edges the registry brings to the kernel."""
  shapes = pw_shapes()
  ks, ns = {s[0] for s in shapes}, {s[1] for s in shapes}
  assert (min(ks), max(ks), min(ns), max(ns)) == (16, 8256, 16, 8256)
  assert {n for n in ns if n % 8} == {36, 810}
  assert sum(1 for k in ks if k % 16 == 8) >= 10                     # a k16 step half past k
  assert max(_cdiv(n, 128) for n in ns) == 65 and max(_cdiv(k, 64) for k in ks) == 129
  # efficientnet-l2 blocks 83-87: expand to 8256 channels, SE-scaled project back with the skip
  assert (1376, 8256, False, False, SWISH) in shapes and (8256, 1376, True, True, NONE) in shapes
  # the class head's K values (the feature-network widths) on the fused arg-max path are those of
  # test_gpu_class_argmax, which checks it against this stored path
  class_ks = {k for k, n, _, _, _ in shapes if n == 810}
  assert class_ks == {64, 88, 112, 160, 200, 224, 288, 384}
  assert class_ks <= {c[2] for c in test_gpu_class_argmax.CASES}


def test_cases_cover_the_registry():
  shapes = pw_shapes()
  covered = {(c[2], c[3], c[6], c[5]) for c in PW_CASES}
  assert covered == {(k, n, piw, res) for k, n, piw, res, _ in shapes}
  assert len(covered) == len(PW_CASES)
  for per_image in (False, True):
    want = {act for _, _, piw, _, act in shapes if piw == per_image}
    assert {c[4] for c in PW_CASES if c[6] == per_image} == want, per_image
  assert {SWISH, RELU6, NONE} == {c[4] for c in PW_CASES if not c[6]}
  for batch, rows, k, nout, act, res, per_image, lda in PW_CASES:
    assert (batch == 1) != per_image
    assert (act, res, per_image, k, nout) in {(s[4], s[3], s[2], s[0], s[1]) for s in shapes}
  tails = {(c[1] - 1) % 128 + 1 for c in PW_CASES}
  assert min(tails) <= 64 < max(tails)
  assert sum(1 for c in PW_CASES if c[7] > c[2]) >= 10


def test_plan_classes_are_covered():
  """Every plan class of the registry has a case; each case's grid-dependent plans are reached at
  a pinned grid of plan_settings.GRIDS: with G = 1 every launch has a 128-row tile and an M block
  per CTA, so the shared-W plan (streamed W; with a residual, >= 10 k-blocks) and hold_a (resident
  W, several N tiles, one k-block) are taken where the shapes allow them."""
  reg = {plan_class(k, n, piw, res) for k, n, piw, res, _ in pw_shapes()}
  cases = {plan_class(c[2], c[3], c[6], c[5]) for c in PW_CASES}
  assert cases == reg
  assert len(reg) >= 25
  assert 1 in ps.GRIDS
  # each feature of the plan is met on both sides
  for i in range(len(next(iter(reg)))):
    assert len({c[i] for c in reg}) >= 2, i
  assert {c[1] for c in reg} == {16, 32, 64} and {c[0] for c in reg} >= {32, 64, 96, 128}
  assert any(c[2] and c[3] and c[4] for c in reg)                    # hold_a
  assert any(not c[2] and not c[6] for c in reg)                     # streamed shared W
  assert any(c[5] and c[6] for c in reg) and any(c[5] and not c[6] for c in reg)


def test_refusal_rule_matches_the_documented_floor():
  """refused() at the widest registry shape gives the floors of plan_settings / automl_b200.h."""
  wide = max(pw_shapes(), key=lambda s: (s[1], -s[0]))
  k, nout, piw = wide[0], wide[1], wide[2]
  assert nout == 8256
  for teams, floor in ((2, ps.SMEM_FLOOR_KB), (3, ps.SMEM_FLOOR_KB_3)):
    assert refused(k, nout, piw, teams, floor - 1) and not refused(k, nout, piw, teams, floor)
  # every registry shape runs at the default budget with two or three consumers
  for c in PW_CASES:
    assert not _setting_refuses(c, ('pw_teams', 2)) and not _setting_refuses(c, ('pw_teams', 3))


# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', PW_CASES, ids=_case_id)
def test_pointwise_registry(case):
  """float64 reference on the device, one fp16 ulp + 5e-5: the epilogue adds bias, activation and
  residual in fp32 and rounds once.  The same bits on two default runs and under every setting of
  plan_settings.SETTINGS (and pw_share_w = 1 on one CTA where W streams); a setting that refuses
  does so exactly where refused() says, before anything is launched."""
  batch, rows, k, nout, act, has_res, per_image, lda = case
  g = torch.Generator().manual_seed(7 * k + nout + rows + batch)
  a = torch.full((batch, rows, lda), float('nan')).half()
  a[..., :k] = torch.randn(batch, rows, k, generator=g).half()
  wb = batch if per_image else 1
  w = (torch.randn(wb, nout, k, generator=g) / k**0.5).half()
  bias = span_bias(nout, g, act != NONE)
  ldo = _round8(nout)
  res = torch.randn(batch, rows, ldo, generator=g).half() if has_res else None
  da, dw, db, dr = carve(a), carve(w if per_image else w[0]), carve(bias), carve(res)

  def launch(out):
    ops.pointwise_conv(da, dw, db, out.t, act, residual=dr, rows=rows, batch=batch, nout=nout)

  ps.reset(ops)
  outs = [Out((batch, rows, ldo)) for _ in range(2)]
  for out in outs:
    launch(out)
  got = outs[0].result()
  assert torch.equal(outs[1].result(), got), 'two default runs differ'
  ref = torch.einsum('brk,bnk->brn', da[..., :k].double(),
                     dw.double().view(wb, nout, k).expand(batch, nout, k))
  ref = act_ref(ref + db.double(), act)
  if has_res:
    ref = ref + dr[..., :nout].double()
  check_close(got[..., :nout], ref, _case_id(case))
  pad = got[..., nout:]
  assert bool(((pad == SENTINEL) | (pad == 0.0)).all())
  # error in fp16 ulps of the reference where the ulp is above the 5e-5 floor (|ref| >= 1/16)
  ref = ref.cpu()
  ulp = torch.from_numpy(np.spacing(ref.abs().numpy().astype(np.float16)).astype(np.float64))
  err = (got[..., :nout].double() - ref).abs()
  print('%s: max error %.3f ulp' % (_case_id(case), float((err / ulp)[ulp > 5e-5].max())))

  settings = list(ps.SETTINGS)
  if not plan(k, nout, per_image)[5]:
    settings.append(('pw_share_w', 1))
  for setting in settings:
    out = Out((batch, rows, ldo))

    def run():
      if setting[0] == 'pw_share_w':
        ops.set_option('max_ctas', 1)    # one CTA: the default plan would share W there
      launch(out)

    ran = ps.run_under(ops, setting, run)
    want_refused = setting[0] != 'pw_share_w' and _setting_refuses(case, setting)
    assert ran != want_refused, ps.setting_id(setting)
    if ran:
      assert torch.equal(out.result(), got), ps.setting_id(setting)
    else:
      assert bool((out.result() == SENTINEL).all()), ps.setting_id(setting)


# ---------------------------------------------------------------------------------------------
# drift guard: the models launch the registry's shapes
DRIFT_DETECTORS = [('efficientdet-d0', 128, ()), ('efficientdet-d7x', 256, ()),
                   ('efficientdet-lite0', 256, ()),
                   ('efficientdet-d0', 128,
                    (('fpn_name', 'qufpn'), ('conv_after_downsample', True)))]
DRIFT_CLASSIFIERS = [('efficientnet-b0', 64), ('efficientnetv2-s', 64), ('efficientnet-l2', 64)]


def _record(monkeypatch):
  """Wraps ops.pointwise_conv: returns the set the launches add (k, nout, wbatch > 1, residual,
  act) to."""
  seen = set()
  real = ops.pointwise_conv

  def spy(a, wt, bias, out, act, residual=None, **kw):
    n = kw.get('nout')
    seen.add((wt.shape[-1], n if n is not None else wt.shape[-2], wt.dim() == 3 and wt.shape[0] > 1,
              residual is not None, act))
    return real(a, wt, bias, out, act, residual=residual, **kw)

  monkeypatch.setattr(ops, 'pointwise_conv', spy)
  return seen


def _drift_id(v):
  return '-'.join('%s=%s' % o for o in v) if isinstance(v, tuple) else str(v)


@pytest.mark.gpu
@pytest.mark.parametrize('name,size,over', DRIFT_DETECTORS, ids=_drift_id)
def test_detector_launches_are_the_registry(name, size, over, monkeypatch):
  """One eager forward() of Engine (network only, so the class predict stores its logits) at
  batch 2: every (k, nout, per-image W, residual, act) it launches is in the registry, and every
  registry entry of the config is launched."""
  from automl_b200 import weights
  from automl_b200.engine import Engine
  seen = _record(monkeypatch)
  c = hparams_config.get_efficientdet_config(name)
  c.override(dict(over, image_size=size))
  w = weights.synthetic_weights(arch.DetArch(c), 0)
  eng = Engine(c, w, 2, device=DEV, use_cuda_graph=False)
  eng.forward(torch.zeros(2, size, size, 3))
  torch.cuda.synchronize()
  want = det_pw_shapes(name, over)
  assert seen <= set(pw_shapes()), sorted(seen - set(pw_shapes()))
  assert seen == want, (sorted(want - seen), sorted(seen - want))


@pytest.mark.gpu
@pytest.mark.parametrize('name,size', DRIFT_CLASSIFIERS)
def test_classifier_launches_are_the_registry(name, size, monkeypatch):
  """The same for one eager pass of EffNetV2Model at batch 2 (per-image SE weights)."""
  seen = _record(monkeypatch)
  model = effnetv2_model.get_model(name, batch_size=2, image_size=size, use_cuda_graph=False)
  model(torch.zeros(2, size, size, 3))
  torch.cuda.synchronize()
  want = cls_pw_shapes(name)
  assert seen <= set(pw_shapes()), sorted(seen - set(pw_shapes()))
  assert seen == want, (sorted(want - seen), sorted(seen - want))
