"""GPU parity of pointwise_tc_kernel across the launch plans pwtc::run() derives from the shapes and
the options: N tile width (block_n), k-block width (block_k), resident or streamed W, A held over
every N tile (hold_a), work units of 1 / 2 / 4 / 8 M blocks, one or two slab sets, the stages per
consumer and the grid.  Each case is checked once against a float64 einsum; every other setting
(plan_settings.SETTINGS) must give the same bits, since only the schedule changes -- block_n and
block_k do not depend on the options, so neither do the MMA and epilogue arithmetic.  The plan
named next to each case is the one a pinned grid G selects (G = 1 / 3 / 8 / 33), which does not
depend on the SM count.

Also: operands with pixel strides wider than the data (lda > k, ldr > nout, ldo > round8(nout)),
for both implementations, and the shared-memory budget floor of include/automl_b200.h."""
import numpy as np
import pytest
import torch

import plan_settings as ps
from automl_b200 import utils

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SENTINEL = 7.0


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def rel_l2(a, b):
  a, b = a.double().flatten(), b.double().flatten()
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


ACT_REF = {utils.ACT_NONE: lambda t: t, utils.ACT_SWISH: lambda t: t * torch.sigmoid(t),
           utils.ACT_RELU6: lambda t: torch.clamp(t, 0, 6)}

CASES = [
    # batch, rows, k, nout, act, residual, per-image weights
    (1, 5000, 16, 32, utils.ACT_NONE, False, False),     # block_k 16, block_n 32, resident W;
                                                         # G1: units of 8, last one 7; G3: of 2
    (2, 3000, 24, 64, utils.ACT_SWISH, False, False),    # block_k 32 (K tail 24), block_n 64;
                                                         # G1: units of 8 (last 7), G3: of 4 (last 3)
    (1, 2000, 64, 96, utils.ACT_RELU6, False, False),    # block_k 64, block_n 96; 96 KiB: one slab
                                                         # set, 3 stages; G1: units of 4
    (1, 1500, 128, 128, utils.ACT_NONE, True, False),    # block_n 128, two resident k-blocks,
                                                         # residual; 96 KiB: refused; G1: units of 2
    (1, 1000, 64, 400, utils.ACT_SWISH, False, False),   # four 128-wide N tiles (last one 16):
                                                         # hold_a at G1 / G3 / G8, not at G33
    (2, 4100, 24, 144, utils.ACT_SWISH, False, False),   # hold_a over 2 N tiles with units of 2
                                                         # M blocks (last one 1) at G1 / G3 / G8
    (4, 6000, 32, 16, utils.ACT_NONE, False, True),      # streamed per-image W; G1 / G3: units of
                                                         # 8 (last 6), G8: of 4 (last 2)
    (1, 1200, 480, 80, utils.ACT_NONE, True, False),     # blocks_8/project: 8 resident k-blocks;
                                                         # 128 / 160 KiB: W streams instead
    (3, 40, 64, 200, utils.ACT_NONE, False, False),      # rows < 64, 2 N tiles; hold_a at G1 / G3
    (1, 25, 64, 36, utils.ACT_NONE, False, False),       # box-predict on a 5x5 level: one unit
    (1, 700, 672, 192, utils.ACT_SWISH, True, False),    # W too large to stay: 11 streamed
                                                         # k-blocks x 2 N tiles
    (2, 400, 1152, 192, utils.ACT_NONE, True, True),     # streamed per-image W, deep K, residual
]


def _inputs(case, seed):
  batch, rows, k, nout, act, has_res, per_image = case
  g = torch.Generator().manual_seed(seed + rows + k + nout)
  a = torch.randn(batch, rows, k, generator=g).half()
  wb = batch if per_image else 1
  w = (torch.randn(wb, nout, k, generator=g) / np.sqrt(k)).half()
  bias = torch.randn(nout, generator=g)
  ldo = -(-nout // 8) * 8
  res = torch.randn(batch, rows, ldo, generator=g).half() if has_res else None
  return a, w, bias, res


def _reference(a, w, bias, res, act, nout):
  batch, _, k = a.shape
  ref = torch.einsum('brk,bnk->brn', a.double(), w.double().expand(batch, nout, k))
  ref = ACT_REF[act](ref + bias.double())
  if res is not None:
    ref = ref + res[..., :nout].double()
  return ref


@pytest.mark.parametrize('case', CASES)
def test_pointwise_plans_agree(case):
  ops = _ops()
  batch, rows, k, nout, act, has_res, per_image = case
  a, w, bias, res = _inputs(case, 31)
  ldo = -(-nout // 8) * 8
  da, dw, db = a.to(DEV), (w if per_image else w[0]).to(DEV), bias.to(DEV)
  dr = res.to(DEV) if has_res else None
  out = torch.empty(batch, rows, ldo, dtype=torch.float16, device=DEV)

  def launch():
    ops.pointwise_conv(da, dw, db, out, act, residual=dr, rows=rows, batch=batch, nout=nout)

  out.fill_(SENTINEL)
  assert ps.run_under(ops, None, launch)
  want = out.clone()
  got = want.cpu()[..., :nout].double()
  ref = _reference(a, w, bias, res, act, nout)
  # fp16 output rounding (2^-11 relative) + fp32 accumulation
  assert torch.allclose(got, ref, rtol=2e-3, atol=2e-3), float((got - ref).abs().max())
  assert rel_l2(got, ref) < 5e-4
  pad = want[..., nout:]
  assert bool(((pad == SENTINEL) | (pad == 0.0)).all())
  for setting in ps.SETTINGS:
    out.fill_(SENTINEL)
    ran = ps.run_under(ops, setting, launch)
    if not ran:
      # a budget the plan cannot hold is refused before anything is launched
      assert not ps.must_run(setting), 'refused at %s' % ps.setting_id(setting)
      assert bool((out == SENTINEL).all()), ps.setting_id(setting)
      continue
    assert torch.equal(out, want), ps.setting_id(setting)


# (consumers, floor in KiB, nout): the widest registered layer, efficientnet-l2's nout 8256 (65 N
# tiles), sets the documented floor; nout 8192 (64 tiles) stages 0.5 KiB less bias and runs from
# 1 KiB lower
FLOOR_CASES = [(2, 162, 8192), (3, 226, 8192),
               (2, ps.SMEM_FLOOR_KB, 8256), (3, ps.SMEM_FLOOR_KB_3, 8256)]


@pytest.mark.parametrize('teams,floor_kb,nout', FLOOR_CASES,
                         ids=['%d-%d' % c[:2] for c in FLOOR_CASES])
def test_pointwise_smem_floor(teams, floor_kb, nout):
  """The widest plans -- 128-column N tiles, 128 x 64 W tiles streamed with a 64 x 64 A tile, the
  bias of every N tile in shared memory -- run from their floor up and are refused 1 KiB below it:
  the bias copy is sized per launch."""
  ops = _ops()
  batch, rows, k = 1, 100, 64
  case = (batch, rows, k, nout, utils.ACT_NONE, False, False)
  a, w, bias, _ = _inputs(case, 5)
  da, dw, db = a.to(DEV), w[0].to(DEV), bias.to(DEV)
  out = torch.empty(batch, rows, nout, dtype=torch.float16, device=DEV)

  def launch():
    ops.pointwise_conv(da, dw, db, out, utils.ACT_NONE, rows=rows, batch=batch, nout=nout)

  out.fill_(SENTINEL)
  assert ps.run_under(ops, None, launch)
  want = out.clone()
  ref = _reference(a, w, bias, None, utils.ACT_NONE, nout)
  assert torch.allclose(want.cpu().double(), ref, rtol=2e-3, atol=2e-3)
  try:
    ops.set_option('pw_teams', teams)
    out.fill_(SENTINEL)
    assert not ps.run_under(ops, ('pw_smem_kb', floor_kb - 1), launch)
    assert bool((out == SENTINEL).all())
    ops.set_option('pw_teams', teams)
    assert ps.run_under(ops, ('pw_smem_kb', floor_kb), launch)
  finally:
    ps.reset(ops)
  assert torch.equal(out, want)


# ---------------------------------------------------------------------------------------------
STRIDED_CASES = [
    # batch, rows, k, lda, nout, ldr, ldo, act, residual, per-image weights
    (2, 1000, 40, 64, 72, 88, 88, utils.ACT_SWISH, True, True),     # K tail 40 of a 64 k-block,
                                                                    # per-image W
    (1, 700, 24, 40, 100, 0, 120, utils.ACT_NONE, False, False),    # 32B rows, nout % 8 != 0
    (3, 300, 200, 208, 48, 64, 56, utils.ACT_NONE, True, True),     # 4 k-blocks, last one 8 wide
    (1, 900, 80, 96, 200, 0, 216, utils.ACT_RELU6, False, False),   # 2 N tiles, resident W
]


@pytest.mark.parametrize('impl_name', ['tcgen05', 'simt'])
@pytest.mark.parametrize('case', STRIDED_CASES)
def test_pointwise_strided_operands(case, impl_name):
  """Pixel strides wider than the data: A columns k..lda, residual columns nout..ldr hold NaN and
  must not reach the output; output columns past round8(nout) are never written, those in
  [nout, round8(nout)) only with zeros."""
  ops = _ops()
  impl = ops.PW_TCGEN05 if impl_name == 'tcgen05' else ops.PW_SIMT
  batch, rows, k, lda, nout, ldr, ldo, act, has_res, per_image = case
  g = torch.Generator().manual_seed(17 + rows + k + nout)
  a = torch.full((batch, rows, lda), float('nan')).half()
  a[..., :k] = torch.randn(batch, rows, k, generator=g).half()
  wb = batch if per_image else 1
  w = (torch.randn(wb, nout, k, generator=g) / np.sqrt(k)).half()
  bias = torch.randn(nout, generator=g)
  res = None
  if has_res:
    res = torch.full((batch, rows, ldr), float('nan')).half()
    res[..., :nout] = torch.randn(batch, rows, nout, generator=g).half()
  out = torch.full((batch, rows, ldo), SENTINEL, dtype=torch.float16, device=DEV)
  ops.pointwise_conv(a.to(DEV), (w if per_image else w[0]).to(DEV), bias.to(DEV), out, act,
                     residual=res.to(DEV) if has_res else None, rows=rows, batch=batch, nout=nout,
                     impl=impl)
  torch.cuda.synchronize()
  out = out.cpu()
  assert not bool(out.isnan().any())
  ref = _reference(a[..., :k], w, bias, res, act, nout)
  got = out[..., :nout].double()
  assert torch.allclose(got, ref, rtol=2e-3, atol=2e-3), float((got - ref).abs().max())
  assert rel_l2(got, ref) < 5e-4
  n8 = -(-nout // 8) * 8
  assert bool((out[..., n8:] == SENTINEL).all())
  pad = out[..., nout:n8]
  assert bool(((pad == SENTINEL) | (pad == 0.0)).all())


# ---------------------------------------------------------------------------------------------
def test_depthwise_tiled_persist_slack():
  """The TMA-tiled depthwise kernel is the other persistent kernel that leaves persist_slack CTAs
  out of its grid (2 x sm_count - slack, at most one CTA per work unit) and whose grid max_ctas
  pins: output bits and SE integers (per-unit sums, 2^-20 fixed point) must not depend on either."""
  ops = _ops()
  # 5x5 stride 1 runs on the tiled kernel when its 8 x 16 output tiles cover the map with <= 30 %
  # waste (dwt::eligible): 80 x 80 is covered exactly.  10 x 5 tiles x 11 64-channel slices = 550
  # work units, more than 2 x 132, so on a 132-SM H100 the grid is 264 / 198 / 132 CTAs.
  n, h, w, c, k, s = 1, 80, 80, 672, 5, 1
  g = torch.Generator().manual_seed(2024)
  x = torch.randn(n, h, w, c, generator=g).half().to(DEV)
  wk = (torch.randn(k * k, c, generator=g) / k).to(DEV)
  bias = (torch.randn(c, generator=g) * 0.1).to(DEV)
  outs, sums = [], []
  settings = [('persist_slack', v) for v in (0, 66, 132)] + [('max_ctas', g) for g in ps.GRIDS]
  for opt, value in settings:
    out = torch.empty(n, h, w, c, dtype=torch.float16, device=DEV)
    part = torch.zeros(n, c, dtype=torch.int64, device=DEV)
    try:
      ops.set_option(opt, value)
      ops.depthwise_conv(x, out, wk, bias, utils.ACT_SWISH, k, s, part)
      torch.cuda.synchronize()
    finally:
      ops.set_option(opt, 0)
    outs.append(out)
    sums.append(part)
  for i in range(1, len(settings)):
    assert torch.equal(outs[i], outs[0]), settings[i]
    assert torch.equal(sums[i], sums[0]), settings[i]
  # and the register-tiled kernel, which does the same fp32 arithmetic, gives the same output bits
  reg = torch.empty(n, h, w, c, dtype=torch.float16, device=DEV)
  try:
    ops.set_option('dw_impl', 1)
    ops.depthwise_conv(x, reg, wk, bias, utils.ACT_SWISH, k, s, None)
    torch.cuda.synchronize()
  finally:
    ops.set_option('dw_impl', 0)
  assert torch.equal(reg, outs[0])
