"""GPU parity of pointwise_tc_kernel's shared-W plan: where W streams with A (per-image SE weights,
or shared weights too large to stay in shared memory), both consumers of a CTA compute one 128-row
tile against one W tile per k-block, instead of one 64-row tile each with a W tile of its own.  Per
output the k16 products are summed in the same order either way, so the plan must give the bits of
the 64-row plan that edet_set_option("pw_share_w", 1) forces -- at the D0 640x640 batch-32 shapes of
the deep backbone, on images whose last 128-row tile is ragged, on pinned grids (one CTA wraps the
shared ring many times), and where the budget or three consumers fall back to 64-row tiles.  Each
case is also checked once against a float64 einsum with the bounds of test_gpu_pointwise_plans."""
import pytest
import torch

from automl_b200 import utils
from automl_b200._lib import EdetError

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SENTINEL = 7.0

CASES = [
    # batch, rows, k, nout, act, residual, per-image weights
    (32, 1600, 80, 480, utils.ACT_SWISH, False, False),     # blocks_6/expand: 32-wide k-blocks,
                                                            # W resident (no shared-W plan)
    (32, 1600, 112, 672, utils.ACT_SWISH, False, False),    # blocks_9/expand: streamed W, 6 N tiles
    (32, 1600, 672, 112, utils.ACT_NONE, True, True),       # blocks_9/project: SE weights, residual
    (32, 400, 192, 1152, utils.ACT_SWISH, False, False),    # blocks_12/expand: 9 N tiles
    (32, 400, 1152, 192, utils.ACT_NONE, True, True),       # blocks_12/project: last tile 16 rows
    (32, 400, 1152, 320, utils.ACT_NONE, False, True),      # blocks_15/project: 3 N tiles
    (3, 1050, 672, 96, utils.ACT_SWISH, True, True),        # last tile 26 rows: one consumer idle
    (5, 1000, 136, 200, utils.ACT_RELU6, False, True),      # last tile 104 rows, 2 N tiles, K tail 8
]
# Pinned grids: with at least one 128-row tile per CTA every case whose W streams takes the shared-W
# plan (at the default grid the two small ragged cases have too few tiles and keep 64-row tiles).
GRIDS = (1, 3)

ACT_REF = {utils.ACT_NONE: lambda t: t, utils.ACT_SWISH: lambda t: t * torch.sigmoid(t),
           utils.ACT_RELU6: lambda t: torch.clamp(t, 0, 6)}


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _reset(ops):
  for opt in ('pw_share_w', 'pw_teams', 'pw_smem_kb', 'max_ctas'):
    ops.set_option(opt, 0)


class _Case:

  def __init__(self, case, seed=11):
    self.batch, self.rows, self.k, self.nout, self.act, has_res, per_image = case
    g = torch.Generator(device=DEV).manual_seed(seed + self.rows + self.k + self.nout)
    self.a = torch.randn(self.batch, self.rows, self.k, generator=g, device=DEV).half()
    wb = self.batch if per_image else 1
    self.w = (torch.randn(wb, self.nout, self.k, generator=g, device=DEV) / self.k ** 0.5).half()
    self.wt = self.w if per_image else self.w[0]
    self.bias = torch.randn(self.nout, generator=g, device=DEV)
    self.ldo = -(-self.nout // 8) * 8
    self.res = (torch.randn(self.batch, self.rows, self.ldo, generator=g, device=DEV).half()
                if has_res else None)

  def run(self, **options):
    """Output under `options` (edet_set_option name -> value), all reset afterwards."""
    ops = _ops()
    out = torch.full((self.batch, self.rows, self.ldo), SENTINEL, dtype=torch.float16, device=DEV)
    try:
      for name, value in options.items():
        ops.set_option(name, value)
      ops.pointwise_conv(self.a, self.wt, self.bias, out, self.act, residual=self.res,
                         rows=self.rows, batch=self.batch, nout=self.nout)
      torch.cuda.synchronize()
    finally:
      _reset(ops)
    return out

  def check_reference(self, out):
    ref = torch.einsum('brk,bnk->brn', self.a.double(),
                       self.w.double().expand(self.batch, self.nout, self.k))
    ref = ACT_REF[self.act](ref + self.bias.double())
    if self.res is not None:
      ref = ref + self.res[..., :self.nout].double()
    got = out[..., :self.nout].double()
    # fp16 output rounding (2^-11 relative) + fp32 accumulation
    assert torch.allclose(got, ref, rtol=2e-3, atol=2e-3), float((got - ref).abs().max())
    assert float((got - ref).norm() / ref.norm()) < 5e-4
    pad = out[..., self.nout:]
    assert bool(((pad == SENTINEL) | (pad == 0.0)).all())


@pytest.mark.parametrize('case', CASES)
def test_shared_w_plan_matches_64_row_plan(case):
  c = _Case(case)
  want = c.run()
  c.check_reference(want)
  assert torch.equal(c.run(pw_share_w=1), want)
  for grid in GRIDS:
    assert torch.equal(c.run(max_ctas=grid), want), 'grid %d' % grid
    assert torch.equal(c.run(max_ctas=grid, pw_share_w=1), want), 'grid %d, 64-row' % grid


@pytest.mark.parametrize('options', [
    {'pw_smem_kb': 160},   # 64-row stages fit, four 32 KiB shared stages do not: 64-row tiles
    {'pw_smem_kb': 192},   # one slab set per consumer next to four shared stages
    {'pw_teams': 3},       # three consumers always take 64-row tiles
    {'pw_smem_kb': 160, 'max_ctas': 3},
])
def test_shared_w_fallback(options):
  c = _Case((32, 400, 1152, 192, utils.ACT_NONE, True, True))   # blocks_12/project
  want = c.run()
  c.check_reference(want)
  assert torch.equal(c.run(**options), want)


def test_shared_w_option_is_reset():
  ops = _ops()
  _Case((2, 300, 640, 64, utils.ACT_NONE, False, True)).run(pw_share_w=1)
  assert ops.get_option('pw_share_w') == 0
  with pytest.raises(EdetError):
    ops.set_option('pw_share_w', 2)
