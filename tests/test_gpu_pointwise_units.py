"""GPU parity of pointwise_tc_kernel's work units: up to 8 consecutive 64-row M blocks of one image
per scheduler claim (the last unit of an image shorter), and units that load an A tile once for
every N tile when W is resident and K fits one k-block.  The unit size follows from the shapes and
the SM count; the comments give what a 132-SM H100 picks.  Both consumer organisations must give
the same bits."""
import pytest
import torch

from automl_b200 import utils

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

CASES = [
    # batch, rows, k, nout, act, residual, per-image weights
    (2, 270000, 32, 16, utils.ACT_NONE, False, True),     # blocks_0/project: streamed SE weights,
                                                          # 8 M blocks per unit, last one 3
    (3, 44990, 24, 144, utils.ACT_SWISH, False, False),   # A held over 2 N tiles (ragged last),
                                                          # 2 M blocks per unit, last one 1
    (4, 40000, 96, 24, utils.ACT_NONE, True, False),      # two k-blocks + residual, 2 per unit
    (2, 100000, 16, 96, utils.ACT_SWISH, False, False),   # blocks_1/expand, 2 per unit
    (1, 3000, 64, 96, utils.ACT_SWISH, False, False),     # 47 units for 132 CTAs
    (3, 40, 64, 200, utils.ACT_NONE, False, False),       # rows < 64, 2 N tiles (too few M
                                                          # blocks to hold A)
]


def _run(case, teams):
  from automl_b200 import ops  # deferred: loads the CUDA library
  batch, rows, k, nout, act, has_res, per_image = case
  g = torch.Generator(device=DEV).manual_seed(7 + rows + k + nout)
  a = torch.randn(batch, rows, k, generator=g, device=DEV).half()
  wb = batch if per_image else 1
  w = (torch.randn(wb, nout, k, generator=g, device=DEV) / k ** 0.5).half()
  bias = torch.randn(nout, generator=g, device=DEV)
  ldo = -(-nout // 8) * 8
  res = torch.randn(batch, rows, ldo, generator=g, device=DEV).half() if has_res else None
  out = torch.full((batch, rows, ldo), 7.0, dtype=torch.float16, device=DEV)
  try:
    ops.set_option('pw_teams', teams)
    ops.pointwise_conv(a, w if per_image else w[0], bias, out, act, residual=res, rows=rows,
                       batch=batch, nout=nout)
    torch.cuda.synchronize()
  finally:
    ops.set_option('pw_teams', 0)
  ref = torch.einsum('brk,bnk->brn', a.double(), w.double().expand(batch, nout, k)) + bias.double()
  ref = {utils.ACT_NONE: lambda t: t, utils.ACT_SWISH: lambda t: t * torch.sigmoid(t)}[act](ref)
  if has_res:
    ref = ref + res[..., :nout].double()
  return out, ref


@pytest.mark.parametrize('case', CASES)
def test_pointwise_work_units(case):
  nout = case[3]
  out2, ref = _run(case, 2)
  out3, _ = _run(case, 3)
  assert torch.equal(out2, out3)
  got = out2[..., :nout].double()
  # fp16 output rounding (2^-11 relative) + fp32 accumulation
  assert torch.allclose(got, ref, rtol=2e-3, atol=2e-3), float((got - ref).abs().max())
  pad = out2[..., nout:]
  assert bool(((pad == 7.0) | (pad == 0.0)).all())
