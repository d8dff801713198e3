"""GPU parity of pointwise_tc_kernel on the tile plans that the resident-weight layout and the
32-column wgmma widths add: weights kept in shared memory for the whole launch (several N tiles,
several k-blocks), narrow layers whose N tile is wider than nout, and per-image (SE-scaled) weights
that keep streaming.  Both consumer organisations must give the same bits."""
import numpy as np
import pytest
import torch

from automl_b200 import utils

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

CASES = [
    # batch, rows, k, nout, act, residual, per-image weights
    (4, 1600, 32, 16, utils.ACT_NONE, False, True),      # blocks_0/project shape, SE weights
    (1, 3000, 32, 16, utils.ACT_NONE, False, False),     # nout 16 in a 32-column tile, resident W
    (2, 2000, 16, 96, utils.ACT_SWISH, False, False),    # blocks_1/expand shape, resident W
    (1, 1200, 480, 80, utils.ACT_NONE, True, False),     # 8 resident k-blocks (blocks_8 project)
    (1, 700, 80, 200, utils.ACT_SWISH, False, False),    # two resident N tiles, ragged last one
    (1, 900, 64, 760, utils.ACT_NONE, False, False),     # 6 resident N tiles, ragged last one
    (1, 500, 672, 192, utils.ACT_SWISH, True, False),    # W too large to stay: streamed
]


def _run(case, teams):
  from automl_b200 import ops  # deferred: loads the CUDA library
  batch, rows, k, nout, act, has_res, per_image = case
  g = torch.Generator().manual_seed(99 + rows + k + nout)
  a = torch.randn(batch, rows, k, generator=g).half()
  wb = batch if per_image else 1
  w = (torch.randn(wb, nout, k, generator=g) / np.sqrt(k)).half()
  bias = torch.randn(nout, generator=g)
  ldo = -(-nout // 8) * 8
  res = torch.randn(batch, rows, ldo, generator=g).half() if has_res else None
  out = torch.full((batch, rows, ldo), 7.0, dtype=torch.float16, device=DEV)
  try:
    ops.set_option('pw_teams', teams)
    ops.pointwise_conv(a.to(DEV), (w if per_image else w[0]).to(DEV), bias.to(DEV), out, act,
                       residual=res.to(DEV) if has_res else None, rows=rows, batch=batch, nout=nout)
    torch.cuda.synchronize()
  finally:
    ops.set_option('pw_teams', 0)
  ref = torch.einsum('brk,bnk->brn', a.double(), w.double().expand(batch, nout, k)) + bias.double()
  ref = {utils.ACT_NONE: lambda t: t, utils.ACT_SWISH: lambda t: t * torch.sigmoid(t)}[act](ref)
  if has_res:
    ref = ref + res[..., :nout].double()
  return out.cpu(), ref


@pytest.mark.parametrize('case', CASES)
def test_pointwise_tile_plans(case):
  nout = case[3]
  out2, ref = _run(case, 2)
  out3, _ = _run(case, 3)
  assert torch.equal(out2, out3)
  got = out2[..., :nout].double()
  # fp16 output rounding (2^-11 relative) + fp32 accumulation
  assert torch.allclose(got, ref, rtol=2e-3, atol=2e-3), float((got - ref).abs().max())
  pad = out2[..., nout:]
  assert bool(((pad == 7.0) | (pad == 0.0)).all())
