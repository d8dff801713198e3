"""edet_conv2d_transpose on its own: the sub-pixel wgmma Conv2DTranspose 3x3 stride 2 'SAME' of the
segmentation head (tf2/efficientdet_keras.py:676-706) against a float64 reference built from the
same fp16 inputs and Keras kernel with the transposed-convolution formula
out[y] = sum_i x[i] w[y - 2i] (per axis, y - 2i in {0, 1, 2}; pinned on the CPU in
test_segmentation_pins.py).  Covers one and two K sources, the D0-D7 widths, ragged maps, every
activation the head uses, strided sources, the output's padding columns and the grid."""
import numpy as np
import pytest
import torch

import plan_settings
from automl_b200 import utils

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6

CASES = [
    # h, w, batch, F, two sources, cout, act
    (1, 1, 1, 64, False, 64, NONE),
    (3, 5, 3, 64, True, 64, SWISH),
    (5, 5, 1, 88, True, 88, RELU6),
    (20, 24, 3, 88, True, 3, NONE),
    (40, 40, 1, 64, True, 3, NONE),
    (20, 24, 1, 224, True, 21, SWISH),
    (5, 5, 3, 384, True, 384, SWISH),
    (3, 5, 1, 384, False, 21, RELU6),
    (40, 40, 3, 64, False, 64, SWISH),
    (20, 24, 3, 224, False, 224, RELU6),
    (1, 1, 3, 88, True, 21, SWISH),
    (5, 5, 1, 224, True, 3, RELU6),
    (40, 40, 1, 88, True, 88, SWISH),
    (3, 5, 3, 64, True, 21, NONE),
]


def _r8(x):
  return (x + 7) // 8 * 8


def reference(x, kernel, bias, act):
  """float64 Conv2DTranspose 3x3 s2 'SAME': x [N,H,W,Cin], kernel [3,3,Cout,Cin] (Keras layout)."""
  n, h, w, _ = x.shape
  cout = kernel.shape[2]
  full = torch.zeros(n, 2 * h + 1, 2 * w + 1, cout, dtype=torch.float64, device=x.device)
  for ky in range(3):
    for kx in range(3):
      full[:, ky:ky + 2 * h:2, kx:kx + 2 * w:2] += torch.einsum('nhwc,oc->nhwo', x, kernel[ky, kx])
  out = full[:, :2 * h, :2 * w] + bias
  if act == SWISH:
    out = out * torch.sigmoid(out)
  elif act == RELU6:
    out = out.clamp(0, 6)
  return out


def make_case(h, w, batch, f, two, cout, act, seed, pad0=0, pad1=0):
  """fp16 sources (pixel strides f + pad), Keras kernel rounded to fp16, fp32 bias."""
  g = torch.Generator(device=DEV).manual_seed(seed)
  cin = 2 * f if two else f
  a0 = torch.randn(batch, h, w, f + pad0, generator=g, device=DEV).half()
  a1 = torch.randn(batch, h, w, f + pad1, generator=g, device=DEV).half() if two else None
  if pad0:
    a0[..., f:] = float('nan')
  if two and pad1:
    a1[..., f:] = float('nan')
  # outputs of std ~3 so that RELU6 and SWISH see both kinks
  kernel = (torch.randn(3, 3, cout, cin, generator=g, device=DEV) * (3.0 / (2.25 * cin) ** 0.5)).half()
  bias = torch.randn(cout, generator=g, device=DEV) * 2
  return a0, a1, kernel, bias


def run(a0, a1, kernel, bias, act, f, ldo=None, fill=0.0):
  from automl_b200 import ops  # deferred: loads the CUDA library
  n, h, w, _ = a0.shape
  cout = kernel.shape[2]
  wt = torch.as_tensor(ops.conv_transpose_weights(kernel.double().cpu().numpy(), f),
                       dtype=torch.float16, device=DEV)
  ldo = ldo or _r8(cout)
  out = torch.full((n, 2 * h, 2 * w, ldo), fill, dtype=torch.float16, device=DEV)
  ops.conv2d_transpose(a0, wt, bias, out, act, cout, a1=a1, c0=f, c1=f if a1 is not None else None)
  torch.cuda.synchronize()
  return out


def check_close(got, ref):
  """Within 1 fp16 ulp of the float64 reference, with an absolute floor for values near zero."""
  ulp = torch.from_numpy(np.spacing(np.abs(ref.cpu().numpy()).astype(np.float16)).astype(np.float64))
  err = (got.double().cpu() - ref.cpu()).abs()
  bad = err > ulp + 5e-5
  assert not bool(bad.any()), 'max err %g at %s' % (float(err.max()), tuple(bad.nonzero()[0].tolist()))


def sources_in(a0, a1, f):
  x = a0[..., :f]
  if a1 is not None:
    x = torch.cat([x, a1[..., :f]], dim=-1)
  return x.double()


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'h%dw%d_n%d_f%d_%s_c%d_a%d' % (
    c[0], c[1], c[2], c[3], 'two' if c[4] else 'one', c[5], c[6]))
def test_conv_transpose_matches_float64(case):
  h, w, batch, f, two, cout, act = case
  a0, a1, kernel, bias = make_case(*case, seed=h * 131 + w * 7 + f + cout + act)
  out = run(a0, a1, kernel, bias, act, f)
  ref = reference(sources_in(a0, a1, f), kernel.double(), bias.double(), act)
  check_close(out[..., :cout], ref)
  assert bool((out[..., cout:] == 0).all())   # channels cout .. round8(cout) are zero


@pytest.mark.parametrize('two', [False, True])
def test_strided_sources_and_output_sentinel(two):
  """Pixel strides wider than the channels (NaN in the gap must not reach the output) and an
  output wider than round8(cout) (the columns past it keep their sentinel)."""
  f, cout = 88, 21
  a0, a1, kernel, bias = make_case(5, 20, 2, f, two, cout, SWISH, seed=5, pad0=16, pad1=8)
  out = run(a0, a1, kernel, bias, SWISH, f, ldo=40, fill=7.0)
  ref = reference(sources_in(a0, a1, f), kernel.double(), bias.double(), SWISH)
  check_close(out[..., :cout], ref)
  assert bool((out[..., cout:24] == 0).all())
  assert bool((out[..., 24:] == 7.0).all())


@pytest.mark.parametrize('grid', plan_settings.GRIDS)
def test_same_bits_for_every_grid(grid):
  """Two launches, and grids pinned to 1/3/8/33 CTAs, give the bits of the default grid."""
  from automl_b200 import ops
  case = (20, 24, 3, 88, True, 21, SWISH)
  a0, a1, kernel, bias = make_case(*case, seed=11)
  base = run(a0, a1, kernel, bias, SWISH, 88)
  again = run(a0, a1, kernel, bias, SWISH, 88)
  assert torch.equal(base, again)
  outs = []
  assert plan_settings.run_under(ops, ('grid', grid),
                                 lambda: outs.append(run(a0, a1, kernel, bias, SWISH, 88)))
  assert torch.equal(base, outs[0])


def test_rejects_bad_arguments():
  from automl_b200 import ops
  from automl_b200._lib import EdetError
  a0, _, kernel, bias = make_case(3, 3, 1, 64, False, 8, NONE, seed=1)
  wt = torch.as_tensor(ops.conv_transpose_weights(kernel.double().cpu().numpy(), 64),
                       dtype=torch.float16, device=DEV)
  out = torch.zeros(1, 6, 6, 8, dtype=torch.float16, device=DEV)
  with pytest.raises(EdetError):
    ops.conv2d_transpose(a0, wt, bias, out, utils.ACT_SIGMOID, 8)
  with pytest.raises(ValueError):
    ops.conv2d_transpose(a0, wt, bias, out[:, :5], NONE, 8)
