"""GPU parity of edet_class_argmax, the class-predict GEMM whose epilogue keeps, per pixel and
anchor, the maximum fp16-rounded logit, its first class and its sigmoid (one anchor per 96-column N
tile; pad columns have zero weights and a -inf bias).  Its scores and classes must be bit-identical
to edet_pre_nms run on the logits edet_pointwise_conv stores for the same unpadded GEMM, the class
must be an arg-max of the float64 logits, and every plan setting must give the same bits.  Entries
outside the level's anchor range keep their sentinel."""
import numpy as np
import pytest
import torch

import plan_settings as ps
from automl_b200 import utils

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
COLS = 96   # ops.CLASS_ARGMAX_COLS
SCORE_SENTINEL, CLASS_SENTINEL = -5.0, -7

# Every k here but lite3x's 200 is a multiple of 16, so the last k-step ends at k and the A columns
# past k never enter an MMA: the lda > k cases check the row pitch of the A map, not a K tail.  K 200
# ends in an 8-wide k16 step, whose other 8 columns are TMA zero fill (lda == k).  K-tail leakage
# (NaN past k in A) is tested on the A map the two paths share, in
# test_gpu_pointwise_plans.test_pointwise_strided_operands.  The arg-max kernel always has two
# consumers, so the pw_teams=3 setting runs the default plan.
CASES = [
    # anchors, classes, k, lda, batch, h, w, anchor_begin, anchors after the level
    (9, 90, 64, 64, 1, 40, 40, 0, 0),          # D0 level 3: 108 KiB of resident W (streamed at
                                               # 96 / 128 KiB); hold_a at G1 / G3 / G8
    (9, 96, 64, 72, 3, 10, 10, 700, 50),       # C = 96 (no -inf pad rows), lda > k; hold_a at G1 / G3
    (3, 20, 64, 64, 3, 8, 8, 0, 0),            # one 64-row M block per image; hold_a at G1 / G3
    (9, 90, 88, 88, 3, 5, 7, 270, 9),          # rows < 64, 2 k-blocks: W streamed
    (3, 20, 112, 128, 1, 33, 31, 123, 7),      # ragged rows, lda > k, resident W, 2 k-blocks
    (1, 1, 160, 168, 1, 17, 19, 5, 3),         # one class of one anchor, lda > k
    (3, 20, 160, 160, 3, 20, 21, 0, 11),       # D3 head width, resident W over 3 k-blocks
    (9, 90, 200, 200, 2, 13, 11, 40, 5),       # lite3x head width: streamed W, K tail of 8
    (9, 90, 224, 224, 1, 12, 12, 0, 0),        # D4 head width, streamed W
    (9, 90, 288, 296, 3, 9, 9, 11, 2),         # D5/D6 head width, streamed W, lda > k
    (9, 90, 384, 384, 1, 5, 5, 81, 0),         # D7 head width, streamed W
]


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _pad(w, b, na, nc):
  """Unpadded [na*nc, k] weights / [na*nc] bias -> the 96-row-per-anchor layout of the engine."""
  k = w.shape[-1]
  wpad = torch.zeros(na, COLS, k, dtype=w.dtype)
  wpad[:, :nc] = w.view(na, nc, k)
  bpad = torch.full((na, COLS), float('-inf'))
  bpad[:, :nc] = b.view(na, nc)
  return wpad.view(na * COLS, k), bpad.view(-1)


def _stored_path(ops, a, w, b, na, nc):
  """pointwise_conv stores the logits, pre_nms reduces them: (logits, scores, classes)."""
  n, h, wd, _ = a.shape
  rows = h * wd
  ld = -(-na * nc // 8) * 8
  logits = torch.empty(n, h, wd, ld, dtype=torch.float16, device=DEV)
  ops.pointwise_conv(a, w, b, logits, utils.ACT_NONE, rows=rows, batch=n, nout=na * nc)
  ld_box = -(-na * 4 // 8) * 8
  box = torch.zeros(n, h, wd, ld_box, dtype=torch.float16, device=DEV)
  anchors = torch.zeros(rows * na, 4, dtype=torch.float32, device=DEV)
  boxes = torch.empty(n, rows * na, 4, dtype=torch.float32, device=DEV)
  scores = torch.empty(n, rows * na, dtype=torch.float32, device=DEV)
  classes = torch.empty(n, rows * na, dtype=torch.int32, device=DEV)
  ops.pre_nms([logits], [box], [(h, wd)], na, nc, anchors, boxes, scores, classes)
  torch.cuda.synchronize()
  return logits, scores, classes


def _check(a, w, b, na, nc, anchor_begin, tail):
  """Runs the fused kernel under the default and every plan setting against the stored path;
  returns (stored logits, scores, classes) of the level's anchor range."""
  ops = _ops()
  n, h, wd, _ = a.shape
  rows = h * wd
  total = anchor_begin + rows * na + tail
  wpad, bpad = _pad(w, b, na, nc)
  da, dw, db = a.to(DEV), w.to(DEV), b.to(DEV)
  dwp, dbp = wpad.to(DEV), bpad.to(DEV)
  logits, want_s, want_c = _stored_path(ops, da, dw, db, na, nc)
  scores = torch.empty(n, total, dtype=torch.float32, device=DEV)
  classes = torch.empty(n, total, dtype=torch.int32, device=DEV)

  def launch():
    ops.class_argmax(da, dwp, dbp, scores, classes, anchor_begin, na)

  lo, hi = anchor_begin, anchor_begin + rows * na
  first = None
  for setting in [None] + ps.SETTINGS:
    scores.fill_(SCORE_SENTINEL)
    classes.fill_(CLASS_SENTINEL)
    # the arg-max plans (no staging slabs) fit every budget from 96 KiB up
    assert ps.run_under(ops, setting, launch), setting
    sid = 'default' if setting is None else ps.setting_id(setting)
    assert torch.equal(scores[:, lo:hi], want_s), sid
    assert torch.equal(classes[:, lo:hi], want_c), sid
    for t in (scores[:, :lo], scores[:, hi:]):
      assert bool((t == SCORE_SENTINEL).all()), sid
    for t in (classes[:, :lo], classes[:, hi:]):
      assert bool((t == CLASS_SENTINEL).all()), sid
    if first is None:
      first = (scores.clone(), classes.clone())
    else:
      assert torch.equal(scores, first[0]) and torch.equal(classes, first[1]), sid
  return logits.cpu(), scores[:, lo:hi].cpu(), classes[:, lo:hi].cpu()


@pytest.mark.parametrize('case', CASES)
def test_class_argmax(case):
  na, nc, k, lda, n, h, wd, anchor_begin, tail = case
  g = torch.Generator().manual_seed(11 + na * nc + k + h * wd)
  a = torch.randn(n, h, wd, lda, generator=g).half()
  w = (torch.randn(na * nc, k, generator=g) / np.sqrt(k)).half()
  b = torch.randn(na * nc, generator=g) - 2.0
  logits, scores, classes = _check(a, w, b, na, nc, anchor_begin, tail)
  rows = h * wd
  ref = torch.einsum('brk,nk->brn', a[..., :k].double().reshape(n, rows, k), w.double()) + b.double()
  ref = ref.view(n, rows, na, nc)
  cls = classes.reshape(n, rows, na).long()
  assert bool(((cls >= 0) & (cls < nc)).all())
  chosen = ref.gather(-1, cls.unsqueeze(-1)).squeeze(-1)
  best = ref.max(-1).values
  # fp32 accumulation, then fp16 rounding of both logits: 2 x 2^-11 relative
  assert bool((chosen >= best - (2.0**-10 * best.abs() + 1e-5)).all()), float((best - chosen).max())
  stored = logits[..., :na * nc].reshape(n, rows, na, nc).gather(-1, cls.unsqueeze(-1)).squeeze(-1)
  want = torch.sigmoid(stored.double())
  assert float((scores.reshape(n, rows, na).double() - want).abs().max()) <= 1e-6


def test_class_argmax_exact_ties():
  """Small-integer inputs make every logit exact, so equal maxima are common: the first (lowest)
  class must win, as in pre_nms.  Pixel 0 is all zeros: anchor 0's class 0 (negative weights, bias
  -0) then sums to -0 if the tensor cores produce one, class 1 (positive weights, bias -0) to +0,
  and every other class of that anchor to -1 or less; -0 and +0 are equal, so class 0 wins."""
  na, nc, k, n, h, wd = 3, 20, 64, 2, 9, 11
  g = torch.Generator().manual_seed(3)
  a = torch.randint(-1, 2, (n, h, wd, k), generator=g).half()
  a[:, 0, 0] = 0
  w = torch.randint(-1, 2, (na * nc, k), generator=g).half()
  w[0] = -1
  w[1] = 1
  b = torch.randint(-2, 3, (na * nc,), generator=g).float()
  b[0] = b[1] = -0.0
  b[2:nc] = torch.minimum(b[2:nc], torch.tensor(-1.0))
  logits, _, classes = _check(a, w, b, na, nc, 0, 0)
  rows = h * wd
  ref = torch.einsum('brk,nk->brn', a.double().view(n, rows, k), w.double()) + b.double()
  want = ref.view(n, rows, na, nc).argmax(-1)   # the first maximal index
  ties = (ref.view(n, rows, na, nc) == ref.view(n, rows, na, nc).max(-1, keepdim=True).values)
  assert int((ties.sum(-1) > 1).sum()) > 50   # the inputs do exercise ties (94 of 594 maxima)
  assert torch.equal(classes.reshape(n, rows, na).long(), want)
  assert bool((logits[:, 0, 0, :2] == 0).all())      # +-0, whichever sign the sum had
  assert bool((classes.reshape(n, rows, na)[:, 0, 0] == 0).all())
