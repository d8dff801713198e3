"""Classification from decoded images on the device: the eval pre-process kernel
(edet_cls_preprocess, both recipes) bit-identical to tests/classify_oracle.py, the softmax top-k
kernel (edet_softmax_topk) against a stable sort and float64 softmax, and
EffNetV2Model.preprocess / classify / classify_stream end to end against the oracle chain
(oracle pre-process -> EffNetV2Oracle + top -> float64 softmax top-k).

Probability bound of edet_softmax_topk.  u = 2^-24.  Every expf is within 2 ulp (<= 4 u relative);
the float32 difference l - max is rounded once, which perturbs exp by a relative u |l - max|.
The sum runs a thread chain of ceil(C / 256) terms (its first add is exact), 5 shuffle levels
and 3 levels over the 8 warps: depth d = ceil(C / 256) + 7, all terms positive, so a relative
error of at most (4 + R + d) u with R the row's max - min.  The numerator adds (4 + |l - max|) u,
the division u:  |p - p64| <= (9 + d + R + |l - max|) u p64, with 1 % for the higher orders.
"""
import ctypes

import numpy as np
import pytest
import torch

import classify_oracle as co
import effnetv2_top_oracle
from automl_b200.efficientnetv2 import effnetv2_model
from automl_b200.efficientnetv2 import preprocessing

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
U = 2.0**-24
GUARD = 256
CANARY = -12345.5


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _images(shapes, seed):
  rng = np.random.default_rng(seed)
  return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes]


def _kernel(images, size, legacy, windows=None):
  """One edet_cls_preprocess launch over `images` -> float32 [N, S, S, 3] (canaries checked)."""
  ops = _ops()
  desc, total = preprocessing.image_table([im.shape[:2] for im in images], size,
                                          legacy) if windows is None else _table(images, windows)
  packed = np.concatenate([im.reshape(-1) for im in images])
  assert packed.size == total
  n = len(images)
  numel = n * size * size * 3
  buf = torch.full((numel + GUARD,), CANARY, dtype=torch.float32, device=DEV)
  ops.cls_preprocess(torch.from_numpy(packed).to(DEV), torch.from_numpy(desc).to(DEV),
                     buf[:numel].view(n, size, size, 3), ops.CLS_BICUBIC if legacy else ops.CLS_BILINEAR,
                     preprocessing.device_table(DEV) if legacy else None)
  torch.cuda.synchronize()
  assert bool((buf[numel:] == CANARY).all()), 'written past the end of the output'
  return buf[:numel].view(n, size, size, 3).cpu()


def _table(images, windows):
  desc, total = preprocessing.image_table([(1, 1)] * len(images), 384, False)
  off = 0
  for i, (im, win) in enumerate(zip(images, windows)):
    desc[i:i + 1, :2].view(np.int64)[0, 0] = off
    desc[i, 2:] = im.shape[:2] + tuple(win)
    off += im.size
  return desc, off


def _oracle_window(im, size, legacy):
  h, w = im.shape[:2]
  try:
    return co.crop_window(h, w, size, legacy)
  except ValueError:          # a 1-pixel side has no eval crop: resize the whole image
    return (0, 0, h, w)


SHAPES = [(375, 500), (500, 375), (333, 501), (224, 224), (384, 384), (100, 150), (1, 300),
          (300, 1), (900, 1200), (7, 5)]
RECIPES = [(224, False), (224, True), (384, False), (384, True), (260, True)]


# ---- pre-process kernel -------------------------------------------------------------------------
@pytest.mark.parametrize('size,legacy', RECIPES)
@pytest.mark.parametrize('shape', SHAPES)
def test_preprocess_kernel_bit_identical(shape, size, legacy):
  im = _images([shape], shape[0] * 7 + shape[1])[0]
  win = _oracle_window(im, size, legacy)
  got = _kernel([im], size, legacy, [win])[0]
  ref = co.preprocess_window(im, size, legacy, win)
  assert got.dtype == torch.float32
  assert torch.equal(got, torch.from_numpy(ref)), float((got - torch.from_numpy(ref)).abs().max())


@pytest.mark.parametrize('size,legacy', RECIPES)
def test_ragged_batch_in_one_launch_equals_one_launch_per_image(size, legacy):
  shapes = [s for s in SHAPES if min(s) > 1]
  ims = _images(shapes, 5)
  got = _kernel(ims, size, legacy)
  for i, im in enumerate(ims):
    assert torch.equal(got[i], _kernel([im], size, legacy)[0]), shapes[i]
    assert torch.equal(got[i], torch.from_numpy(co.preprocess_image(im, size, legacy))), shapes[i]


@pytest.mark.parametrize('augname,size', [('randaug', 384), ('randaug', 224), ('effnetv1_autoaug', 224)])
def test_preprocess_image(augname, size):
  im = _images([(375, 500)], 3)[0]
  got = preprocessing.preprocess_image(im, size, augname=augname, image_dtype=np.float32)
  assert got.is_cuda and got.dtype == torch.float32 and tuple(got.shape) == (size, size, 3)
  ref = co.preprocess_image(im, size, preprocessing.is_legacy(augname))
  assert torch.equal(got.cpu(), torch.from_numpy(ref))
  assert torch.equal(preprocessing.preprocess_image(torch.from_numpy(im), size, augname=augname), got)


# ---- softmax top-k ------------------------------------------------------------------------------
def _topk(logits, k):
  ops = _ops()
  n = logits.shape[0]
  buf_p = torch.full((n * k + GUARD,), CANARY, dtype=torch.float32, device=DEV)
  buf_c = torch.full((n * k + GUARD,), -7, dtype=torch.int32, device=DEV)
  ops.softmax_topk(logits, buf_p[:n * k].view(n, k), buf_c[:n * k].view(n, k))
  torch.cuda.synchronize()
  assert bool((buf_p[n * k:] == CANARY).all()) and bool((buf_c[n * k:] == -7).all())
  return buf_p[:n * k].view(n, k).cpu(), buf_c[:n * k].view(n, k).cpu()


def _check_topk(logits, probs, classes):
  x = logits.cpu().numpy()
  k = probs.shape[1]
  p64, c64 = co.softmax_topk(x, k)
  assert np.array_equal(classes.numpy(), c64)
  x64 = x.astype(np.float64)
  mx = x64.max(1, keepdims=True)
  r = mx - x64.min(1, keepdims=True)
  d = -(-x.shape[1] // 256) + 7
  sel = np.take_along_axis(x64, c64, 1)
  bound = (9 + d + r + (mx - sel)) * U * p64 * 1.01
  err = np.abs(probs.numpy().astype(np.float64) - p64)
  assert (err <= bound).all(), float((err / bound).max())


@pytest.mark.parametrize('c,k', [(10, 1), (10, 5), (10, 10)] + [
    (c, k) for c in (1000, 1001, 21843) for k in (1, 5, 32)])
def test_softmax_topk(c, k):
  g = torch.Generator(device=DEV).manual_seed(c * 40 + k)
  logits = torch.randn((128, c), generator=g, device=DEV) * 3
  logits[1] = torch.round(logits[1] * 2) / 2               # many ties
  logits[2, ::3] = logits[2].max()                         # the maximum repeated
  logits[3] = -50.0                                        # constant: classes 0 .. k-1
  logits[4] = 0.0
  logits[4, 1::2] = -0.0                                   # -0 ties with +0, as top_k compares them
  probs, classes = _topk(logits, k)
  _check_topk(logits, probs, classes)
  assert classes[3].tolist() == list(range(k)) and classes[4].tolist() == list(range(k))
  assert torch.equal(probs[3], torch.full((k,), float(np.float32(1.0) / np.float32(c))))
  for i in (0, 1, 2, 77, 127):                              # rows do not depend on N
    p1, c1 = _topk(logits[i:i + 1].contiguous(), k)
    assert torch.equal(p1[0], probs[i]) and torch.equal(c1[0], classes[i])


def test_softmax_topk_refuses_bad_k():
  from automl_b200 import _lib
  ops = _ops()
  logits = torch.zeros((2, 10), device=DEV)
  for k in (0, 11, 33):
    with pytest.raises(_lib.EdetError, match='k='):
      ops.softmax_topk(logits, torch.zeros((2, k), device=DEV),
                       torch.zeros((2, k), dtype=torch.int32, device=DEV))
  with pytest.raises(_lib.EdetError, match='k='):
    ops.softmax_topk(torch.zeros((2, 40), device=DEV), torch.zeros((2, 33), device=DEV),
                     torch.zeros((2, 33), dtype=torch.int32, device=DEV))
  with pytest.raises(ValueError):
    ops.softmax_topk(logits, torch.zeros((2, 3), device=DEV),
                     torch.zeros((2, 4), dtype=torch.int32, device=DEV))


def test_bad_arguments_are_refused_with_a_message():
  from automl_b200 import _lib
  lib = _lib.load()
  b = torch.zeros(64, dtype=torch.float32, device=DEV)
  p = ctypes.c_void_p(b.data_ptr())
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  cases = [
      ('edet_cls_preprocess', (None, p, 1, 4, 0, None, p, s), 'null'),
      ('edet_cls_preprocess', (p, p, 0, 4, 0, None, p, s), 'shape'),
      ('edet_cls_preprocess', (p, p, 1, 4, 2, None, p, s), 'mode'),
      ('edet_cls_preprocess', (p, p, 1, 4, 1, None, p, s), 'table'),
      ('edet_softmax_topk', (p, 1, 8, 1, None, p, s), 'null'),
      ('edet_softmax_topk', (p, 0, 8, 1, p, p, s), 'shape'),
      ('edet_softmax_topk', (p, 1, 8, 9, p, p, s), 'k='),
  ]
  for name, args, text in cases:
    assert getattr(lib, name)(*args) == 1, (name, args)
    assert text in lib.edet_last_error().decode(), (name, lib.edet_last_error())


# ---- the models ---------------------------------------------------------------------------------
def _model(name, size, batch, seed=11, include_top=True):
  arch = effnetv2_model.EffNetV2Arch(name)
  w = effnetv2_model.synthetic_weights(arch, seed, include_top=include_top)
  model = effnetv2_model.get_model(name, include_top=include_top, weights=w, batch_size=batch,
                                   image_size=size)
  return arch, w, model


def _decided_prefix(ref_sorted, err, k):
  """Length of the leading run of ranks whose margins to both neighbours exceed 2 err."""
  p = 0
  while p < k and ref_sorted[p] - ref_sorted[p + 1] > 2 * err:
    p += 1
  return p


@pytest.mark.parametrize('name,size', [('efficientnet-b0', 64), ('efficientnetv2-b0', 96),
                                       ('efficientnetv2-s', 128), ('efficientnetv2-s', 320)])
def test_classify_vs_oracle(name, size):
  import precision_model as pm
  from oracle import efficientdet_oracle as eo
  batch, k = 3, 5
  arch, w, model = _model(name, size, batch)
  legacy = preprocessing.is_legacy(model.cfg.data.augname)
  assert legacy == (name != 'efficientnetv2-s')
  ims = _images([(90, 120), (121, 77), (size, size)], 17)
  probs, classes = model.classify(ims, top_k=k)
  assert probs.dtype == np.float32 and classes.dtype == np.int32
  assert probs.shape == (batch, k) and classes.shape == (batch, k)
  x = np.stack([co.preprocess_image(im, size, legacy) for im in ims])
  assert torch.equal(model.input.cpu(), torch.from_numpy(x))      # the pre-process, bit for bit
  logits = model.output.double().cpu()
  ref = effnetv2_top_oracle.EffNetV2TopOracle(arch, w, torch.float32)(x)['logits'].double()
  err = float((logits - ref).norm() / ref.norm())
  if name == 'efficientnetv2-s':   # the fp16-storage format bar of DESIGN section 6
    wd = pm.effnetv2_device_weights(arch, w)
    wd[arch.model_name + '/dense/kernel'] = np.asarray(
        w[arch.model_name + '/dense/kernel'], np.float32).astype(np.float16).astype(np.float32)
    mod = effnetv2_top_oracle.EffNetV2TopOracle(arch, wd, torch.float32, store=eo.fp16_store)(x)
    merr = float((mod['logits'].double() - ref).norm() / ref.norm())
    print('%s %d: device %.2e, format model %.2e' % (name, size, err, merr))
    assert err < pm.bar(merr)
  else:
    assert err <= 1e-3, err
  # the top-k of the device logits exactly; the oracle's wherever its margins exceed the error
  _check_topk(model.output, torch.from_numpy(probs), torch.from_numpy(classes))
  for i in range(batch):
    e = float((logits[i] - ref[i]).abs().max())
    order = torch.sort(ref[i], descending=True, stable=True)
    p = _decided_prefix(order.values.tolist(), e, k)
    assert classes[i, :p].tolist() == order.indices[:p].tolist(), (i, p)


def test_pinned_cuda_and_list_inputs_give_the_same_input():
  arch, w, model = _model('efficientnetv2-b0', 96, 4)
  ims = _images([(120, 90)] * 4, 23)
  t = torch.from_numpy(np.stack(ims))
  want = model.preprocess(ims).clone()
  assert torch.equal(model.preprocess(t.pin_memory()), want)
  assert torch.equal(model.preprocess(t.to(DEV)), want)
  assert torch.equal(model.preprocess(t), want)                 # pageable: staged like a list
  assert torch.equal(want.cpu(), torch.from_numpy(np.stack([co.preprocess_image(im, 96, True) for im in ims])))


def test_classify_stream_equals_classify():
  arch, w, model = _model('efficientnetv2-s', 128, 3, seed=5)
  reqs = [_images([(90, 120), (200, 150), (64, 64)], 1),
          torch.from_numpy(np.stack(_images([(100, 130)] * 3, 2))).pin_memory(),
          _images([(300, 301), (33, 40), (128, 128)], 3),
          torch.from_numpy(np.stack(_images([(140, 100)] * 3, 4))).to(DEV),
          _images([(90, 90)] * 3, 5)]
  want = [model.classify(r, top_k=7) for r in reqs]
  got = list(model.classify_stream(reqs, top_k=7))
  assert len(got) == len(reqs)
  for (gp, gc), (wp, wc) in zip(got, want):
    assert np.array_equal(gp, wp) and np.array_equal(gc, wc)
  assert not np.array_equal(want[0][0], want[2][0])


def test_errors():
  _, _, plain = _model('efficientnetv2-b0', 64, 2, include_top=False)
  ims = _images([(80, 90), (70, 60)], 9)
  with pytest.raises(ValueError, match='include_top'):
    plain.classify(ims)
  _, _, model = _model('efficientnetv2-b0', 64, 2)
  for k in (0, 33):
    with pytest.raises(ValueError, match='top_k'):
      model.classify(ims, top_k=k)
  with pytest.raises(ValueError, match='expected 2 images'):
    model.classify(ims[:1])
  with pytest.raises(ValueError):
    model.classify([ims[0].astype(np.float32), ims[1]])
  with pytest.raises(ValueError):
    model.preprocess(torch.zeros((2, 80, 90, 3), dtype=torch.float32))
  with pytest.raises(ValueError):
    model.preprocess([np.zeros((1, 90, 3), np.uint8), ims[1]])     # empty crop
  rect = effnetv2_model.get_model('efficientnetv2-b0', include_top=True, batch_size=2,
                                  image_size=(64, 96))
  with pytest.raises(ValueError, match='square'):
    rect.classify(ims)
  with pytest.raises(NotImplementedError):
    preprocessing.preprocess_image(ims[0], 64, is_training=True)
  with pytest.raises(ValueError):
    preprocessing.preprocess_image(ims[0], 64, image_dtype=torch.float16)
  assert model.classify(ims)[1].shape == (2, 5)                   # still usable after the refusals
