"""The classification top of the EfficientNet V1 / V2 models on the device: the pooling and Dense
kernels alone (edet_global_avg_pool, edet_dense) against float64 with bounds derived from their
summation trees, and the models with include_top=True against the oracle
(tests/effnetv2_top_oracle.py).

Error bounds.  u = 2^-24 is the float32 unit roundoff; a sum evaluated by any tree of depth d has
an error of at most d u sum|terms| to first order (1 % is allowed for the higher orders).
  * pool: thread partial of ceil(hw / 64) rows (ceil(hw / 64) - 1 adds), 3 shuffle levels, 3
    levels over the warps, then the product with float32(1 / hw), itself rounded once:
    |err| <= (ceil(hw / 64) + 7) u mean|x|.
  * dense: per k chunk of len <= 2560 a lane chain of 4 ceil(len / 128) fused multiply-adds, 5
    shuffle levels and one add of the bias or of the previous chunk's sum:
    |err| <= sum_chunks (4 ceil(len / 128) + 6) u (sum_k |a_k w_k| + |bias|).
The float64 references are computed with torch on the device from the same fp16 / float32 bits.
"""
import ctypes

import numpy as np
import pytest
import torch

import effnetv2_top_oracle
from automl_b200.efficientnetv2 import effnetv2_model

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
U = 2.0**-24
GUARD = 256                 # canary words after every output
CANARY = -12345.5

MODELS = ['efficientnet-b%d' % i for i in range(9)] + ['efficientnet-l2'] + [
    'efficientnetv2-%s' % s for s in ('s', 'm', 'l', 'xl', 'b0', 'b1', 'b2', 'b3')]
HEAD_WIDTHS = sorted({effnetv2_model.EffNetV2Arch(m).head_filters for m in MODELS})


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


class Out(object):
  """A float32 device output of `shape` followed by GUARD canary words."""

  def __init__(self, shape):
    self.numel = int(np.prod(shape))
    self.buf = torch.full((self.numel + GUARD,), CANARY, dtype=torch.float32, device=DEV)
    self.t = self.buf[:self.numel].view(shape)

  def result(self):
    torch.cuda.synchronize()
    assert bool((self.buf[self.numel:] == CANARY).all()), 'written past the end of the output'
    return self.t.clone()


def _randn(shape, seed, dtype, scale=1.0):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return (torch.randn(shape, generator=g, device=DEV, dtype=torch.float32) * scale).to(dtype)


def rel_l2(a, b):
  a, b = a.double().flatten(), b.double().flatten()
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


# ---- kernels alone ------------------------------------------------------------------------------
def test_head_widths_of_the_registered_models():
  assert HEAD_WIDTHS == [1280, 1408, 1536, 1792, 2048, 2304, 2560, 2816, 5504]


def _pool(x):
  out = Out((x.shape[0], x.shape[-1]))
  _ops().global_avg_pool(x, out.t)
  return out.result()


def check_pool(got, x):
  """got [N, C] within the bound of the fp32 mean of x [N, h, w, C] over its pixels."""
  n, h, w, c = x.shape
  x64 = x.double().view(n, h * w, c)
  ref, mean_abs = x64.mean(1), x64.abs().mean(1)
  bound = (-(-h * w // 64) + 7) * U * mean_abs * 1.01
  assert bool(((got.double() - ref).abs() <= bound).all()), float(((got.double() - ref).abs() / bound.clamp_min(1e-30)).max())


@pytest.mark.parametrize('c', HEAD_WIDTHS)
@pytest.mark.parametrize('hw', [(1, 1), (7, 7), (10, 10), (12, 12), (19, 19), (7, 12)])
def test_global_avg_pool(hw, c):
  h, w = hw
  n = 128
  x = _randn((n, h, w, c), 1000 * h * w + c, torch.float16, 2.0) + 0.5   # a mean that is not ~0
  got = _pool(x)
  check_pool(got, x)
  assert torch.equal(_pool(x), got)                                # two launches, same bits
  assert torch.equal(_pool(x[:3].contiguous()), got[:3])           # rows do not depend on N
  for i in (0, 77, 127):
    assert torch.equal(_pool(x[i:i + 1].contiguous()), got[i:i + 1])


def _dense(x, wt, bias):
  out = Out((x.shape[0], wt.shape[0]))
  _ops().dense(x, wt, bias, out.t)
  return out.result()


@pytest.mark.parametrize('classes,k', [(m, k) for m in (1, 8, 1000, 1001, 21843)
                                       for k in (1280, 1792, 2560)] + [(1000, 5504), (21, 8)])
def test_dense(classes, k):
  n = 128
  x = _randn((n, k), 7 * classes + k, torch.float32).abs()          # pooled swish maps are mostly positive
  wt = _randn((classes, k), classes + 3 * k, torch.float16, k**-0.5)
  bias = _randn((classes,), classes, torch.float32, 0.5)
  got = _dense(x, wt, bias)
  ref = x.double() @ wt.double().t() + bias.double()
  mag = x.double() @ wt.double().abs().t() + bias.double().abs()
  depth = sum(4 * -(-min(2560, k - k0) // 128) + 6 for k0 in range(0, k, 2560))
  bound = depth * U * mag * 1.01
  assert bool(((got.double() - ref).abs() <= bound).all()), float(((got.double() - ref).abs() / bound).max())
  assert torch.equal(_dense(x, wt, bias), got)
  assert torch.equal(_dense(x[:5].contiguous(), wt, bias), got[:5])
  for i in (0, 64, 127):
    assert torch.equal(_dense(x[i:i + 1].contiguous(), wt, bias), got[i:i + 1])


def test_bad_arguments_are_refused_with_a_message():
  """Status and message only: every call returns before a launch."""
  from automl_b200 import _lib
  lib = _lib.load()
  x = torch.zeros(2 * 4 * 16, dtype=torch.float16, device=DEV)
  f = torch.zeros(64, dtype=torch.float32, device=DEV)
  px, pf = ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(f.data_ptr())
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  cases = [
      ('edet_global_avg_pool', (None, pf, 2, 4, 16, stream), 'null'),
      ('edet_global_avg_pool', (px, None, 2, 4, 16, stream), 'null'),
      ('edet_global_avg_pool', (px, pf, 0, 4, 16, stream), 'shape'),
      ('edet_global_avg_pool', (px, pf, 2, 0, 16, stream), 'shape'),
      ('edet_global_avg_pool', (px, pf, 2, 4, 12, stream), 'multiple of 8'),
      ('edet_dense', (None, px, pf, pf, 2, 16, 4, stream), 'null'),
      ('edet_dense', (pf, px, None, pf, 2, 16, 4, stream), 'null'),
      ('edet_dense', (pf, px, pf, pf, 0, 16, 4, stream), 'shape'),
      ('edet_dense', (pf, px, pf, pf, 2, 16, 0, stream), 'shape'),
      ('edet_dense', (pf, px, pf, pf, 2, 12, 4, stream), 'multiple of 8'),
  ]
  for name, args, text in cases:
    assert getattr(lib, name)(*args) == 1, (name, args)              # EDET_ERR_INVALID
    assert text in lib.edet_last_error().decode(), (name, lib.edet_last_error())
  ops = _ops()
  with pytest.raises(ValueError):
    ops.global_avg_pool(x.view(2, 4, 16), f[:16].view(1, 16))
  with pytest.raises(ValueError):
    ops.dense(f[:32].view(2, 16), x[:64].view(4, 16), f[:4], f[:6].view(2, 3))
  with pytest.raises(_lib.EdetError, match='multiple of 8'):
    ops.global_avg_pool(x[:96].view(2, 4, 12), f[:24].view(2, 12))


# ---- the models ---------------------------------------------------------------------------------
def top_format_model(arch, w, x):
  """The oracle through the top at device precision (tests/precision_model.py: fp16 storage of
  every map, BN folded into fp16 conv kernels) with what the top adds: the Dense kernel rounded to
  fp16; pooled features, bias and logits stay float32.  Returns (format-model endpoints, fp32
  endpoints)."""
  import precision_model as pm
  from oracle import efficientdet_oracle as eo
  wd = pm.effnetv2_device_weights(arch, w)
  name = arch.model_name + '/dense/kernel'
  if name in w:
    wd[name] = np.asarray(w[name], np.float32).astype(np.float16).astype(np.float32)
  ref = effnetv2_top_oracle.EffNetV2TopOracle(arch, w, torch.float32)(x)
  mod = effnetv2_top_oracle.EffNetV2TopOracle(arch, wd, torch.float32, store=eo.fp16_store)(x)
  return mod, ref


def _check_argmax(logits, ref):
  """The arg-max agrees wherever the oracle's top-2 margin exceeds twice the largest logit error
  of that image (an error of e per logit can close a margin of 2 e)."""
  logits, ref = logits.double().cpu(), ref.double()
  top2 = ref.topk(2, dim=1).values
  margin = top2[:, 0] - top2[:, 1]
  err = (logits - ref).abs().max(dim=1).values
  decided = margin > 2 * err
  assert bool((logits.argmax(1)[decided] == ref.argmax(1)[decided]).all())
  return int(decided.sum())


def _build(name, size, batch, seed=11, config=None, **kw):
  arch = effnetv2_model.EffNetV2Arch(name, config)
  w = effnetv2_model.synthetic_weights(arch, seed, include_top=True)
  model = effnetv2_model.get_model(name, config, include_top=True, weights=w, batch_size=batch,
                                   image_size=size, **kw)
  h, wd = model.image_size
  x = np.random.default_rng(3).uniform(-1, 1, size=(batch, h, wd, 3)).astype(np.float32)
  return arch, w, model, x


@pytest.mark.parametrize('name,size,batch', [('efficientnet-b0', 64, 3), ('efficientnetv2-b0', (64, 80), 2)])
def test_logits_vs_oracle(name, size, batch):
  arch, w, model, x = _build(name, size, batch)
  outs = model(torch.from_numpy(x), with_endpoints=True)
  torch.cuda.synchronize()
  logits = outs[0].clone()
  assert outs[0] is model.output and logits.dtype == torch.float32 and tuple(logits.shape) == (batch, 1000)
  assert len(outs) == 6 and all(outs[i] is model.endpoints['reduction_%d' % i] for i in range(1, 6))
  ref = effnetv2_top_oracle.EffNetV2TopOracle(arch, w, torch.float32)(x)
  pooled = model.endpoints['pooled_features']
  assert pooled.dtype == torch.float32 and tuple(pooled.shape) == (batch, arch.head_filters)
  assert model.endpoints['head'] is pooled
  assert rel_l2(pooled.cpu(), ref['pooled_features']) <= 1e-3
  assert rel_l2(logits.cpu(), ref['logits']) <= 1e-3
  _check_argmax(logits, ref['logits'])
  # the pooled endpoint is the mean of the head_1x1 endpoint, the logits its Dense image
  head = model.endpoints['head_1x1']
  assert rel_l2(pooled, head.double().mean((1, 2))) < 1e-6
  assert torch.equal(model(torch.from_numpy(x)), logits)           # graph replay
  info = {o['name']: o for o in model.op_info}
  assert [o['name'] for o in model.op_info[-3:]] == ['head_1x1', 'avg_pool', 'dense']
  assert info['avg_pool']['bytes'] == 2 * head.numel() + 4 * pooled.numel()
  assert info['dense']['flops'] == 2 * batch * arch.head_filters * 1000


def test_v2_s_384_logits_within_the_format_model():
  """EfficientNetV2-S at its own resolution: the logits are held to 1.5 x the format model + 1e-4,
  like its deepest endpoints (40 residual blocks of fp16 storage)."""
  import precision_model as pm
  arch, w, model, x = _build('efficientnetv2-s', 384, 2)
  logits = model(torch.from_numpy(x))
  torch.cuda.synchronize()
  mod, ref = top_format_model(arch, w, x)
  for key, got in (('pooled_features', model.endpoints['pooled_features']), ('logits', logits)):
    merr, err = rel_l2(mod[key], ref[key]), rel_l2(got.cpu(), ref[key])
    print('%s: device %.2e, format model %.2e' % (key, err, merr))
    assert err < pm.bar(merr), (key, err, merr)
  assert tuple(logits.shape) == (2, 1000)
  _check_argmax(logits, ref['logits'])


def test_top_leaves_the_backbone_bits_and_graph_equals_eager():
  name, size, batch = 'efficientnetv2-b0', 64, 2
  arch, w, model, x = _build(name, size, batch)
  plain = effnetv2_model.get_model(name, weights=w, batch_size=batch, image_size=size)
  eager = effnetv2_model.get_model(name, include_top=True, weights=w, batch_size=batch,
                                   image_size=size, use_cuda_graph=False)
  xt = torch.from_numpy(x)
  logits, feat, logits_eager = model(xt), plain(xt), eager(xt)
  torch.cuda.synchronize()
  assert feat.dtype == torch.float16 and feat is plain.endpoints['head_1x1']
  assert 'pooled_features' not in plain.endpoints and len(plain.op_info) == len(model.op_info) - 2
  assert [o['name'] for o in plain.op_info] == [o['name'] for o in model.op_info[:-2]]
  for key, t in plain.endpoints.items():
    assert torch.equal(t, model.endpoints[key]), key
  assert torch.equal(logits, logits_eager)
  for key, t in eager.endpoints.items():
    assert torch.equal(t, model.endpoints[key]), key


def test_serve_stream_yields_the_logits():
  arch, w, model, _ = _build('efficientnetv2-b0', 64, 2, seed=5)
  rng = np.random.default_rng(9)
  batches = [torch.from_numpy(rng.uniform(-1, 1, size=(2, 64, 64, 3)).astype(np.float32)).pin_memory()
             for _ in range(5)]
  want = [model(b).cpu().clone() for b in batches]
  got = [r.clone() for r in model.serve_stream(batches)]
  assert len(got) == 5
  for g, e in zip(got, want):
    assert g.dtype == torch.float32 and tuple(g.shape) == (2, 1000)
    assert torch.equal(g, e)
  first = next(iter(model.serve_stream(iter(batches[:1]))))
  assert first.is_pinned() and first.numel() * first.element_size() == 2 * 1000 * 4


@pytest.mark.parametrize('name,config', [
    ('efficientnet-b3', None),                                                 # width 1.2, depth 1.4, stem 40
    ('efficientnetv2-b0', {'width_coefficient': 1.3, 'depth_coefficient': 1.2}),
    ('efficientnetv2-b0', {'act_fn': 'relu6'})])
def test_unrun_structures_end_to_end(name, config):
  """Structures no other test runs through the whole device network, against the oracle's own
  structure (oracle/effnetv2_structure.py, pinned to the reference constructor): every reduction
  endpoint, 'head_1x1' and the logits within 1e-3 rel-L2, or within 1.5 x the format model + 1e-4
  where that is the larger (DESIGN.md section 6)."""
  _check_end_to_end(name, config)


def _check_end_to_end(name, config):
  import precision_model as pm
  arch, w, model, x = _build(name, 64, 2, config=config)
  logits = model(torch.from_numpy(x)).clone()
  torch.cuda.synchronize()
  mod, ref = top_format_model(arch, w, x)
  keys = ['reduction_%d' % i for i in range(1, len(arch.reductions) + 1)] + ['head_1x1', 'logits']
  assert len(arch.reductions) == 5 and set(keys) <= set(ref)
  for key in keys:
    got = logits.cpu() if key == 'logits' else model.endpoints[key].float().cpu().permute(0, 3, 1, 2)
    merr, err = rel_l2(mod[key], ref[key]), rel_l2(got, ref[key])
    print('%s %s %s: device %.2e, format model %.2e' % (name, config, key, err, merr))
    assert err <= max(1e-3, pm.bar(merr)), (key, err, merr)
  _check_argmax(logits, ref['logits'])


def test_efficientnet_l2_end_to_end():
  """efficientnet-l2 at 64 x 64, batch 2, include_top=True, as test_unrun_structures_end_to_end
  checks the others.  Its blocks 83-87 expand 1376 to 8256 channels, the widest 1x1 convolution
  of any registered model (65 N tiles of 128 columns), which pointwise_tc once refused as too wide
  for its shared-memory bias.  481 M parameters: the synthetic weights alone are 1.9 GB of float32
  on the host.  On an H100 80GB HBM3 host the test took 31 s (weights, upload, the device pass and
  two CPU oracle passes) and its process peaked at 8.6 GB of resident host memory."""
  _check_end_to_end('efficientnet-l2', None)


@pytest.mark.parametrize('config', [{'num_classes': 0}, {'local_pooling': True},
                                    {'num_classes': 1001, 'headbias': -2.5}])
def test_config_overrides(config):
  arch, w, model, x = _build('efficientnetv2-b0', 64, 2, config=config)
  out = model(torch.from_numpy(x))
  torch.cuda.synchronize()
  ref = effnetv2_top_oracle.EffNetV2TopOracle(arch, w, torch.float32)(x)
  pooled = model.endpoints['pooled_features']
  c = arch.head_filters
  if config.get('local_pooling'):
    assert tuple(pooled.shape) == (2, 1, 1, c) and tuple(ref['pooled_features'].shape) == (2, 1, 1, c)
  else:
    assert tuple(pooled.shape) == (2, c)
  assert rel_l2(pooled.cpu(), ref['pooled_features']) <= 1e-3
  if config.get('num_classes') == 0:
    assert 'logits' not in ref and [o['name'] for o in model.op_info[-2:]] == ['head_1x1', 'avg_pool']
    assert out.dtype == torch.float32 and tuple(out.shape) == (2, c)
    assert out.data_ptr() == pooled.data_ptr()
  else:
    assert tuple(out.shape) == (2, arch.mconfig.num_classes)
    assert rel_l2(out.cpu(), ref['logits']) <= 1e-3
  if 'headbias' in config:
    assert abs(float(out.mean()) + 2.5) < 0.5       # the bias constant reaches the logits


def test_npz_weights_need_the_dense_keys(tmp_path):
  name = 'efficientnetv2-b0'
  arch = effnetv2_model.EffNetV2Arch(name)
  w = effnetv2_model.synthetic_weights(arch, 2, include_top=True)
  full, backbone = str(tmp_path / 'full.npz'), str(tmp_path / 'backbone.npz')
  np.savez(full, **w)
  np.savez(backbone, **{k: v for k, v in w.items() if '/dense/' not in k})
  x = torch.from_numpy(np.random.default_rng(1).uniform(-1, 1, size=(1, 64, 64, 3)).astype(np.float32))
  a = effnetv2_model.get_model(name, include_top=True, weights=full, batch_size=1, image_size=64)(x)
  b = effnetv2_model.get_model(name, include_top=True, weights=w, batch_size=1, image_size=64)(x)
  assert torch.equal(a, b)
  with pytest.raises(ValueError, match='dense/kernel.*dense/bias'):
    effnetv2_model.get_model(name, include_top=True, weights=backbone, batch_size=1, image_size=64)
  effnetv2_model.get_model(name, weights=backbone, batch_size=1, image_size=64)   # no top, no Dense keys
