"""CPU pins of the EfficientNet V1 / V2 classification top (global average pooling + Dense).

Structure comes from the REAL reference constructor: tests/golden/effnetv2_top.json records what
`Head.__init__` and `EffNetV2Model._build` create for every registered model and a few overridden
configs (tests/golden/make_effnetv2_top_golden.py).  The recording stand-in runs no `call` and no
Keras naming, so two things are pinned from the cited lines instead:
  * the Dense layer gets no `name` keyword (golden: name null), and Keras names the first un-named
    Dense of a model 'dense': <model>/dense/kernel [head_filters, units], <model>/dense/bias;
  * `Head.call` (effnetv2_model.py:472-496) pools 'head_1x1', applies Dropout (identity at
    inference) and stores the result as 'pooled_features' and 'head'; `call` :644-646 applies `_fc`.
The oracle's pooling and Dense (tests/effnetv2_top_oracle.py) are held to plain numpy loops in float64, like
tests/test_oracle_definitions.py does for the TensorFlow-owned ops.
"""
import json
import os

import numpy as np
import pytest
import torch

import effnetv2_top_oracle
from automl_b200.efficientnetv2 import effnetv2_model
from oracle import effnetv2_oracle

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'effnetv2_top.json')) as _f:
  GOLDEN = json.load(_f)


def test_golden_covers_every_registered_model_and_the_overrides():
  models = {e['model'] for e in GOLDEN.values()}
  assert len(models) == 18 and {'efficientnet-b0', 'efficientnet-l2', 'efficientnetv2-xl'} <= models
  for m in models:
    assert GOLDEN[m + '/top']['dense'] == {'units': 1000, 'name': None, 'bias_constant': 0}
    assert GOLDEN[m + '/notop']['dense'] is None
  assert GOLDEN['v2s_21k']['dense']['units'] == 21843
  assert GOLDEN['v2s_headbias']['dense']['bias_constant'] == -2.5
  assert GOLDEN['v2s_no_classes']['dense'] is None
  assert GOLDEN['v2s_local_pooling']['local_pooling'] is True
  assert GOLDEN['v2b0_no_dropout']['dropout'] is None and GOLDEN['efficientnetv2-b0/top']['dropout'] == 0.2


@pytest.mark.parametrize('key', sorted(GOLDEN))
def test_specs_match_what_the_reference_constructs(key):
  g = GOLDEN[key]
  arch = effnetv2_model.EffNetV2Arch(g['model'], g['override'])
  mn = g['model']
  assert arch.head_filters == g['head_conv']['filters']
  assert g['head_conv'] == {'filters': arch.head_filters, 'kernel_size': 1, 'use_bias': False,
                            'name': 'conv2d'}
  assert g['pooling'] == ['GlobalAveragePooling2D', {'data_format': 'channels_last'}]
  assert bool(arch.mconfig.local_pooling) == g['local_pooling']
  base = effnetv2_model.variable_specs(arch)
  specs = effnetv2_model.variable_specs(arch, g['include_top'])
  names = list(specs)
  assert names[:len(base)] == list(base)              # the top comes after every existing entry
  if g['dense'] is None:
    assert names == list(base)
    assert not any('/dense/' in n for n in names)
  else:
    assert g['dense']['name'] is None                  # un-named -> Keras' default 'dense'
    assert names[len(base):] == [mn + '/dense/kernel', mn + '/dense/bias']
    assert specs[mn + '/dense/kernel'].shape == (g['head_conv']['filters'], g['dense']['units'])
    assert specs[mn + '/dense/bias'].shape == (g['dense']['units'],)
    assert g['dense']['bias_constant'] == (arch.mconfig.headbias or 0)
  assert effnetv2_model.count_params(arch, g['include_top']) == sum(
      int(np.prod(v.shape)) for v in specs.values())
  dense_params = 0 if g['dense'] is None else (arch.head_filters + 1) * g['dense']['units']
  assert effnetv2_model.count_params(arch, g['include_top']) == (
      effnetv2_model.count_params(arch, False) + dense_params)


@pytest.mark.parametrize('key', ['efficientnetv2-b0/top', 'v2s_headbias', 'b0_1001'])
def test_synthetic_top_weights(key):
  """The backbone of a seed keeps its bits when the top is drawn; the Dense bias is centred on the
  reference's constant (`headbias or 0`, :576), the kernel has variance 1 / K."""
  g = GOLDEN[key]
  arch = effnetv2_model.EffNetV2Arch(g['model'], g['override'])
  w0 = effnetv2_model.synthetic_weights(arch, 7)
  w1 = effnetv2_model.synthetic_weights(arch, 7, include_top=True)
  assert list(w1)[:len(w0)] == list(w0) and len(w1) == len(w0) + 2
  for k in w0:
    assert w0[k].dtype == w1[k].dtype and np.array_equal(w0[k], w1[k]), k
  kernel, bias = w1[g['model'] + '/dense/kernel'], w1[g['model'] + '/dense/bias']
  assert kernel.dtype == np.float32 and bias.dtype == np.float32
  assert abs(float(bias.mean()) - g['dense']['bias_constant']) < 0.02
  assert 0.05 < float(bias.std()) < 0.2
  assert abs(float(kernel.std()) * np.sqrt(arch.head_filters) - 1.0) < 0.02


def _run_oracle(model, override, dtype, n=3, size=(32, 48), seed=5):
  arch = effnetv2_model.EffNetV2Arch(model, override)
  w = effnetv2_model.synthetic_weights(arch, seed, include_top=True)
  x = np.random.default_rng(seed + 1).uniform(-1, 1, size=(n,) + size + (3,)).astype(np.float32)
  return arch, w, x, effnetv2_top_oracle.EffNetV2TopOracle(arch, w, dtype)(x)


@pytest.mark.parametrize('key', ['efficientnet-b0/top', 'v2s_local_pooling', 'b0_1001'])
def test_oracle_top_equals_its_definition(key):
  """pooled[i, c] = sum_{y, x} head_1x1[i, c, y, x] / (H W); logits = pooled @ kernel + bias, as
  plain float64 loops -> 1e-12.  Under local_pooling the endpoints keep the [N, 1, 1, C] shape of
  avg_pool and the Dense sees the squeezed tensor (:487)."""
  g = GOLDEN[key]
  arch, w, _, ep = _run_oracle(g['model'], g['override'], torch.float64)
  head = ep['head_1x1'].numpy()
  n, c, h, wd = head.shape
  assert c == arch.head_filters and h * wd > 1
  pooled = np.zeros((n, c))
  for i in range(n):
    for y in range(h):
      for xx in range(wd):
        pooled[i] += head[i, :, y, xx]
  pooled /= h * wd
  got = ep['pooled_features'].numpy()
  assert ep['head'] is ep['pooled_features']            # Dropout is the identity at inference
  assert got.shape == ((n, 1, 1, c) if g['local_pooling'] else (n, c))
  assert np.abs(got.reshape(n, c) - pooled).max() <= 1e-12 * max(1.0, np.abs(pooled).max())
  kernel = np.float64(w[g['model'] + '/dense/kernel'])
  bias = np.float64(w[g['model'] + '/dense/bias'])
  units = g['dense']['units']
  logits = np.zeros((n, units))
  for i in range(n):
    for j in range(units):
      logits[i, j] = sum(pooled[i, k] * kernel[k, j] for k in range(c)) + bias[j]
  assert ep['logits'].shape == (n, units)
  assert np.abs(ep['logits'].numpy() - logits).max() <= 1e-12 * max(1.0, np.abs(logits).max())


def test_oracle_without_classes_has_no_logits_and_default_is_unchanged():
  arch, w, x, ep = _run_oracle('efficientnetv2-b0', {'num_classes': 0}, torch.float32, n=1)
  assert GOLDEN['v2s_no_classes']['dense'] is None
  assert 'logits' not in ep and ep['pooled_features'].shape == (1, arch.head_filters)
  assert not any('/dense/' in k for k in w)
  plain = effnetv2_oracle.EffNetV2Oracle(arch, w, torch.float32)(x)
  assert sorted(plain) == sorted(k for k in ep if k not in ('pooled_features', 'head'))
  for k in plain:
    assert torch.equal(plain[k], ep[k]), k
