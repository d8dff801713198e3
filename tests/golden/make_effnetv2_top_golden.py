"""Generates tests/golden/effnetv2_top.json: what the REAL reference constructs for the
classification top of the EfficientNet V1 / V2 models, run under the recording TensorFlow stand-in
(tests/golden/tf_stub.py).

For every registered model name with include_top True and False, and for a few overridden configs,
the unmodified /root/reference/efficientnetv2/effnetv2_model.py::EffNetV2Model is constructed and
the layers its `Head.__init__` (:438-470) and `_build` (:568-578) create are read back from the
constructor log:
  head_conv   keyword arguments of the head Conv2D (filters, kernel_size, use_bias, name)
  pooling     [layer class, keyword arguments] of the pooling layer
  dropout     the Dropout rate, or null when no Dropout layer is built
  dense       null when no `_fc` is built, else {units, name, bias_constant}: `name` is the `name`
              keyword the Dense constructor got (null: the layer is un-named and Keras calls the
              first such layer 'dense'), `bias_constant` the argument of tf.constant_initializer
  num_classes, headbias, local_pooling   the resolved model config values
The stand-in runs no `call`, so the order of the ops in `Head.call` is not recorded here;
tests/test_effnetv2_top_pins.py pins that from the cited lines.
Run from the repo root:
  python tests/golden/make_effnetv2_top_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/efficientnetv2'

MODELS = ['efficientnet-b%d' % i for i in range(9)] + ['efficientnet-l2'] + [
    'efficientnetv2-%s' % s for s in ('s', 'm', 'l', 'xl', 'b0', 'b1', 'b2', 'b3')]

# name -> (model, model_config override)
OVERRIDES = {
    'v2s_21k': ('efficientnetv2-s', {'num_classes': 21843}),
    'v2s_headbias': ('efficientnetv2-s', {'headbias': -2.5}),
    'v2s_no_classes': ('efficientnetv2-s', {'num_classes': 0}),
    'v2s_local_pooling': ('efficientnetv2-s', {'local_pooling': True}),
    'v2b0_no_dropout': ('efficientnetv2-b0', {'dropout_rate': 0.0}),
    'b0_1001': ('efficientnet-b0', {'num_classes': 1001, 'headbias': 0.5}),
    'v2s_feature_size': ('efficientnetv2-s', {'feature_size': 1792}),
}


def record(tf_stub, module, model, override, include_top):
  del tf_stub.LOG[:]
  net = module.EffNetV2Model(model, dict(override) if override else None, include_top)
  log = list(tf_stub.LOG)
  at = [i for i, e in enumerate(log) if e[0] == 'Head']
  assert len(at) == 1, at
  top = log[at[0] + 1:]
  names = [e[0].split('.')[-1] for e in top]
  conv = top[names.index('Conv2D')][2]
  pool = top[names.index('GlobalAveragePooling2D')]
  dropout = top[names.index('Dropout')][1][0] if 'Dropout' in names else None
  dense = None
  if 'Dense' in names:
    d = top[names.index('Dense')]
    dense = {'units': d[1][0], 'name': d[2].get('name'),
             'bias_constant': top[names.index('constant_initializer')][1][0]}
  assert (net._fc is None) == (dense is None)   # pylint: disable=protected-access
  m = net.cfg.model
  return {'model': model, 'override': override, 'include_top': include_top,
          'head_conv': {k: conv[k] for k in ('filters', 'kernel_size', 'use_bias', 'name')},
          'pooling': [pool[0].split('.')[-1], pool[2]], 'dropout': dropout, 'dense': dense,
          'num_classes': m.num_classes, 'headbias': m.headbias,
          'local_pooling': bool(m.local_pooling)}


def main():
  sys.path.insert(0, HERE)
  import tf_stub  # pylint: disable=g-import-not-at-top
  tf_stub.install()
  # the classifier's utils.py imports a sub-module the detector goldens never needed
  sys.modules['tensorflow_addons.layers'] = tf_stub._module('tensorflow_addons.layers')  # pylint: disable=protected-access
  sys.path.insert(0, REF)
  import effnetv2_model  # pylint: disable=g-import-not-at-top

  out = {}
  for model in MODELS:
    for include_top in (True, False):
      out['%s/%s' % (model, 'top' if include_top else 'notop')] = record(
          tf_stub, effnetv2_model, model, None, include_top)
  for key, (model, override) in sorted(OVERRIDES.items()):
    out[key] = record(tf_stub, effnetv2_model, model, override, True)
  path = os.path.join(os.environ.get('EFFNETV2_TOP_GOLDEN_OUT', HERE), 'effnetv2_top.json')
  with open(path, 'w') as f:
    json.dump(out, f, sort_keys=True, indent=1)
    f.write('\n')
  print('wrote', path, len(out), 'entries')


if __name__ == '__main__':
  main()
