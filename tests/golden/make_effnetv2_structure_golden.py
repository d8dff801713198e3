"""Generates tests/golden/effnetv2_structure.json.gz: the EfficientNet V1 / V2 classifier STRUCTURE as
resolved by the REAL reference constructor, run under the recording TensorFlow stand-in
(tests/golden/tf_stub.py).

For every registered model name (include_top=True), and for overrides that change the structure,
the unmodified /root/reference/efficientnetv2/effnetv2_model.py::EffNetV2Model is constructed and
recorded:

  blocks   per block, the layer class, the name it was given and the reference's own resolved
           `_block_args` (conv_type, kernel_size, strides, expand_ratio, input_filters,
           output_filters, se_ratio) and `_has_se`;
  layers   every Conv2D / DepthwiseConv2D / BatchNormalization / Dense the constructor created, in
           creation order:
             [scope, kind, filters, kernel, strides, use_bias, name, bn_epsilon, bn_momentum]
           scope is 'stem', 'head', 'blocks_<i>', 'blocks_<i>/se' or '' (the model itself).
           The stand-in runs no Keras naming, so two names are Keras' defaults rather than read
           from the log: an un-named layer is named after its class in snake case (Stem -> 'stem',
           Head -> 'head', the Dense -> 'dense'; tests/golden/effnetv2_top.json pins that the
           Dense gets no name), and a Dense has a bias (Keras' use_bias=True default);
  act_fn, bn_epsilon   the resolved model config values.

The two SE convs are the ones SE.__init__ creates (effnetv2_model.py:116-133), so the two Conv2D
after an 'SE' entry of the log are given the '<block>/se' scope.
tests/test_effnetv2_structure_pins.py holds the oracle's own structure
(oracle/effnetv2_structure.py) and the product's EffNetV2Arch to exactly this.  Run from the repo
root:
  python tests/golden/make_effnetv2_structure_golden.py
"""
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/efficientnetv2'

MODELS = ['efficientnet-b%d' % i for i in range(9)] + ['efficientnet-l2'] + [
    'efficientnetv2-%s' % s for s in ('s', 'm', 'l', 'xl', 'b0', 'b1', 'b2', 'b3')]

# name -> (model, model_config override)
OVERRIDES = {
    'v2b0_width_depth': ('efficientnetv2-b0', {'width_coefficient': 1.3, 'depth_coefficient': 1.2}),
    'v2b0_depth': ('efficientnetv2-b0', {'depth_coefficient': 1.6}),
    'b0_divisor16': ('efficientnet-b0', {'depth_divisor': 16}),
    'b3_divisor16_min_depth': ('efficientnet-b3', {'depth_divisor': 16, 'min_depth': 32}),
    'v2s_feature_size': ('efficientnetv2-s', {'feature_size': 1792}),
    'v2b0_bn': ('efficientnetv2-b0', {'bn_epsilon': 1e-5, 'bn_momentum': 0.99}),
    'v2b0_relu6': ('efficientnetv2-b0', {'act_fn': 'relu6'}),
    'b0_swish': ('efficientnet-b0', {'act_fn': 'swish'}),
}

BLOCK_ARGS = ('conv_type', 'kernel_size', 'strides', 'expand_ratio', 'input_filters',
              'output_filters', 'se_ratio')


def canonical_layers(log):
  out, scope, block, se_left = [], '', None, 0
  for cls, args, kw in log:
    cls = cls.split('.')[-1]
    if cls in ('Stem', 'Head'):
      assert kw.get('name') is None
      scope = cls.lower()
      continue
    if cls in ('MBConvBlock', 'FusedMBConvBlock'):
      scope = block = kw['name']
      continue
    if cls == 'SE':
      scope, se_left = '%s/%s' % (block, kw['name']), 2
      continue
    if cls == 'GlobalAveragePooling2D':
      scope = ''
      continue
    if cls in ('Conv2D', 'DepthwiseConv2D'):
      filters = kw.get('filters', args[0] if args else None) if cls == 'Conv2D' else None
      out.append([scope, 'conv' if cls == 'Conv2D' else 'dw', filters, kw['kernel_size'],
                  kw.get('strides', 1), kw['use_bias'], kw['name'], None, None])
      if se_left:
        se_left -= 1
        if not se_left:
          scope = block
    elif cls == 'BatchNormalization':
      out.append([scope, 'bn', None, None, None, None, kw['name'], kw['epsilon'], kw['momentum']])
    elif cls == 'Dense':
      assert kw.get('name') is None and 'use_bias' not in kw, kw
      out.append([scope, 'dense', args[0], None, None, True, 'dense', None, None])
  return out


def record(tf_stub, module, model, override):
  del tf_stub.LOG[:]
  net = module.EffNetV2Model(model, dict(override) if override else None, True)
  log = list(tf_stub.LOG)
  markers = [(cls, kw['name']) for cls, _, kw in log if cls in ('MBConvBlock', 'FusedMBConvBlock')]
  assert len(markers) == len(net._blocks)   # pylint: disable=protected-access
  blocks = []
  for (cls, name), b in zip(markers, net._blocks):   # pylint: disable=protected-access
    ba = b._block_args                                # pylint: disable=protected-access
    assert type(b).__name__ == cls
    entry = {'class': cls, 'name': name, 'has_se': bool(b._has_se)}  # pylint: disable=protected-access
    entry.update({k: ba[k] for k in BLOCK_ARGS})
    blocks.append(entry)
  m = net.cfg.model
  return {'model': model, 'override': override, 'act_fn': m.act_fn, 'bn_epsilon': m.bn_epsilon,
          'blocks': blocks, 'layers': canonical_layers(log)}


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
    out[model] = record(tf_stub, effnetv2_model, model, None)
  for key, (model, override) in sorted(OVERRIDES.items()):
    out[key] = record(tf_stub, effnetv2_model, model, override)
  for key, e in sorted(out.items()):
    print(key, len(e['blocks']), 'blocks', len(e['layers']), 'layers')
  path = os.path.join(os.environ.get('EFFNETV2_STRUCTURE_GOLDEN_OUT', HERE),
                      'effnetv2_structure.json.gz')
  with gzip.GzipFile(path, 'wb', mtime=0) as f:
    f.write(json.dumps(out, sort_keys=True).encode())
  print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
  main()
