"""Generates tests/golden/fpn_variants.json: the feature-network variants (QuFPN, channel-wise
fusion weights, conv_after_downsample, conv_bn_act_pattern) as the REAL reference resolves them,
run under the recording TensorFlow stand-in (tests/golden/tf_stub.py).

It records
  qufpn : the node lists of /root/reference/efficientdet/tf2/fpn_configs.py::qufpn_config for
          several level ranges and weight methods (weight_method, quad_method, nodes);
  nets  : for overridden detector configs, what EfficientDetNet(config=...) constructs:
          fnodes   per cell and node: [feat_level, inputs_offsets, weight_method, filters,
                   conv_after_downsample, conv_bn_act_pattern] as the FNode constructor got them;
          resample the P6.. ResampleFeatureMap layers: [feat_level, channels, apply_bn,
                   conv_after_downsample].
The stand-in does not run FNode.build, so the WSM shapes and the op-after-combine layers are not
recorded here; tests/test_fpn_variant_pins.py pins those from the cited reference lines.
Run from the repo root:
  python tests/golden/make_fpn_variant_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/efficientdet'

LEVELS = [(3, 7), (3, 8), (2, 7), (3, 5)]
METHODS = [None, 'sum', 'channel_fastattn']

# name -> (model, overrides)
NETS = {
    'd0_qufpn': ('efficientdet-d0', {'fpn_name': 'qufpn'}),
    'd0_qufpn_sum': ('efficientdet-d0', {'fpn_name': 'qufpn', 'fpn_weight_method': 'sum'}),
    'd1_channel_fastattn': ('efficientdet-d1', {'fpn_weight_method': 'channel_fastattn'}),
    'd1_channel_attn': ('efficientdet-d1', {'fpn_weight_method': 'channel_attn'}),
    'd0_conv_after_downsample': ('efficientdet-d0', {'conv_after_downsample': True}),
    'd0_qufpn_conv_after_downsample': ('efficientdet-d0', {'fpn_name': 'qufpn',
                                                           'conv_after_downsample': True}),
    'd0_conv_bn_act_pattern': ('efficientdet-d0', {'conv_bn_act_pattern': True}),
    'lite0_qufpn': ('efficientdet-lite0', {'fpn_name': 'qufpn'}),
}


def main():
  sys.path.insert(0, HERE)
  import tf_stub
  tf_stub.install()
  sys.path.insert(0, REF)
  import hparams_config  # pylint: disable=g-import-not-at-top
  from tf2 import efficientdet_keras as ek  # pylint: disable=g-import-not-at-top
  from tf2 import fpn_configs  # pylint: disable=g-import-not-at-top

  qufpn = {}
  for lo, hi in LEVELS:
    for method in METHODS:
      p = fpn_configs.qufpn_config(lo, hi, method)
      qufpn['%d-%d-%s' % (lo, hi, method)] = {
          'min_level': lo, 'max_level': hi, 'weight_method_arg': method,
          'weight_method': p.weight_method, 'quad_method': p.quad_method,
          'nodes': [dict(n) for n in p.nodes]}

  nets = {}
  for key, (model, over) in sorted(NETS.items()):
    config = hparams_config.get_efficientdet_config(model)
    config.override(over)
    del tf_stub.LOG[:]
    m = ek.EfficientDetNet(config=config)
    fnodes = [[[fn.feat_level, list(fn.inputs_offsets), fn.weight_method, fn.fpn_num_filters,
                bool(fn.conv_after_downsample), bool(fn.conv_bn_act_pattern)]
               for fn in cell.fnodes] for cell in m.fpn_cells.cells]
    resample = [[r.feat_level, r.target_num_channels, bool(r.apply_bn),
                 bool(r.conv_after_downsample)] for r in m.resample_layers]
    nets[key] = {'model': model, 'overrides': over, 'min_level': config.min_level,
                 'max_level': config.max_level, 'fpn_cell_repeats': config.fpn_cell_repeats,
                 'fnodes': fnodes, 'resample': resample}
    print(key, len(fnodes), 'cells', len(fnodes[0]), 'nodes')
  path = os.path.join(os.environ.get('FPN_VARIANT_GOLDEN_OUT', HERE), 'fpn_variants.json')
  with open(path, 'w') as f:
    json.dump({'qufpn': qufpn, 'nets': nets}, f, sort_keys=True)
    f.write('\n')
  print('wrote', path)


if __name__ == '__main__':
  main()
