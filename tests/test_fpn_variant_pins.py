"""Feature-network variants on the CPU: QuFPN node lists, channel-wise fusion weights,
conv_after_downsample and conv_bn_act_pattern.  The product (fpn_configs, DetArch, weights) and the
oracle's own QuFPN derivation (tests/fpn_variant_oracle.py) are held to what the REAL reference
resolves (tests/golden/fpn_variants.json, made by tests/golden/make_fpn_variant_golden.py)."""
import json
import os

import pytest

from automl_b200 import arch
from automl_b200 import fpn_configs
from automl_b200 import hparams_config
from automl_b200 import weights
import fpn_variant_oracle as fvo

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'fpn_variants.json')
with open(GOLDEN) as _f:
  GOLD = json.load(_f)
QUFPN = sorted(GOLD['qufpn'])
NETS = sorted(GOLD['nets'])


def _config(name, **over):
  c = hparams_config.get_efficientdet_config(name)
  c.override(over)
  return c


@pytest.mark.parametrize('key', QUFPN)
def test_product_qufpn_config_equals_real_reference(key):
  g = GOLD['qufpn'][key]
  p = fpn_configs.qufpn_config(g['min_level'], g['max_level'], g['weight_method_arg'])
  assert p.weight_method == g['weight_method'] and p.quad_method == g['quad_method']
  assert [dict(n) for n in p.nodes] == g['nodes']
  via_name = fpn_configs.get_fpn_config('qufpn', g['min_level'], g['max_level'], g['weight_method_arg'])
  assert [dict(n) for n in via_name.nodes] == g['nodes']


@pytest.mark.parametrize('key', QUFPN)
def test_oracle_qufpn_derivation_equals_real_reference(key):
  g = GOLD['qufpn'][key]
  assert [[lvl, offs] for lvl, offs in fvo.qufpn_nodes(g['min_level'], g['max_level'])] == \
      [[n['feat_level'], n['inputs_offsets']] for n in g['nodes']]


def test_qufpn_levels_3_7_spot_values():
  """Shape of the 3-7 cell (tf2/fpn_configs_test.py:60-90): 21 nodes; path 3 starts with
  [P4, P3] at level 4 (node 8), path 4 ends with [P3, node 19] at level 3 (node 15), and the
  quad-add nodes 16-20 add the path-2 and path-4 outputs of levels 7..3."""
  nodes = GOLD['qufpn']['3-7-None']['nodes']
  assert len(nodes) == 21
  assert nodes[8]['feat_level'] == 4 and nodes[8]['inputs_offsets'] == [1, 0]
  assert nodes[15]['feat_level'] == 3 and nodes[15]['inputs_offsets'] == [0, 19]
  assert [n['feat_level'] for n in nodes[16:]] == [7, 6, 5, 4, 3]
  assert [n['inputs_offsets'] for n in nodes[16:]] == [[12, 16], [11, 17], [10, 18], [9, 19], [8, 20]]
  assert all(n['weight_method'] == 'fastattn' for n in nodes)
  # with an explicit method the quad-add nodes keep quad_method in their dicts ...
  summed = GOLD['qufpn']['3-7-sum']['nodes']
  assert [n['weight_method'] for n in summed] == ['sum'] * 16 + ['fastattn'] * 5


@pytest.mark.parametrize('key', NETS)
def test_product_arch_equals_real_reference_network(key):
  """... but the networks fuse every node with the config-level method
  (tf2/efficientdet_keras.py:773), quad-add nodes included: DetArch does the same."""
  g = GOLD['nets'][key]
  c = _config(g['model'], **g['overrides'])
  a = arch.DetArch(c)
  assert len(a.cells) == g['fpn_cell_repeats'] == len(g['fnodes'])
  for cell, ref in zip(a.cells, g['fnodes']):
    assert [[n.feat_level - c.min_level, [r.src for r in n.inputs]] for n in cell['nodes']] == \
        [[r[0], r[1]] for r in ref]
    assert all(r[2] == a.fpn_weight_method for r in ref)
    assert all(r[3] == a.fpn_filters for r in ref)
    assert all(r[4] == a.conv_after_downsample and r[5] == a.conv_bn_act_pattern for r in ref)
  assert [[r.scope, a.fpn_filters, c.apply_bn_for_resampling, a.conv_after_downsample]
          for r in a.extra_levels] == \
      [['resample_p%d' % (lvl + c.min_level), ch, bn, cad] for lvl, ch, bn, cad in g['resample']]
  if (c.fpn_name or 'bifpn') == 'qufpn':
    for cell in a.cells:
      assert [(n.feat_level, [r.src for r in n.inputs]) for n in cell['nodes']] == \
          [(lvl, offs) for lvl, offs in fvo.qufpn_nodes(c.min_level, c.max_level)]


def test_conv_after_downsample_moves_only_shrinking_channel_changes():
  """efficientdet_arch.py:100-115: only a down-resample that also changes the channel count pools
  before its 1x1 conv: resample_p6 (320 -> 64 channels in D0) and, in a QuFPN cell 0, node 8's
  P3 input at level 4."""
  a = arch.DetArch(_config('efficientdet-d0', fpn_name='qufpn', conv_after_downsample=True))
  assert [a.conv_after_pool(r) for r in a.extra_levels] == [True, False]
  moved = [(i, j) for i, n in enumerate(a.cells[0]['nodes']) for j, r in enumerate(n.inputs)
           if a.conv_after_pool(r)]
  assert moved == [(8, 1)]
  r = a.cells[0]['nodes'][8].inputs[1]
  assert (r.in_channels, r.in_hw, r.out_hw, r.pool) == (40, (64, 64), (32, 32), (3, 3, 2, 2))
  assert not any(a.conv_after_pool(r) for cell in a.cells[1:] for n in cell['nodes'] for r in n.inputs)
  plain = arch.DetArch(_config('efficientdet-d0', fpn_name='qufpn'))
  assert not any(plain.conv_after_pool(r) for r in plain.extra_levels)


@pytest.mark.parametrize('method', ['channel_attn', 'channel_fastattn'])
def test_channel_weight_specs(method):
  """tf2/efficientdet_keras.py:101-115: one WSM variable of shape [F] per node input; nothing
  else changes."""
  base = weights.variable_specs(arch.DetArch(_config('efficientdet-d1')))
  a = arch.DetArch(_config('efficientdet-d1', fpn_weight_method=method))
  specs = weights.variable_specs(a)
  assert list(specs) == list(base)
  wsm = [k for k in specs if '/WSM' in k]
  assert len(wsm) == sum(len(n.inputs) for cell in a.cells for n in cell['nodes'])
  assert all(specs[k].shape == (88,) and base[k].shape == () for k in wsm)
  assert all(specs[k] == base[k] for k in specs if k not in wsm)
  w = weights.synthetic_weights(a, 0)
  assert w[wsm[0]].shape == (88,) and len(set(w[wsm[0]].tolist())) > 1


def test_conv_bn_act_pattern_weight_specs():
  """use_bias=not conv_bn_act_pattern (tf2/efficientdet_keras.py:205): the node convs lose their
  bias and nothing else changes."""
  base = weights.variable_specs(arch.DetArch(_config('efficientdet-d0')))
  specs = weights.variable_specs(arch.DetArch(_config('efficientdet-d0', conv_bn_act_pattern=True)))
  gone = [k for k in base if k not in specs]
  assert gone and all(k.startswith('fpn_cells/') and '/op_after_combine' in k and
                      k.endswith('/conv/bias') for k in gone)
  assert len(gone) == 3 * 8
  assert all(specs[k] == base[k] for k in specs)


@pytest.mark.parametrize('name', ['efficientdet-d0', 'efficientdet-d4', 'efficientdet-lite0',
                                  'efficientdet-d7x'])
def test_registered_models_keep_their_weight_specs(name):
  c = _config(name)
  assert not c.conv_bn_act_pattern and not c.conv_after_downsample
  a = arch.DetArch(c)
  specs = weights.variable_specs(a)
  for cell in a.cells:
    for n in cell['nodes']:
      assert n.op_scope + '/conv/bias' in specs
  shapes = {specs[k].shape for k in specs if '/WSM' in k}
  assert shapes <= {()}


def test_qufpn_weight_specs_follow_the_graph():
  a = arch.DetArch(_config('efficientdet-d0', fpn_name='qufpn'))
  specs = weights.variable_specs(a)
  assert len(a.cells[0]['nodes']) == 21
  # quad-add node 16 of cell 0 reads ids 12 and 16 of a 21-node cell: scopes count len(feats)
  n16 = a.cells[0]['nodes'][16]
  assert n16.op_scope == 'fpn_cells/cell_0/fnode16/op_after_combine21'
  assert [r.scope for r in n16.inputs] == ['fpn_cells/cell_0/fnode16/resample_0_12_21',
                                           'fpn_cells/cell_0/fnode16/resample_1_16_21']
  assert specs['fpn_cells/cell_0/fnode16/WSM_1'].shape == ()
  # cell 0 reads the 40 / 112 / 320-channel backbone features through 1x1 convs
  convs = [k for k in specs if k.startswith('fpn_cells/cell_0/') and k.endswith('/conv2d/kernel')]
  assert len(convs) == sum(1 for n in a.cells[0]['nodes'] for r in n.inputs if r.has_conv) == 11


def test_separable_conv_false_still_raises():
  with pytest.raises(NotImplementedError):
    arch.DetArch(_config('efficientdet-d0', separable_conv=False))
