"""CPU pins of the EfficientNet V1 / V2 classifier STRUCTURE against the REAL reference constructor.

tests/golden/effnetv2_structure.json.gz records what /root/reference/efficientnetv2/
effnetv2_model.py::EffNetV2Model constructs for all 18 registered names and for overrides that
change the structure (tests/golden/make_effnetv2_structure_golden.py).  Two things are held to it:

  * the oracle's OWN structure (oracle/effnetv2_structure.py), which oracle/effnetv2_oracle.py and
    tests/precision_model.py walk: every block's resolved block args and SE flag, every layer the
    constructor logs, the resolved act_fn and bn_epsilon;
  * the product's EffNetV2Arch, field by field against the oracle structure, and its
    `variable_specs` names and shapes against the variables the logged layers create (the names a
    real checkpoint's .npz is read by).

So a wrong stride, residual, SE width, rounding, layer name or reduction endpoint in the product
fails here on the CPU, and fails the GPU parity tests, instead of being repeated by the checker.
"""
import ast
import gzip
import json
import os

import pytest

from automl_b200 import utils
from automl_b200.efficientnetv2 import effnetv2_configs
from automl_b200.efficientnetv2 import effnetv2_model
from oracle import effnetv2_oracle
from oracle import effnetv2_structure as es

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
with gzip.open(os.path.join(HERE, 'golden', 'effnetv2_structure.json.gz'), 'rt') as _f:
  GOLDEN = json.load(_f)

BLOCK_ARGS = ('conv_type', 'kernel_size', 'strides', 'expand_ratio', 'input_filters',
              'output_filters', 'se_ratio', 'has_se')


def arch_mismatches(arch, s):
  """Every difference between a product EffNetV2Arch and the oracle Structure `s`, one message per
  field, naming the block."""
  out = []
  for field, want in (('stem_filters', s.stem_filters), ('head_filters', s.head_filters),
                      ('bn_eps', s.bn_epsilon), ('reductions', s.reductions),
                      ('act', utils.ACT_RELU6 if s.act_fn == 'relu6' else utils.ACT_SWISH),
                      ('len(blocks)', len(s.blocks))):
    got = len(arch.blocks) if field == 'len(blocks)' else getattr(arch, field)
    if got != want:
      out.append('%s: product %r, oracle %r' % (field, got, want))
  for i, (b, o) in enumerate(zip(arch.blocks, s.blocks)):
    for field, got in b._asdict().items():
      if got != o[field]:
        out.append('block %d (%s) %s: product %r, oracle %r' % (i, o['name'], field, got, o[field]))
  return out


def test_golden_covers_every_registered_model_and_the_structural_overrides():
  names = {e['model'] for e in GOLDEN.values() if e['override'] is None}
  registered = set(effnetv2_configs.efficientnetv1_params) | set(effnetv2_configs.efficientnetv2_params)
  assert len(names) == 18 and names == registered == set(es.MODELS)
  keys = set()
  for e in GOLDEN.values():
    keys |= set(e['override'] or {})
  assert {'width_coefficient', 'depth_coefficient', 'depth_divisor', 'min_depth', 'feature_size',
          'bn_epsilon', 'bn_momentum', 'act_fn'} <= keys
  assert {GOLDEN[k]['act_fn'] for k in GOLDEN} == {'silu', 'swish', 'relu6'}


@pytest.mark.parametrize('key', sorted(GOLDEN))
def test_oracle_structure_equals_the_reference_constructor(key):
  g = GOLDEN[key]
  s = es.Structure(g['model'], g['override'])
  assert s.act_fn == g['act_fn'] and s.bn_epsilon == g['bn_epsilon']
  assert len(s.blocks) == len(g['blocks'])
  for o, r in zip(s.blocks, g['blocks']):
    assert o['name'] == r['name'] and o['conv_type'] == {'MBConvBlock': 0, 'FusedMBConvBlock': 1}[r['class']]
    assert {k: o[k] for k in BLOCK_ARGS} == {k: r[k] for k in BLOCK_ARGS}, r['name']
  log = s.layer_log(include_top=True)
  for i, (o, r) in enumerate(zip(log, g['layers'])):
    assert o == r, (i, o, r)
  assert len(log) == len(g['layers'])


@pytest.mark.parametrize('key', sorted(GOLDEN))
def test_product_arch_equals_the_oracle_structure(key):
  g = GOLDEN[key]
  arch = effnetv2_model.EffNetV2Arch(g['model'], g['override'])
  assert arch_mismatches(arch, es.Structure(g['model'], g['override'])) == []


@pytest.mark.parametrize('key', sorted(GOLDEN))
def test_variable_specs_are_the_variables_the_reference_creates(key):
  g = GOLDEN[key]
  arch = effnetv2_model.EffNetV2Arch(g['model'], g['override'])
  got = [(n, tuple(v.shape)) for n, v in effnetv2_model.variable_specs(arch, include_top=True).items()]
  want = es.layer_variables(g['model'], g['layers'])
  for i, (a, b) in enumerate(zip(got, want)):
    assert a == b, (i, a, b)
  assert len(got) == len(want)


def _mutated(arch, changes):
  """A copy of `arch` whose blocks get the field changes [(block index, {field: value})]."""
  blocks = list(arch.blocks)
  for i, fields in changes:
    blocks[i] = blocks[i]._replace(**fields)
  out = effnetv2_model.EffNetV2Arch.__new__(effnetv2_model.EffNetV2Arch)
  out.__dict__.update(arch.__dict__, blocks=blocks)
  return out


@pytest.mark.parametrize('name,changes,block,field', [
    # the stride moves one block later: every shape and every param count stay the same
    ('efficientnetv2-s', [(10, {'strides': 1}), (11, {'strides': 2})], 'blocks_10', 'strides'),
    ('efficientnet-b3', [(5, {'strides': 1}), (6, {'strides': 2})], 'blocks_6', 'strides'),
    ('efficientnet-b0', [(7, {'se_filters': 0})], 'blocks_7', 'se_filters'),
    ('efficientnetv2-b0', [(4, {'has_skip': False})], 'blocks_4', 'has_skip'),
    ('efficientnetv2-b0', [(3, {'has_skip': True})], 'blocks_3', 'has_skip'),
    ('efficientnetv2-b0', [(6, {'project_bn': 'tpu_batch_normalization_1'})], 'blocks_6', 'project_bn'),
])
def test_the_pin_fails_a_broken_product(name, changes, block, field):
  arch = effnetv2_model.EffNetV2Arch(name)
  s = es.Structure(name)
  assert arch_mismatches(arch, s) == []
  msgs = arch_mismatches(_mutated(arch, changes), s)
  assert any(('(%s) %s:' % (block, field)) in m for m in msgs), msgs


def test_a_moved_stride_also_moves_a_reduction_endpoint():
  """The reductions of a product arch re-derived after a moved stride no longer match."""
  arch = effnetv2_model.EffNetV2Arch('efficientnetv2-s')
  s = es.Structure('efficientnetv2-s')
  bad = _mutated(arch, [(10, {'strides': 1}), (11, {'strides': 2})])
  bad.reductions = [i for i, b in enumerate(bad.blocks)
                    if i == len(bad.blocks) - 1 or bad.blocks[i + 1].strides > 1]
  assert any(m.startswith('reductions:') for m in arch_mismatches(bad, s))


def _imports(path):
  tree = ast.parse(open(path).read(), path)
  out = set()
  for node in ast.walk(tree):
    if isinstance(node, ast.Import):
      out |= {a.name for a in node.names}
    elif isinstance(node, ast.ImportFrom):
      out.add(node.module or '')
      out |= {'%s.%s' % (node.module, a.name) for a in node.names}
  return out


def test_the_oracle_imports_nothing_from_the_product():
  """oracle/effnetv2_oracle.py and every oracle module it reaches import no automl_b200 module."""
  todo, seen = ['oracle.effnetv2_oracle'], set()
  while todo:
    mod = todo.pop()
    if mod in seen:
      continue
    seen.add(mod)
    path = os.path.join(ROOT, *mod.split('.')) + '.py'
    for name in _imports(path):
      assert not name.split('.')[0] == 'automl_b200', (mod, name)
      if name.startswith('oracle.') and os.path.exists(os.path.join(ROOT, *name.split('.')) + '.py'):
        todo.append(name)
  assert {'oracle.effnetv2_oracle', 'oracle.effnetv2_structure', 'oracle.efficientdet_oracle'} <= seen


class _NameOnly(object):
  """Carries what the oracle may read from an arch, and nothing else: no blocks, no config."""

  def __init__(self, model_name, model_config=None):
    self.model_name, self.model_config = model_name, model_config


def test_the_oracle_reads_only_the_name_and_the_override_and_never_drops_one():
  w = effnetv2_model.synthetic_weights(effnetv2_model.EffNetV2Arch('efficientnetv2-b0'), 1)
  relu6, width = {'act_fn': 'relu6'}, {'width_coefficient': 1.3}
  assert effnetv2_oracle.EffNetV2Oracle(_NameOnly('efficientnetv2-b0'), w).s.act_fn == 'silu'
  assert effnetv2_oracle.EffNetV2Oracle('efficientnetv2-b0', w).s.act_fn == 'silu'
  # the arch's override is taken, whether or not the caller repeats it
  for arch, given in ((_NameOnly('efficientnetv2-b0', relu6), None),
                      (_NameOnly('efficientnetv2-b0', relu6), relu6),
                      (_NameOnly('efficientnetv2-b0'), relu6),
                      ('efficientnetv2-b0', relu6),
                      (effnetv2_model.EffNetV2Arch('efficientnetv2-b0', relu6), None)):
    assert effnetv2_oracle.EffNetV2Oracle(arch, w, model_config=given).s.act_fn == 'relu6'
  s = effnetv2_oracle.structure_of(effnetv2_model.EffNetV2Arch('efficientnetv2-b0', width))
  assert s.stem_filters == 40 and s.mconfig['width_coefficient'] == 1.3
  with pytest.raises(ValueError, match='built with model_config'):
    effnetv2_oracle.EffNetV2Oracle(_NameOnly('efficientnetv2-b0', relu6), w, model_config=width)
  for key in ('blocks_args', 'data_format', 'bn_type', 'no_such_key'):
    with pytest.raises(NotImplementedError):
      es.Structure('efficientnetv2-b0', {key: None})
