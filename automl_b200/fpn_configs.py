"""BiFPN / QuFPN node graphs (which inputs feed which node).

Mirrors /root/reference/efficientdet/tf2/fpn_configs.py:24-72 (bifpn_config),
:75-163 (qufpn_config) and :166-176 (get_fpn_config).
"""
from automl_b200 import hparams_config


def bifpn_config(min_level, max_level, weight_method):
  """Top-down then bottom-up node list; node ids count up from the inputs."""
  p = hparams_config.Config()
  p.weight_method = weight_method or 'fastattn'

  num_levels = max_level - min_level + 1
  # ids of all nodes living at each level so far; inputs are 0..num_levels-1.
  ids_at = {min_level + i: [i] for i in range(num_levels)}
  next_id = num_levels
  nodes = []

  for level in range(max_level - 1, min_level - 1, -1):  # top-down
    nodes.append({
        'feat_level': level,
        'inputs_offsets': [ids_at[level][-1], ids_at[level + 1][-1]],
    })
    ids_at[level].append(next_id)
    next_id += 1

  for level in range(min_level + 1, max_level + 1):  # bottom-up
    nodes.append({
        'feat_level': level,
        'inputs_offsets': list(ids_at[level]) + [ids_at[level - 1][-1]],
    })
    ids_at[level].append(next_id)
    next_id += 1

  p.nodes = nodes
  return p


def qufpn_config(min_level, max_level, weight_method=None):
  """Quad FPN: four paths, then one 2-input node per level that adds the outputs of paths 2 and 4.

    path 1  top-down over the inputs (BiFPN's first half);
    path 2  bottom-up over the path-1 outputs (BiFPN's second half);
    path 3  bottom-up straight from the inputs;
    path 4  top-down over the path-3 outputs, each node also reading its level's input.

  A level a path skips (path 1 and 4: the top level, path 2 and 3: the bottom level) passes the
  previous path's output on.  Every node dict carries a 'weight_method' key like the reference's
  (the quad-add nodes `quad_method`, fixed to 'fastattn'); the networks ignore it and fuse every
  node with the config's `weight_method` (tf2/efficientdet_keras.py:773,
  efficientdet_arch.py:506)."""
  p = hparams_config.Config()
  p.weight_method = weight_method or 'fastattn'
  p.quad_method = 'fastattn'
  lo, hi = min_level, max_level
  inp = {l: l - lo for l in range(lo, hi + 1)}   # node ids of the cell inputs
  nodes = []

  def add(level, offsets, method):
    nodes.append({'feat_level': level, 'inputs_offsets': offsets, 'weight_method': method})
    return len(inp) + len(nodes) - 1

  wm = p.weight_method
  td1 = {hi: inp[hi]}
  for l in range(hi - 1, lo - 1, -1):
    td1[l] = add(l, [inp[l], td1[l + 1]], wm)
  bu2 = {lo: td1[lo]}
  for l in range(lo + 1, hi):
    bu2[l] = add(l, [inp[l], td1[l], bu2[l - 1]], wm)
  bu2[hi] = add(hi, [inp[hi], bu2[hi - 1]], wm)
  bu3 = {lo: inp[lo]}
  for l in range(lo + 1, hi + 1):
    bu3[l] = add(l, [inp[l], bu3[l - 1]], wm)
  td4 = {hi: bu3[hi]}
  for l in range(hi - 1, lo, -1):
    td4[l] = add(l, [inp[l], bu3[l], td4[l + 1]], wm)
  td4[lo] = add(lo, [inp[lo], td4[lo + 1]], wm)
  for l in range(hi, lo - 1, -1):
    add(l, [bu2[l], td4[l]], p.quad_method)
  p.nodes = nodes
  return p


def get_fpn_config(fpn_name, min_level, max_level, weight_method):
  if not fpn_name:
    fpn_name = 'bifpn'
  if fpn_name in ('bifpn', 'bifpn_dyn'):
    return bifpn_config(min_level, max_level, weight_method)
  if fpn_name == 'qufpn':
    return qufpn_config(min_level, max_level, weight_method)
  raise KeyError(fpn_name)
