"""BiFPN node graph (which inputs feed which node).

Mirrors /root/reference/efficientdet/tf2/fpn_configs.py:24-72 (bifpn_config) and
:166-176 (get_fpn_config). QuFPN (:75-163) is not used by any registered model
and is out of scope (SURVEY.md section 2 row 5); asking for it raises.
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


def get_fpn_config(fpn_name, min_level, max_level, weight_method):
  if not fpn_name:
    fpn_name = 'bifpn'
  if fpn_name in ('bifpn', 'bifpn_dyn'):
    return bifpn_config(min_level, max_level, weight_method)
  if fpn_name == 'qufpn':
    raise NotImplementedError('qufpn is out of scope for the H100 path')
  raise KeyError(fpn_name)
