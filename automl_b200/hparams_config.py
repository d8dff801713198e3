"""Model registry + attribute-dict config for the EfficientDet forward path.

Host-side mirror of the reference registry so callers of the H100 path can keep
using `get_efficientdet_config('efficientdet-d0')`, `Config.override('a=1,b.c=2')`
and friends unchanged.

Reference behaviour mirrored (file:line under /root/reference/efficientdet):
  * hparams_config.py:25-31    eval_str_fn ('true'/'false', literal_eval, else str)
  * hparams_config.py:35-166   Config (update / override / parse_from_str / as_dict)
  * hparams_config.py:170-298  default_detection_configs
  * hparams_config.py:301-467  efficientdet_model_param_dict / lite dict
  * hparams_config.py:470-487  get_efficientdet_config / get_detection_config

No TensorFlow here: yaml files are opened with the builtin `open`.
"""
import ast
import collections.abc
import copy

import yaml


def eval_str_fn(val):
  """'true'/'false' -> bool, python literals -> value, anything else stays str."""
  if val == 'true':
    return True
  if val == 'false':
    return False
  try:
    return ast.literal_eval(val)
  except (ValueError, SyntaxError):
    return val


def _kv_to_nested(key, value):
  """'x.y.z', 'tt' -> {x: {y: {z: tt}}}; '*' in the value splits a list."""
  head, dot, rest = key.partition('.')
  if dot:
    return {head: _kv_to_nested(rest, value)}
  if '*' in value:
    return {head: [eval_str_fn(piece) for piece in value.split('*')]}
  return {head: eval_str_fn(value)}


def _deep_merge(dst, src):
  for k, v in src.items():
    if k in dst and isinstance(dst[k], dict) and isinstance(
        v, collections.abc.Mapping):
      _deep_merge(dst[k], v)
    else:
      dst[k] = v


class Config(object):
  """Attribute dictionary: nested dicts become nested Configs, values are copied."""

  def __init__(self, config_dict=None):
    self.update(config_dict)

  # -- attribute / item protocol -------------------------------------------
  def __setattr__(self, k, v):
    self.__dict__[k] = Config(v) if isinstance(v, dict) else copy.deepcopy(v)

  def __getattr__(self, k):
    # Only reached when normal lookup fails: mirror the reference (KeyError).
    return self.__dict__[k]

  def __getitem__(self, k):
    return self.__dict__[k]

  def __contains__(self, k):
    return k in self.__dict__

  def __repr__(self):
    return repr(self.as_dict())

  def __str__(self):
    try:
      return yaml.dump(self.as_dict(), indent=4)
    except TypeError:
      return str(self.as_dict())

  def __deepcopy__(self, memodict):
    return type(self)(self.as_dict())

  def get(self, k, default_value=None):
    return self.__dict__.get(k, default_value)

  def keys(self):
    return self.__dict__.keys()

  def as_dict(self):
    out = {}
    for k, v in self.__dict__.items():
      out[k] = v.as_dict() if isinstance(v, Config) else copy.deepcopy(v)
    return out

  # -- update / override ----------------------------------------------------
  def _update(self, config_dict, allow_new_keys=True):
    if not config_dict:
      return
    for k, v in config_dict.items():
      if k not in self.__dict__:
        if not allow_new_keys:
          raise KeyError('Key `{}` does not exist for overriding. '.format(k))
        setattr(self, k, v)
        continue
      cur = self.__dict__[k]
      if isinstance(cur, Config) and isinstance(v, dict):
        cur._update(v, allow_new_keys)  # pylint: disable=protected-access
      elif isinstance(cur, Config) and isinstance(v, Config):
        cur._update(v.as_dict(), allow_new_keys)  # pylint: disable=protected-access
      else:
        setattr(self, k, v)

  def update(self, config_dict):
    """Update members; unknown keys are added."""
    self._update(config_dict, allow_new_keys=True)

  def override(self, config_dict_or_str, allow_new_keys=False):
    """Update members; unknown keys raise KeyError unless allow_new_keys."""
    if isinstance(config_dict_or_str, str):
      if not config_dict_or_str:
        return
      if '=' in config_dict_or_str:
        config_dict = self.parse_from_str(config_dict_or_str)
      elif config_dict_or_str.endswith('.yaml'):
        config_dict = self.parse_from_yaml(config_dict_or_str)
      else:
        raise ValueError(
            'Invalid string {}, must end with .yaml or contains "=".'.format(
                config_dict_or_str))
    elif isinstance(config_dict_or_str, dict):
      config_dict = config_dict_or_str
    else:
      raise ValueError('Unknown value type: {}'.format(config_dict_or_str))
    self._update(config_dict, allow_new_keys)

  def parse_from_yaml(self, yaml_file_path):
    with open(yaml_file_path, 'r') as f:
      return yaml.load(f, Loader=yaml.FullLoader)

  def save_to_yaml(self, yaml_file_path):
    with open(yaml_file_path, 'w') as f:
      yaml.dump(self.as_dict(), f, default_flow_style=False)

  def parse_from_str(self, config_str):
    """'x.y=1,x.z=2' -> {x: {y: 1, z: 2}}; empty pieces between commas skipped."""
    if not config_str:
      return {}
    parsed = {}
    try:
      for piece in config_str.split(','):
        if not piece:
          continue
        key, value = piece.split('=')  # ValueError unless exactly one '='
        _deep_merge(parsed, _kv_to_nested(key.strip(), value))
    except ValueError:
      raise ValueError('Invalid config_str: {}'.format(config_str))
    return parsed


# Everything the reference's default_detection_configs() sets, as one table.
_DETECTION_DEFAULTS = (
    ('name', 'efficientdet-d1'),
    ('act_type', 'swish'),
    # input preprocessing
    ('image_size', 640),
    ('target_size', None),
    ('input_rand_hflip', True),
    ('jitter_min', 0.1),
    ('jitter_max', 2.0),
    ('autoaugment_policy', None),
    ('grid_mask', False),
    ('sample_image', None),
    ('map_freq', 5),
    # dataset
    ('num_classes', 90),
    ('seg_num_classes', 3),
    ('heads', ['object_detection']),
    ('skip_crowd_during_training', True),
    ('label_map', None),
    ('max_instances_per_image', 100),
    ('regenerate_source_id', False),
    # architecture
    ('min_level', 3),
    ('max_level', 7),
    ('num_scales', 3),
    ('aspect_ratios', [1.0, 2.0, 0.5]),
    ('anchor_scale', 4.0),
    ('is_training_bn', True),
    # optimisation (unused by the forward path; kept so overrides resolve)
    ('momentum', 0.9),
    ('optimizer', 'sgd'),
    ('learning_rate', 0.08),
    ('lr_warmup_init', 0.008),
    ('lr_warmup_epoch', 1.0),
    ('first_lr_drop_epoch', 200.0),
    ('second_lr_drop_epoch', 250.0),
    ('poly_lr_power', 0.9),
    ('clip_gradients_norm', 10.0),
    ('num_epochs', 300),
    ('data_format', 'channels_last'),
    ('mean_rgb', [0.485 * 255, 0.456 * 255, 0.406 * 255]),
    ('stddev_rgb', [0.229 * 255, 0.224 * 255, 0.225 * 255]),
    ('scale_range', False),
    ('label_smoothing', 0.0),
    ('alpha', 0.25),
    ('gamma', 1.5),
    ('delta', 0.1),
    ('box_loss_weight', 50.0),
    ('iou_loss_type', None),
    ('iou_loss_weight', 1.0),
    ('weight_decay', 4e-5),
    ('strategy', None),
    ('mixed_precision', False),
    ('loss_scale', None),
    # detection heads / fpn
    ('box_class_repeats', 3),
    ('fpn_cell_repeats', 3),
    ('fpn_num_filters', 88),
    ('separable_conv', True),
    ('apply_bn_for_resampling', True),
    ('conv_after_downsample', False),
    ('conv_bn_act_pattern', False),
    ('drop_remainder', True),
    ('nms_configs', {
        'method': 'gaussian',
        'iou_thresh': None,
        'score_thresh': 0.,
        'sigma': None,
        'pyfunc': False,
        'max_nms_inputs': 0,
        'max_output_size': 100,
    }),
    ('tflite_max_detections', 100),
    ('fpn_name', None),
    ('fpn_weight_method', None),
    ('fpn_config', None),
    ('survival_prob', None),
    ('img_summary_steps', None),
    ('lr_decay_method', 'cosine'),
    ('moving_average_decay', 0.9998),
    ('ckpt_var_scope', None),
    ('skip_mismatch', True),
    ('backbone_name', 'efficientnet-b1'),
    ('backbone_config', None),
    ('var_freeze_expr', None),
    ('use_keras_model', True),
    ('dataset_type', None),
    ('positives_momentum', None),
    ('grad_checkpoint', False),
    ('verbose', 1),
    ('save_freq', 'epoch'),
)


def default_detection_configs():
  """Returns a fresh Config with the detection defaults."""
  h = Config()
  for k, v in _DETECTION_DEFAULTS:
    setattr(h, k, v)
  return h


def _det(name, backbone, image_size, filters, cells, repeats, **extra):
  d = dict(
      name=name,
      backbone_name=backbone,
      image_size=image_size,
      fpn_num_filters=filters,
      fpn_cell_repeats=cells,
      box_class_repeats=repeats)
  d.update(extra)
  return d


# (backbone, image_size, fpn_num_filters, fpn_cell_repeats, box_class_repeats, extras)
efficientdet_model_param_dict = {
    'efficientdet-d0': _det('efficientdet-d0', 'efficientnet-b0', 512, 64, 3, 3),
    'efficientdet-d1': _det('efficientdet-d1', 'efficientnet-b1', 640, 88, 4, 3),
    'efficientdet-d2': _det('efficientdet-d2', 'efficientnet-b2', 768, 112, 5, 3),
    'efficientdet-d3': _det('efficientdet-d3', 'efficientnet-b3', 896, 160, 6, 4),
    'efficientdet-d4': _det('efficientdet-d4', 'efficientnet-b4', 1024, 224, 7, 4),
    'efficientdet-d5': _det('efficientdet-d5', 'efficientnet-b5', 1280, 288, 7, 4),
    'efficientdet-d6': _det('efficientdet-d6', 'efficientnet-b6', 1280, 384, 8, 5,
                            fpn_weight_method='sum'),
    'efficientdet-d7': _det('efficientdet-d7', 'efficientnet-b6', 1536, 384, 8, 5,
                            anchor_scale=5.0, fpn_weight_method='sum'),
    'efficientdet-d7x': _det('efficientdet-d7x', 'efficientnet-b7', 1536, 384, 8, 5,
                             anchor_scale=4.0, max_level=8,
                             fpn_weight_method='sum'),
}

lite_common_param = dict(
    mean_rgb=127.0,
    stddev_rgb=128.0,
    act_type='relu6',
    fpn_weight_method='sum',
)

efficientdet_lite_param_dict = {
    'efficientdet-lite0': _det('efficientdet-lite0', 'efficientnet-lite0', 320, 64,
                               3, 3, anchor_scale=3.0, **lite_common_param),
    'efficientdet-lite1': _det('efficientdet-lite1', 'efficientnet-lite1', 384, 88,
                               4, 3, anchor_scale=3.0, **lite_common_param),
    'efficientdet-lite2': _det('efficientdet-lite2', 'efficientnet-lite2', 448, 112,
                               5, 3, anchor_scale=3.0, **lite_common_param),
    'efficientdet-lite3': _det('efficientdet-lite3', 'efficientnet-lite3', 512, 160,
                               6, 4, **lite_common_param),
    'efficientdet-lite3x': _det('efficientdet-lite3x', 'efficientnet-lite3', 640,
                                200, 6, 4, anchor_scale=3.0, **lite_common_param),
    'efficientdet-lite4': _det('efficientdet-lite4', 'efficientnet-lite4', 640, 224,
                               7, 4, **lite_common_param),
}


def get_efficientdet_config(model_name='efficientdet-d1'):
  """Default config for an EfficientDet model name (ValueError if unknown)."""
  h = default_detection_configs()
  for table in (efficientdet_model_param_dict, efficientdet_lite_param_dict):
    if model_name in table:
      h.override(table[model_name])
      return h
  raise ValueError('Unknown model name: {}'.format(model_name))


def get_detection_config(model_name):
  if model_name.startswith('efficientdet'):
    return get_efficientdet_config(model_name)
  raise ValueError('model name must start with efficientdet.')
