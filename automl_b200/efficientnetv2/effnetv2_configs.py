"""Model configs of the reference's efficientnetv2/effnetv2_configs.py (block-string grammar
:25-93, V1 table :96-136, V2 tables :139-231) and the `model` section of hparams.base_config
(efficientnetv2/hparams.py:221-243).  Only what the inference forward pass reads is kept; the
train / eval sections keep the image sizes, the data section the eval pre-process recipe
(`augname`: 'effnetv1_*' selects the legacy bicubic recipe, preprocessing.py:133)."""
import re

from automl_b200.hparams_config import Config


class BlockDecoder(object):
  """Block-string notation: r<repeat>_k<kernel>_s<stride>_e<expand>_i<in>_o<out>[_c<conv_type>]
  [_se<ratio>] (effnetv2_configs.py:25-45)."""

  def _decode_block_string(self, block_string):
    assert isinstance(block_string, str)
    options = {}
    for op in block_string.split('_'):
      m = re.match(r'([a-z]+)(\d.*)$', op)
      if m:
        options[m.group(1)] = m.group(2)
    return Config(dict(
        kernel_size=int(options['k']), num_repeat=int(options['r']),
        input_filters=int(options['i']), output_filters=int(options['o']),
        expand_ratio=int(options['e']),
        se_ratio=float(options['se']) if 'se' in options else None,
        strides=int(options['s']), conv_type=int(options['c']) if 'c' in options else 0))

  def decode(self, string_list):
    assert isinstance(string_list, list)
    return [self._decode_block_string(s) for s in string_list]


v1_b0_block_str = [
    'r1_k3_s1_e1_i32_o16_se0.25', 'r2_k3_s2_e6_i16_o24_se0.25', 'r2_k5_s2_e6_i24_o40_se0.25',
    'r3_k3_s2_e6_i40_o80_se0.25', 'r3_k5_s1_e6_i80_o112_se0.25', 'r4_k5_s2_e6_i112_o192_se0.25',
    'r1_k3_s1_e6_i192_o320_se0.25',
]
# (width_coefficient, depth_coefficient, resolution, dropout_rate)
efficientnetv1_params = {
    'efficientnet-b0': (1.0, 1.0, 224, 0.2), 'efficientnet-b1': (1.0, 1.1, 240, 0.2),
    'efficientnet-b2': (1.1, 1.2, 260, 0.3), 'efficientnet-b3': (1.2, 1.4, 300, 0.3),
    'efficientnet-b4': (1.4, 1.8, 380, 0.4), 'efficientnet-b5': (1.6, 2.2, 456, 0.4),
    'efficientnet-b6': (1.8, 2.6, 528, 0.5), 'efficientnet-b7': (2.0, 3.1, 600, 0.5),
    'efficientnet-b8': (2.2, 3.6, 672, 0.5), 'efficientnet-l2': (4.3, 5.3, 800, 0.5),
}

v2_base_block = ['r1_k3_s1_e1_i32_o16_c1', 'r2_k3_s2_e4_i16_o32_c1', 'r2_k3_s2_e4_i32_o48_c1',
                 'r3_k3_s2_e4_i48_o96_se0.25', 'r5_k3_s1_e6_i96_o112_se0.25',
                 'r8_k3_s2_e6_i112_o192_se0.25']
v2_s_block = ['r2_k3_s1_e1_i24_o24_c1', 'r4_k3_s2_e4_i24_o48_c1', 'r4_k3_s2_e4_i48_o64_c1',
              'r6_k3_s2_e4_i64_o128_se0.25', 'r9_k3_s1_e6_i128_o160_se0.25',
              'r15_k3_s2_e6_i160_o256_se0.25']
v2_m_block = ['r3_k3_s1_e1_i24_o24_c1', 'r5_k3_s2_e4_i24_o48_c1', 'r5_k3_s2_e4_i48_o80_c1',
              'r7_k3_s2_e4_i80_o160_se0.25', 'r14_k3_s1_e6_i160_o176_se0.25',
              'r18_k3_s2_e6_i176_o304_se0.25', 'r5_k3_s1_e6_i304_o512_se0.25']
v2_l_block = ['r4_k3_s1_e1_i32_o32_c1', 'r7_k3_s2_e4_i32_o64_c1', 'r7_k3_s2_e4_i64_o96_c1',
              'r10_k3_s2_e4_i96_o192_se0.25', 'r19_k3_s1_e6_i192_o224_se0.25',
              'r25_k3_s2_e6_i224_o384_se0.25', 'r7_k3_s1_e6_i384_o640_se0.25']
v2_xl_block = ['r4_k3_s1_e1_i32_o32_c1', 'r8_k3_s2_e4_i32_o64_c1', 'r8_k3_s2_e4_i64_o96_c1',
               'r16_k3_s2_e4_i96_o192_se0.25', 'r24_k3_s1_e6_i192_o256_se0.25',
               'r32_k3_s2_e6_i256_o512_se0.25', 'r8_k3_s1_e6_i512_o640_se0.25']
# (block, width, depth, train_size, eval_size, dropout, augname); the reference's randaug /
# mixup magnitudes only matter for training and are not kept
efficientnetv2_params = {
    'efficientnetv2-s': (v2_s_block, 1.0, 1.0, 300, 384, 0.2, 'randaug'),
    'efficientnetv2-m': (v2_m_block, 1.0, 1.0, 384, 480, 0.3, 'randaug'),
    'efficientnetv2-l': (v2_l_block, 1.0, 1.0, 384, 480, 0.4, 'randaug'),
    'efficientnetv2-xl': (v2_xl_block, 1.0, 1.0, 384, 512, 0.4, 'randaug'),
    'efficientnetv2-b0': (v2_base_block, 1.0, 1.0, 192, 224, 0.2, 'effnetv1_autoaug'),
    'efficientnetv2-b1': (v2_base_block, 1.0, 1.1, 192, 240, 0.2, 'effnetv1_autoaug'),
    'efficientnetv2-b2': (v2_base_block, 1.1, 1.2, 208, 260, 0.3, 'effnetv1_autoaug'),
    'efficientnetv2-b3': (v2_base_block, 1.2, 1.4, 240, 300, 0.3, 'effnetv1_autoaug'),
}


def base_model_config():
  """hparams.base_config.model (efficientnetv2/hparams.py:223-243)."""
  return dict(model_name='efficientnet-b0', data_format='channels_last', feature_size=1280,
              bn_type=None, bn_momentum=0.9, bn_epsilon=1e-3, gn_groups=8, depth_divisor=8,
              min_depth=8, act_fn='silu', survival_prob=0.8, local_pooling=False, headbias=None,
              conv_dropout=None, dropout_rate=None, depth_coefficient=None,
              width_coefficient=None, blocks_args=None, num_classes=1000)


def efficientnetv1_config(model_name='efficientnet-b0'):
  width, depth, isize, dropout = efficientnetv1_params[model_name]
  model = base_model_config()
  model.update(model_name=model_name, blocks_args=BlockDecoder().decode(v1_b0_block_str),
               width_coefficient=width, depth_coefficient=depth, dropout_rate=dropout)
  return Config(dict(model=model, eval=dict(isize=isize), train=dict(isize=0.8),
                     data=dict(augname='effnetv1_autoaug')))


def efficientnetv2_config(model_name='efficientnetv2-s'):
  block, width, depth, train_size, eval_size, dropout, aug = efficientnetv2_params[model_name]
  model = base_model_config()
  model.update(model_name=model_name, blocks_args=BlockDecoder().decode(block),
               width_coefficient=width, depth_coefficient=depth, dropout_rate=dropout)
  return Config(dict(model=model, eval=dict(isize=eval_size), train=dict(isize=train_size),
                     data=dict(augname=aug)))


def get_model_config(model_name):
  """Main entry for model name to config (effnetv2_configs.py:234-240)."""
  if model_name.startswith('efficientnet-'):
    return efficientnetv1_config(model_name)
  if model_name.startswith('efficientnetv2-'):
    return efficientnetv2_config(model_name)
  raise ValueError(f'Unknown model_name {model_name}')
