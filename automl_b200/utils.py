"""Size helpers and activation names shared by the host side of the H100 path.

Mirrors (reference file:line under /root/reference/efficientdet):
  * utils.py:484-506   parse_image_size  (int | 'WxH' string | (H, W) tuple)
  * utils.py:509-526   get_feat_sizes    (ceil-halving per level)
  * utils.py:529-549   verify_feats_size (ValueError text kept)
  * utils.py:36-53     activation_fn names -> integer codes understood by the kernels
"""

# Activation codes shared with csrc/common.cuh (enum EdetAct).
ACT_NONE = 0
ACT_SWISH = 1
ACT_RELU = 2
ACT_RELU6 = 3
ACT_HSWISH = 4
ACT_SIGMOID = 5

_ACT_CODES = {
    None: ACT_NONE,
    'silu': ACT_SWISH,
    'swish': ACT_SWISH,
    'swish_native': ACT_SWISH,
    'relu': ACT_RELU,
    'relu6': ACT_RELU6,
    'hswish': ACT_HSWISH,
}


def activation_code(act_type):
  """Kernel activation code for a reference act_type string."""
  if act_type not in _ACT_CODES:
    # mish / srelu exist in the reference (utils.py:48-51) but no registered
    # model uses them; they are not implemented as fused epilogues.
    raise ValueError('Unsupported act_type {}'.format(act_type))
  return _ACT_CODES[act_type]


def parse_image_size(image_size):
  """Returns (height, width) from an int, a 'WxH' string or an (H, W) tuple."""
  if isinstance(image_size, int):
    return (image_size, image_size)
  if isinstance(image_size, str):
    width, height = image_size.lower().split('x')
    return (int(height), int(width))
  if isinstance(image_size, tuple):
    return image_size
  raise ValueError('image_size must be an int, WxH string, or (height, width)'
                   'tuple. Was %r' % image_size)


def get_feat_sizes(image_size, max_level):
  """[{'height','width'}] for levels 0..max_level; each level is ceil(prev / 2)."""
  h, w = parse_image_size(image_size)
  sizes = [{'height': h, 'width': w}]
  for _ in range(max_level):
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    sizes.append({'height': h, 'width': w})
  return sizes


def verify_feats_size(feat_shapes, feat_sizes, min_level, max_level):
  """feat_shapes: list of (H, W) for levels min_level..max_level."""
  for cnt, size in enumerate(feat_sizes[min_level:max_level + 1]):
    h, w = feat_shapes[cnt]
    if h != size['height']:
      raise ValueError(
          'feats[{}] has shape {} but its height should be {}.'
          '(input_height: {}, min_level: {}, max_level: {}.)'.format(
              cnt, feat_shapes[cnt], size['height'], feat_sizes[0]['height'],
              min_level, max_level))
    if w != size['width']:
      raise ValueError(
          'feats[{}] has shape {} but its width should be {}.'
          '(input_width: {}, min_level: {}, max_level: {}.)'.format(
              cnt, feat_shapes[cnt], size['width'], feat_sizes[0]['width'],
              min_level, max_level))


def same_pad(in_size, kernel, stride):
  """TensorFlow 'SAME' padding: (out, pad_before, pad_after); extra goes after."""
  out = (in_size + stride - 1) // stride
  total = max((out - 1) * stride + kernel - in_size, 0)
  before = total // 2
  return out, before, total - before
