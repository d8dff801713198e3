"""Structural description of an EfficientDet network (host side, no tensors).

`DetArch(config)` resolves a `hparams_config.Config` into everything the engine
needs to lower the network to kernels and everything `weights.py` needs to name
and size the variables: backbone blocks, feature sizes, the extra P6.. levels,
the BiFPN node graph with per-input resample kinds, and the head layout.

Reference structure followed (file:line under /root/reference/efficientdet):
  * efficientdet_arch.py:305-349   build_backbone -> {0: image, 1..5: reduction_k}
  * efficientdet_arch.py:352-415   build_feature_network (extra levels, cell loop)
  * efficientdet_arch.py:55-132    resample_feature_map (1x1 conv only if channels differ;
                                   max-pool (s+1)x(s+1) stride s when shrinking; TF1 nearest
                                   neighbour when growing; mixed up/down raises ValueError)
  * efficientdet_arch.py:478-544   build_bifpn_layer (variable scopes, node outputs per level)
  * efficientdet_arch.py:252-302   heads: shared convs, per-level BN
Variable scope names follow the Keras twin (tf2/efficientdet_keras.py:123-131,
152-160, 399-420) so real checkpoints can be mapped later.
"""
import collections

from automl_b200 import fpn_configs
from automl_b200 import utils
from automl_b200.backbone import efficientnet_builder

# How one BiFPN node input reaches the node's resolution.
ResampleSpec = collections.namedtuple('ResampleSpec', [
    'scope',        # e.g. 'fpn_cells/cell_0/fnode1/resample_0_2_6'
    'src',          # index into the running feats list
    'in_hw', 'out_hw', 'in_channels',
    'has_conv',     # 1x1 conv(+bias)+BN because in_channels != fpn_num_filters
    'mode',         # 'same' | 'down' | 'up'
    'pool',         # (pool_h, pool_w, stride_h, stride_w) for 'down', else None
])

NodeSpec = collections.namedtuple('NodeSpec', [
    'scope',        # 'fpn_cells/cell_0/fnode3'
    'feat_level', 'hw', 'inputs',  # inputs: [ResampleSpec]
    'op_scope',     # 'fpn_cells/cell_0/fnode3/op_after_combine8'
    'out_index',    # index of this node's output in the running feats list
])


HEADS = ('object_detection', 'segmentation')

# One Conv2DTranspose 3x3 stride 2 'SAME' of the segmentation head
# (tf2/efficientdet_keras.py:676-706): max_level - min_level stages (+ BN + act, then the concat
# with the next finer BiFPN level), then the final layer (bias, no BN / act).
SegStageSpec = collections.namedtuple('SegStageSpec', [
    'kernel_scope',  # 'segmentation_head/conv2d_transpose[_i]'
    'bn_scope',      # 'segmentation_head/bn_<i>', None for the final layer
    'in_hw', 'out_hw',
    'in_channels',   # F for the first stage, 2F (x, skip) after it
    'out_channels',  # F, seg_num_classes for the final layer
    'skip_level',    # BiFPN level concatenated after the stage, None for the final layer
])


def _seg_stages(arch):
  """Layer list of SegmentationHead for a resolved architecture.  Variable names follow Keras'
  default layer naming in a fresh model (the unnamed Conv2DTranspose layers become
  conv2d_transpose, conv2d_transpose_1, ... in creation order, the head's own last); they cannot
  be checked against a real checkpoint offline."""
  f = arch.fpn_filters
  stages = []
  n = arch.max_level - arch.min_level
  for i in range(n + 1):
    level = arch.max_level - i
    in_hw = arch.level_hw[level] if i == 0 else stages[-1].out_hw
    out_hw = (2 * in_hw[0], 2 * in_hw[1])
    final = i == n
    if not final and out_hw != arch.level_hw[level - 1]:
      # the reference's tf.concat (efficientdet_keras.py:703) fails on these shapes
      raise ValueError(
          'segmentation head: P{} is {}x{}, upsampled to {}x{}, but P{} is {}x{}; every level '
          'must be exactly twice the next one (image size {})'.format(
              level, in_hw[0], in_hw[1], out_hw[0], out_hw[1], level - 1,
              arch.level_hw[level - 1][0], arch.level_hw[level - 1][1], arch.image_hw))
    stages.append(SegStageSpec(
        kernel_scope='segmentation_head/conv2d_transpose' + ('_%d' % i if i else ''),
        bn_scope=None if final else 'segmentation_head/bn_%d' % i,
        in_hw=in_hw, out_hw=out_hw,
        in_channels=f if i == 0 else 2 * f,
        out_channels=arch.config.seg_num_classes if final else f,
        skip_level=None if final else level - 1))
  return stages


def _resample_mode(in_hw, out_hw):
  (h, w), (th, tw) = in_hw, out_hw
  if h > th and w > tw:
    sh, sw = (h - 1) // th + 1, (w - 1) // tw + 1
    return 'down', (sh + 1, sw + 1, sh, sw)
  if h <= th and w <= tw:
    return ('up' if (h < th or w < tw) else 'same'), None
  raise ValueError(
      'Incompatible target feature map size: target_height: {},'
      'target_width: {}'.format(th, tw))


class DetArch(object):
  """Resolved architecture for one detection config."""

  def __init__(self, config):
    p = config
    if p.data_format not in ('channels_last', 'channels_first'):
      raise ValueError('bad data_format %r' % (p.data_format,))
    if not p.separable_conv:
      raise NotImplementedError('separable_conv=False is not on the H100 path')
    if p.backbone_config is not None:
      raise NotImplementedError('custom backbone_config')
    self.config = p
    self._resolve_heads(p)
    self.act_type = p.act_type
    # node op: fuse -> sepconv without bias -> BN -> act instead of fuse -> act -> sepconv + bias
    # -> BN (efficientdet_arch.py:508-533)
    self.conv_bn_act_pattern = bool(p.conv_bn_act_pattern)
    # a shrinking resample with a channel change max-pools first and applies its 1x1 conv + BN
    # at the pooled size (efficientdet_arch.py:100-115)
    self.conv_after_downsample = bool(p.conv_after_downsample)
    self.image_hw = utils.parse_image_size(p.image_size)
    self.min_level, self.max_level = p.min_level, p.max_level
    self.num_levels = p.max_level - p.min_level + 1
    self.fpn_filters = p.fpn_num_filters
    self.num_anchors = len(p.aspect_ratios) * p.num_scales
    self.num_classes = p.num_classes
    self.head_repeats = p.box_class_repeats
    self.feat_sizes = utils.get_feat_sizes(p.image_size, p.max_level)

    # ---- backbone ------------------------------------------------------------
    if 'efficientnet' not in p.backbone_name:
      raise ValueError(
          'backbone model {} is not supported.'.format(p.backbone_name))
    self.backbone_name = p.backbone_name
    gp, stem_filters, blocks = efficientnet_builder.backbone_spec(
        p.backbone_name, {'act_type': p.act_type})
    self.backbone_params = gp
    self.stem_filters = stem_filters
    self.blocks = blocks
    self.bn_eps = gp.batch_norm_epsilon
    # channels of reduction_1..5
    self.reduction_channels = {
        b.reduction: b.output_filters for b in blocks if b.reduction
    }
    if p.min_level not in range(1, 6):
      raise ValueError('features.keys ({}) should include min_level ({})'.format(
          [0, 1, 2, 3, 4, 5], p.min_level))

    def hw(level):
      return (self.feat_sizes[level]['height'], self.feat_sizes[level]['width'])

    self.level_hw = {l: hw(l) for l in range(0, p.max_level + 1)}

    # ---- extra levels (P6.. from the last available level) --------------------
    # feats: list of (level, channels) in pyramid order.
    feats = []
    self.extra_levels = []  # [ResampleSpec] in creation order, scope resample_p{l}
    for level in range(p.min_level, p.max_level + 1):
      if level <= 5:
        feats.append((level, self.reduction_channels[level]))
        continue
      prev_level, prev_c = feats[-1]
      in_hw = hw(prev_level)
      out_hw = ((in_hw[0] - 1) // 2 + 1, (in_hw[1] - 1) // 2 + 1)
      mode, pool = _resample_mode(in_hw, out_hw)
      self.extra_levels.append(
          ResampleSpec(
              scope='resample_p%d' % level,
              src=len(feats) - 1,
              in_hw=in_hw,
              out_hw=out_hw,
              in_channels=prev_c,
              has_conv=(prev_c != self.fpn_filters),
              mode=mode,
              pool=pool))
      feats.append((level, self.fpn_filters))
    utils.verify_feats_size([hw(l) for l, _ in feats], self.feat_sizes,
                            p.min_level, p.max_level)
    self.pyramid_in = list(feats)

    # ---- BiFPN cells ----------------------------------------------------------
    if p.fpn_config:
      fpn_config = p.fpn_config
    else:
      fpn_config = fpn_configs.get_fpn_config(p.fpn_name, p.min_level,
                                              p.max_level, p.fpn_weight_method)
    self.fpn_weight_method = fpn_config.weight_method
    if self.fpn_weight_method not in ('fastattn', 'sum', 'attn',
                                      'channel_attn', 'channel_fastattn'):
      raise ValueError('unknown weight_method {}'.format(self.fpn_weight_method))
    self.fpn_nodes = [dict(n) if isinstance(n, dict) else n.as_dict()
                      for n in fpn_config.nodes]
    self.cells = []  # [[NodeSpec]]
    for rep in range(p.fpn_cell_repeats):
      cell_feats = list(feats)  # (level, channels)
      nodes = []
      for i, fnode in enumerate(self.fpn_nodes):
        level = fnode['feat_level']
        scope = 'fpn_cells/cell_%d/fnode%d' % (rep, i)
        inputs = []
        for idx, off in enumerate(fnode['inputs_offsets']):
          src_level, src_c = cell_feats[off]
          mode, pool = _resample_mode(hw(src_level), hw(level))
          inputs.append(
              ResampleSpec(
                  scope='%s/resample_%d_%d_%d' % (scope, idx, off,
                                                  len(cell_feats)),
                  src=off,
                  in_hw=hw(src_level),
                  out_hw=hw(level),
                  in_channels=src_c,
                  has_conv=(src_c != self.fpn_filters),
                  mode=mode,
                  pool=pool))
        nodes.append(
            NodeSpec(
                scope=scope,
                feat_level=level,
                hw=hw(level),
                inputs=inputs,
                op_scope='%s/op_after_combine%d' % (scope, len(cell_feats)),
                out_index=len(cell_feats)))
        cell_feats.append((level, self.fpn_filters))
      # outputs: the last node at each level
      out_idx = {}
      for l in range(p.min_level, p.max_level + 1):
        for i, fnode in enumerate(reversed(self.fpn_nodes)):
          if fnode['feat_level'] == l:
            out_idx[l] = len(cell_feats) - 1 - i
            break
      self.cells.append({'nodes': nodes, 'out_index': out_idx})
      feats = [(l, self.fpn_filters)
               for l in range(p.min_level, p.max_level + 1)]

    # ---- segmentation head -------------------------------------------------------
    self.seg_stages = _seg_stages(self) if self.has_segmentation else []

  def _resolve_heads(self, p):
    """config.heads: a non-empty subset of HEADS (tf2/efficientdet_keras.py:842-884; anything else
    builds no head in the reference and train_lib.py:637 raises)."""
    heads = p.get('heads', None)
    heads = ['object_detection'] if heads is None else list(heads)
    if not heads or any(h not in HEADS for h in heads):
      raise ValueError('No valid head found: {}'.format(heads))
    self.heads = heads
    self.has_detection = 'object_detection' in heads
    self.has_segmentation = 'segmentation' in heads
    if self.has_segmentation and p.data_format == 'channels_first':
      # tf2/efficientdet_keras.py:703 concatenates on axis -1, the WIDTH axis in NCHW
      raise NotImplementedError(
          'segmentation head with channels_first: the reference concatenates on axis -1, '
          'which is a width concat there, not a channel concat')

  # -- convenience ---------------------------------------------------------------
  def conv_after_pool(self, r):
    """True when resample `r` applies its 1x1 conv after the max-pool, at r.out_hw."""
    return self.conv_after_downsample and r.has_conv and r.mode == 'down'

  @property
  def levels(self):
    return list(range(self.min_level, self.max_level + 1))

  def num_anchors_total(self):
    return sum(self.level_hw[l][0] * self.level_hw[l][1] * self.num_anchors
               for l in self.levels)
