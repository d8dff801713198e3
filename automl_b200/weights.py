"""Variable inventory and seeded synthetic weights, keyed by reference variable names.

The weight format of the reference is de facto its TF variable names
(SURVEY.md section 5); this module enumerates them for a resolved `DetArch` with
Keras kernel layouts so that a real checkpoint can be dropped in later:

  Conv2D.kernel                 [kh, kw, Cin, Cout]
  DepthwiseConv2D.depthwise_kernel / SeparableConv2D.depthwise_kernel [kh, kw, C, 1]
  SeparableConv2D.pointwise_kernel [1, 1, C, Cout], .bias [Cout]
  BatchNormalization            gamma, beta, moving_mean, moving_variance [C]
  BiFPN fusion weights          WSM, WSM_1, WSM_2 (scalar; [F] for channel_* methods)

Name generators follow efficientnet_model.py:272-277 (conv2d[_n], tpu_batch_normalization[_n]),
efficientdet_keras.py:123-131 (WSM names), :152-160 (op_after_combine{n}/conv, bn),
:399-420 (class-{i}, class-{i}-bn-{level}, class-predict), :306-333 (resample_p{level}).

Synthetic initialisation (no checkpoints offline): the reference initialiser
*scales* (conv N(0, sqrt(2/fan_out)) efficientnet_model.py:52-73, class bias
-log(99) efficientdet_arch.py:188) but non-trivial BN moving statistics and WSM
so BN folding and fusion weighting are exercised (SURVEY.md section 8d).
"""
import collections
import math

import numpy as np

VarSpec = collections.namedtuple('VarSpec', ['shape', 'kind', 'trainable'])


def _bn(specs, scope, c):
  specs[scope + '/gamma'] = VarSpec((c,), 'gamma', True)
  specs[scope + '/beta'] = VarSpec((c,), 'beta', True)
  specs[scope + '/moving_mean'] = VarSpec((c,), 'mean', False)
  specs[scope + '/moving_variance'] = VarSpec((c,), 'var', False)


def variable_specs(arch):
  """OrderedDict name -> VarSpec for every variable of the network."""
  s = collections.OrderedDict()
  bb = arch.backbone_name
  # stem
  s['%s/stem/conv2d/kernel' % bb] = VarSpec((3, 3, 3, arch.stem_filters),
                                            'conv', True)
  _bn(s, '%s/stem/tpu_batch_normalization' % bb, arch.stem_filters)
  # blocks
  for b in arch.blocks:
    scope = '%s/%s' % (bb, b.name)
    if b.expand_name:
      s['%s/%s/kernel' % (scope, b.expand_name)] = VarSpec(
          (1, 1, b.input_filters, b.mid_filters), 'conv', True)
      _bn(s, '%s/%s' % (scope, b.expand_bn), b.mid_filters)
    s['%s/depthwise_conv2d/depthwise_kernel' % scope] = VarSpec(
        (b.kernel_size, b.kernel_size, b.mid_filters, 1), 'dw', True)
    _bn(s, '%s/%s' % (scope, b.dw_bn), b.mid_filters)
    if b.se_filters:
      s['%s/se/conv2d/kernel' % scope] = VarSpec(
          (1, 1, b.mid_filters, b.se_filters), 'conv', True)
      s['%s/se/conv2d/bias' % scope] = VarSpec((b.se_filters,), 'se_bias', True)
      s['%s/se/conv2d_1/kernel' % scope] = VarSpec(
          (1, 1, b.se_filters, b.mid_filters), 'conv', True)
      s['%s/se/conv2d_1/bias' % scope] = VarSpec((b.mid_filters,), 'se_bias',
                                                 True)
    s['%s/%s/kernel' % (scope, b.project_name)] = VarSpec(
        (1, 1, b.mid_filters, b.output_filters), 'conv', True)
    _bn(s, '%s/%s' % (scope, b.project_bn), b.output_filters)

  f = arch.fpn_filters

  def resample(r):
    if r.has_conv:
      s[r.scope + '/conv2d/kernel'] = VarSpec((1, 1, r.in_channels, f), 'conv',
                                              True)
      s[r.scope + '/conv2d/bias'] = VarSpec((f,), 'bias', True)
      if arch.config.apply_bn_for_resampling:
        _bn(s, r.scope + '/bn', f)

  for r in arch.extra_levels:
    resample(r)
  for cell in arch.cells:
    for node in cell['nodes']:
      for r in node.inputs:
        resample(r)
      if arch.fpn_weight_method in ('attn', 'fastattn', 'channel_attn',
                                    'channel_fastattn'):
        shape = (f,) if arch.fpn_weight_method.startswith('channel') else ()
        for i in range(len(node.inputs)):
          s['%s/WSM%s' % (node.scope, '' if i == 0 else '_%d' % i)] = VarSpec(
              shape, 'wsm', True)
      s[node.op_scope + '/conv/depthwise_kernel'] = VarSpec((3, 3, f, 1),
                                                            'sep_dw', True)
      s[node.op_scope + '/conv/pointwise_kernel'] = VarSpec((1, 1, f, f),
                                                            'sep_pw', True)
      if not arch.conv_bn_act_pattern:   # use_bias=not conv_bn_act_pattern (:520)
        s[node.op_scope + '/conv/bias'] = VarSpec((f,), 'bias', True)
      _bn(s, node.op_scope + '/bn', f)

  dets = ((('class', arch.num_classes * arch.num_anchors, 'class_bias'),
           ('box', 4 * arch.num_anchors, 'bias')) if arch.has_detection else ())
  for net, pred_c, pred_kind in dets:
    scope = '%s_net' % net
    for i in range(arch.head_repeats):
      s['%s/%s-%d/depthwise_kernel' % (scope, net, i)] = VarSpec(
          (3, 3, f, 1), 'sep_dw', True)
      s['%s/%s-%d/pointwise_kernel' % (scope, net, i)] = VarSpec(
          (1, 1, f, f), 'sep_pw', True)
      s['%s/%s-%d/bias' % (scope, net, i)] = VarSpec((f,), 'bias', True)
      for level in arch.levels:
        _bn(s, '%s/%s-%d-bn-%d' % (scope, net, i, level), f)
    s['%s/%s-predict/depthwise_kernel' % (scope, net)] = VarSpec(
        (3, 3, f, 1), 'sep_dw', True)
    s['%s/%s-predict/pointwise_kernel' % (scope, net)] = VarSpec(
        (1, 1, f, pred_c), 'sep_pw', True)
    s['%s/%s-predict/bias' % (scope, net)] = VarSpec((pred_c,), pred_kind, True)

  # segmentation head (tf2/efficientdet_keras.py:676-692), only when configured; the names are
  # Keras' default layer names (arch._seg_stages), not checkable offline
  for st in arch.seg_stages:
    s[st.kernel_scope + '/kernel'] = VarSpec((3, 3, st.out_channels, st.in_channels),
                                             'conv_transpose', True)
    if st.bn_scope:
      _bn(s, st.bn_scope, st.out_channels)
    else:
      s[st.kernel_scope + '/bias'] = VarSpec((st.out_channels,), 'bias', True)
  return s


def count_params(arch, trainable_only=True):
  n = 0
  for spec in variable_specs(arch).values():
    if spec.trainable or not trainable_only:
      n += int(np.prod(spec.shape)) if spec.shape else 1
  return n


def synthetic_weights(arch, seed=0):
  """Seeded float32 numpy weights: OrderedDict name -> ndarray."""
  rng = np.random.default_rng(seed)
  out = collections.OrderedDict()
  for name, spec in variable_specs(arch).items():
    shape, kind = spec.shape, spec.kind
    if kind in ('conv', 'dw', 'sep_dw', 'sep_pw'):
      kh, kw, cin, cout = shape
      if kind in ('dw', 'sep_dw'):
        # keras depthwise: fan_out as written in conv_kernel_initializer uses
        # shape[-1]==1, giving a large stddev; keep activations O(1) instead.
        std = math.sqrt(2.0 / (kh * kw)) * 0.7
      elif kind == 'sep_pw':
        std = math.sqrt(1.0 / cin)
      else:
        # fan_in scaling keeps 200 stacked layers O(1) with swish in between.
        std = math.sqrt(2.0 / (kh * kw * cin))
      w = rng.normal(0.0, std, size=shape)
    elif kind == 'conv_transpose':
      # Keras' default glorot_uniform on the (kh, kw, out, in) kernel: fan_in = kh*kw*out,
      # fan_out = kh*kw*in (Conv2DTranspose keeps the reference's default initialiser)
      kh, kw, cout, cin = shape
      limit = math.sqrt(6.0 / (kh * kw * (cout + cin)))
      w = rng.uniform(-limit, limit, size=shape)
    elif kind == 'gamma':
      w = rng.uniform(0.8, 1.2, size=shape)
    elif kind == 'beta':
      w = rng.normal(0.0, 0.1, size=shape)
    elif kind == 'mean':
      w = rng.normal(0.0, 0.1, size=shape)
    elif kind == 'var':
      w = rng.uniform(0.5, 1.5, size=shape)
    elif kind == 'wsm':
      w = rng.uniform(0.5, 1.5, size=shape)
    elif kind == 'se_bias':
      w = rng.normal(0.0, 0.1, size=shape)
    elif kind == 'bias':
      w = rng.normal(0.0, 0.02, size=shape)
    elif kind == 'class_bias':
      w = np.full(shape, -math.log((1 - 0.01) / 0.01)) + rng.normal(
          0.0, 0.02, size=shape)
    else:
      raise AssertionError(kind)
    out[name] = np.asarray(w, dtype=np.float32)
  return out
