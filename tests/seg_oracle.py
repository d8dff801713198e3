"""CPU oracle of the segmentation head (TEST INFRASTRUCTURE ONLY): SegmentationHead restated in
torch (float32 / float64) on top of oracle/efficientdet_oracle.py's backbone and feature network.

Restated from (paths under /root/reference/efficientdet):
  tf2/efficientdet_keras.py:644-692   layers: max_level - min_level Conv2DTranspose(F, 3, 2,
                                      'same', use_bias=False) + BN 'bn_<i>', then
                                      Conv2DTranspose(seg_num_classes, 3, 2, 'same') with bias
  tf2/efficientdet_keras.py:694-706   call: x = P_max; per stage convT -> BN -> act -> concat
                                      [x, skip] on the channel axis; skips P_max-1 .. P_min
  tf2/efficientdet_keras.py:875-884, 912-915   built / returned when 'segmentation' in heads

Conv2DTranspose 'SAME' stride 2 is tf.nn.conv2d_transpose, the adjoint of the k3 s2 'SAME' conv2d
(whose extra padding cell lies after the data, tests/test_tf_semantics_pins.py): per axis
out[y] = sum_i x[i] w[y - 2i] for y - 2i in {0, 1, 2}, output size 2H.  That is torch's
conv_transpose2d without padding (size 2H + 1) cropped to its FIRST 2H rows / columns -- not the
padding=1, output_padding=1 convention, which keeps rows 1 .. 2H instead.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import efficientdet_oracle as eo


def conv2d_transpose_same(x, kernel):
  """x [N, Cin, H, W]; kernel [3, 3, Cout, Cin] (Keras layout) -> [N, Cout, 2H, 2W]."""
  h, w = x.shape[2], x.shape[3]
  full = F.conv_transpose2d(x, kernel.permute(3, 2, 0, 1), stride=2)
  return full[:, :, :2 * h, :2 * w]


def layers(config):
  """The layer list SegmentationHead.__init__ creates, in tests/golden/seg_structure.json's form."""
  out = []
  for i in range(config.max_level - config.min_level):
    out.append(['conv_transpose', config.fpn_num_filters, 3, 2, 'same', False])
    out.append(['bn', 'bn_%d' % i])
  out.append(['conv_transpose', config.seg_num_classes, 3, 2, 'same', True])
  return out


def seg_head(config, w, feats, eps, store=None):
  """SegmentationHead.call: feats = BiFPN outputs P_min .. P_max (NCHW); w = the Oracle's weight
  tensors.  Returns NHWC logits.  Scope names as automl_b200/arch.py names the variables."""
  store = store or (lambda t: t)
  x = feats[-1]
  skips = list(reversed(feats[:-1]))
  for i, skip in enumerate(skips):
    scope = 'segmentation_head/conv2d_transpose' + ('_%d' % i if i else '')
    x = conv2d_transpose_same(x, w[scope + '/kernel'])
    x = eo.batch_norm_inference(x, w, 'segmentation_head/bn_%d' % i, eps)
    x = store(eo.activation_fn(x, config.act_type))
    x = torch.cat([x, skip], dim=1)
  scope = 'segmentation_head/conv2d_transpose_%d' % len(skips)
  x = conv2d_transpose_same(x, w[scope + '/kernel']) + w[scope + '/bias'].view(1, -1, 1, 1)
  return store(x).permute(0, 2, 3, 1).contiguous()


def seg_logits(config, weights, images_nhwc, dtype=torch.float32, store=None):
  """Backbone + feature network of the detection oracle, then the segmentation head; `store`
  models the rounding of every stored tensor (eo.Oracle)."""
  o = eo.Oracle(config, weights, dtype, store=store)
  x = o.store(torch.as_tensor(np.asarray(images_nhwc)).to(dtype).permute(0, 3, 1, 2))
  feats, eps = o.backbone(x)
  features = {0: x}
  features.update(feats)
  fpn = o.build_feature_network(features, eps)
  return seg_head(config, o.w, [fpn[l] for l in range(config.min_level, config.max_level + 1)], eps,
                  store=o.store)
