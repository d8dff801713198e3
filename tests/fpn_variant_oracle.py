"""CPU oracle of the feature-network variants (TEST INFRASTRUCTURE ONLY): QuFPN, the channel_attn /
channel_fastattn fusion weights and conv_bn_act_pattern, on top of oracle/efficientdet_oracle.py
(whose resample_feature_map already covers conv_after_downsample).

The QuFPN node list is derived here on its own, by closed-form node ids, NOT by the product's
automl_b200/fpn_configs.py; both are held to the real reference by tests/golden/fpn_variants.json.

Restated from (paths under /root/reference/efficientdet):
  tf2/fpn_configs.py:75-163          QuFPN: paths 1-4 and the quad-add nodes
  efficientdet_arch.py:448-468       channel_attn / channel_fastattn (channel axis last, NHWC)
  efficientdet_arch.py:504-533       node op; conv_bn_act_pattern: fuse -> sepconv without bias
                                     -> BN -> act instead of fuse -> act -> sepconv + bias -> BN
"""
import numpy as np
import torch

from oracle import efficientdet_oracle as eo
from oracle import structure_oracle as so
import precision_model as pm


def qufpn_nodes(min_level, max_level):
  """[(feat_level, [input offsets])] of one QuFPN cell.  With L levels, the ids are: inputs
  0..L-1, path 1 (top-down, levels max-1..min), path 2 (bottom-up, min+1..max), path 3
  (bottom-up, min+1..max), path 4 (top-down, max-1..min), L-1 nodes each, then L quad-add nodes
  (max..min).  A level a path skips reads the previous path's output at that level."""
  lo, hi = min_level, max_level
  n = hi - lo + 1
  inp = lambda l: l - lo
  td1 = lambda l: inp(hi) if l == hi else n + (hi - 1 - l)
  bu2 = lambda l: td1(lo) if l == lo else (2 * n - 1) + (l - lo - 1)
  bu3 = lambda l: inp(lo) if l == lo else (3 * n - 2) + (l - lo - 1)
  td4 = lambda l: bu3(hi) if l == hi else (4 * n - 3) + (hi - 1 - l)
  nodes = [(l, [inp(l), td1(l + 1)]) for l in range(hi - 1, lo - 1, -1)]
  nodes += [(l, [inp(l), td1(l), bu2(l - 1)]) for l in range(lo + 1, hi)]
  nodes += [(hi, [inp(hi), bu2(hi - 1)])]
  nodes += [(l, [inp(l), bu3(l - 1)]) for l in range(lo + 1, hi + 1)]
  nodes += [(l, [inp(l), bu3(l), td4(l + 1)]) for l in range(hi - 1, lo, -1)]
  nodes += [(lo, [inp(lo), td4(lo + 1)])]
  nodes += [(l, [bu2(l), td4(l)]) for l in range(hi, lo - 1, -1)]
  assert len(nodes) == 5 * n - 4
  return nodes


class VariantOracle(eo.Oracle):
  """eo.Oracle whose BiFPN layer also builds QuFPN cells, channel-wise fusion and the
  conv_bn_act_pattern node op.  Every other layer is the base oracle's."""

  def build_bifpn_layer(self, feats, feat_sizes, rep, eps):
    p, w = self.p, self.w
    assert not p.fpn_config
    method = p.fpn_weight_method or 'fastattn'
    if (p.fpn_name or 'bifpn') == 'qufpn':
      nodes_cfg = qufpn_nodes(p.min_level, p.max_level)
    else:
      nodes_cfg = so.bifpn_nodes(p.min_level, p.max_level)
    act = lambda t: eo.activation_fn(t, p.act_type)
    feats = list(feats)
    for i, (level, offsets) in enumerate(nodes_cfg):
      scope = 'fpn_cells/cell_%d/fnode%d' % (rep, i)
      th, tw = feat_sizes[level]
      nodes = [self.resample_feature_map(feats[off], '%s/resample_%d_%d_%d' % (scope, idx, off, len(feats)),
                                         th, tw, eps)
               for idx, off in enumerate(offsets)]
      if method.startswith('channel_'):
        # the reference's channel axis is the last one (NHWC)
        names = [scope + '/WSM' + ('' if j == 0 else '_%d' % j) for j in range(len(nodes))]
        new = eo.fuse_features([t.permute(0, 2, 3, 1) for t in nodes], method,
                               [w[nm] for nm in names]).permute(0, 3, 1, 2)
      else:
        new = self.fuse_features(nodes, method, scope)
      op = '%s/op_after_combine%d' % (scope, len(feats))
      if not p.conv_bn_act_pattern:
        new = act(new)
      new = self.store(eo.depthwise_conv2d_same(new, w[op + '/conv/depthwise_kernel']))
      new = eo.conv2d_same(new, w[op + '/conv/pointwise_kernel'])
      if not p.conv_bn_act_pattern:
        new = new + w[op + '/conv/bias'].view(1, -1, 1, 1)
      new = eo.batch_norm_inference(new, w, op + '/bn', eps)
      if p.conv_bn_act_pattern:
        new = act(new)
      feats.append(self.store(new))
    out = {}
    for l in range(p.min_level, p.max_level + 1):
      last = max(j for j, (lvl, _) in enumerate(nodes_cfg) if lvl == l)
      out[l] = feats[len(feats) - len(nodes_cfg) + last]
    return out


def device_weights(arch, w):
  """precision_model.device_weights for the variants: without a node conv bias
  (conv_bn_act_pattern) the fold uses a zero bias."""
  if not arch.conv_bn_act_pattern:
    return pm.device_weights(arch, w)
  w = dict(w)
  added = []
  for cell in arch.cells:
    for node in cell['nodes']:
      name = node.op_scope + '/conv/bias'
      w[name] = np.zeros(arch.fpn_filters, np.float32)
      added.append(name)
  out = pm.device_weights(arch, w)
  for name in added:
    del out[name]
  return out


class DeviceModel(pm.DeviceModel):
  """pm.DeviceModel with the variant oracle."""

  def __init__(self, config, arch, w, x):  # pylint: disable=super-init-not-called
    self.ref = VariantOracle(config, w, torch.float32)
    self.cls_ref, self.box_ref = self.ref(x)
    self.model = VariantOracle(config, device_weights(arch, w), torch.float32, store=eo.fp16_store)
    self.cls_model, self.box_model = self.model(x)
