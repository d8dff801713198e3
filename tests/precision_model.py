"""CPU model of the device's PRECISION (not of its kernels): the oracle network evaluated with

  * every tensor the engine writes to HBM rounded to fp16 (`Oracle(store=fp16_store)`), and
  * the GEMM weights the engine uploads: inference BatchNorm folded into the 1x1 / stem kernels in
    float64, THEN rounded to fp16 (`lowering.py::bn_fold` + `_dev(..., f16)`); depthwise taps and
    biases stay fp32, as on the device.

All arithmetic stays fp32 on the CPU.  The difference between this model and the plain fp32
oracle is therefore the error that the fp16 STORAGE FORMAT mandates for a given network, weights
and input, independent of any kernel.  Tests use it where the 1e-3 bar of north_star cannot be
met by an fp16-storage design on seeded random weights (55-block D7x, relu6 lite nets, an
ill-conditioned draw of the un-normalised 'sum' fusion): the device must then stay within a
small factor of the model, i.e. the kernels add nothing beyond the format (DESIGN.md section 6).

Test infrastructure: imports the product only for the variable NAMES of a resolved architecture.
"""
import numpy as np
import torch

from oracle import efficientdet_oracle as eo

EPS = eo.BN_EPSILON


def _r16(a):
  return np.asarray(a, np.float64).astype(np.float16).astype(np.float32)


def _fold(w, out, kernel, bn, conv_bias=None, depthwise=False, rnd=None):
  """kernel' = kernel * bn_scale (rounded to fp16 unless depthwise); the BN that follows becomes
  the identity scale with beta' chosen so that (conv' + conv_bias) + beta' == BN(conv + conv_bias)."""
  g, b = np.float64(w[bn + '/gamma']), np.float64(w[bn + '/beta'])
  m, v = np.float64(w[bn + '/moving_mean']), np.float64(w[bn + '/moving_variance'])
  s = g / np.sqrt(v + EPS)
  sh = b - m * s
  k = np.float64(w[kernel])
  k = k * (s.reshape(1, 1, -1, 1) if depthwise else s.reshape(1, 1, 1, -1))
  out[kernel] = k.astype(np.float32) if depthwise else (rnd or _r16)(k)
  cb = np.float64(w[conv_bias]) if conv_bias else 0.0
  out[bn + '/gamma'] = np.ones_like(g, np.float32)
  out[bn + '/moving_variance'] = np.full(g.shape, 1.0 - EPS, np.float32)
  out[bn + '/moving_mean'] = np.zeros_like(g, np.float32)
  out[bn + '/beta'] = (sh + cb * s - cb).astype(np.float32)


def device_weights(arch, w, round_gemm_weights=True):
  """The weight dict the oracle must be given to see the values the engine computes with
  (round_gemm_weights=False: only the BN fold, which must leave the fp32 network unchanged)."""
  out = dict(w)
  rnd = _r16 if round_gemm_weights else (lambda k: np.asarray(k, np.float32))
  bb = arch.backbone_name
  _fold(w, out, bb + '/stem/conv2d/kernel', bb + '/stem/tpu_batch_normalization', rnd=rnd)
  for b in arch.blocks:
    sc = '%s/%s' % (bb, b.name)
    if b.expand_name:
      _fold(w, out, '%s/%s/kernel' % (sc, b.expand_name), '%s/%s' % (sc, b.expand_bn), rnd=rnd)
    _fold(w, out, sc + '/depthwise_conv2d/depthwise_kernel', '%s/%s' % (sc, b.dw_bn), depthwise=True)
    _fold(w, out, '%s/%s/kernel' % (sc, b.project_name), '%s/%s' % (sc, b.project_bn), rnd=rnd)
  def resample(r):
    if r.has_conv:
      if arch.config.apply_bn_for_resampling:
        _fold(w, out, r.scope + '/conv2d/kernel', r.scope + '/bn', r.scope + '/conv2d/bias', rnd=rnd)
      else:
        out[r.scope + '/conv2d/kernel'] = rnd(w[r.scope + '/conv2d/kernel'])
  for r in arch.extra_levels:
    resample(r)
  for cell in arch.cells:
    for node in cell['nodes']:
      for r in node.inputs:
        resample(r)
      op = node.op_scope
      _fold(w, out, op + '/conv/pointwise_kernel', op + '/bn', op + '/conv/bias', rnd=rnd)
  for net in ('class', 'box'):
    # tower layers: one pointwise kernel shared by the levels, one BN per level -> the engine folds
    # per level; modelled by rounding the shared kernel (the per-level scale is a per-column factor
    # of O(1), so the relative rounding error is the same)
    for i in range(arch.head_repeats):
      name = '%s_net/%s-%d/pointwise_kernel' % (net, net, i)
      out[name] = rnd(w[name])
    name = '%s_net/%s-predict/pointwise_kernel' % (net, net)
    out[name] = rnd(w[name])
  return out


def effnetv2_device_weights(arch, w, model_config=None):
  """The same for the EfficientNet V1 / V2 backbone (EffNetV2Model._build, lowering.py): BN
  folded into fp16 conv kernels (1x1 and k x k), fp32 depthwise taps.  The layers are the oracle's
  own (oracle/effnetv2_oracle.py::structure_of), not the product's."""
  from oracle import effnetv2_oracle  # pylint: disable=g-import-not-at-top
  st = effnetv2_oracle.structure_of(arch, model_config)
  out = dict(w)
  mn, eps = st.model_name, st.bn_epsilon

  def fold(kernel, bn, depthwise=False):
    g, b = np.float64(w[bn + '/gamma']), np.float64(w[bn + '/beta'])
    m, v = np.float64(w[bn + '/moving_mean']), np.float64(w[bn + '/moving_variance'])
    s = g / np.sqrt(v + eps)
    k = np.float64(w[kernel]) * (s.reshape(1, 1, -1, 1) if depthwise else s.reshape(1, 1, 1, -1))
    out[kernel] = k.astype(np.float32) if depthwise else _r16(k)
    out[bn + '/gamma'] = np.ones_like(g, np.float32)
    out[bn + '/moving_variance'] = np.full(g.shape, 1.0 - eps, np.float32)
    out[bn + '/moving_mean'] = np.zeros_like(g, np.float32)
    out[bn + '/beta'] = (b - m * s).astype(np.float32)

  fold(mn + '/stem/conv2d/kernel', mn + '/stem/tpu_batch_normalization')
  for b in st.blocks:
    sc = '%s/%s' % (mn, b['name'])
    if b['expand_name']:
      fold('%s/%s/kernel' % (sc, b['expand_name']), '%s/%s' % (sc, b['expand_bn']))
    if b['dw_bn']:
      fold(sc + '/depthwise_conv2d/depthwise_kernel', '%s/%s' % (sc, b['dw_bn']), depthwise=True)
    fold('%s/%s/kernel' % (sc, b['project_name']), '%s/%s' % (sc, b['project_bn']))
  fold(mn + '/head/conv2d/kernel', mn + '/head/tpu_batch_normalization')
  return out


def effnetv2_format_errors(arch, w, x, model_config=None):
  """{endpoint: rel-L2 of the format model vs the fp32 oracle} and the fp32 endpoints."""
  from oracle import effnetv2_oracle  # pylint: disable=g-import-not-at-top
  ref = effnetv2_oracle.EffNetV2Oracle(arch, w, torch.float32, model_config=model_config)(x)
  mod = effnetv2_oracle.EffNetV2Oracle(arch, effnetv2_device_weights(arch, w, model_config),
                                       torch.float32, store=eo.fp16_store,
                                       model_config=model_config)(x)
  return {k: DeviceModel.rel_l2(mod[k], ref[k]) for k in ref}, ref


class DeviceModel(object):
  """fp32 oracle + the oracle at device precision for one (config, weights, input)."""

  def __init__(self, config, arch, w, x):
    self.ref = eo.Oracle(config, w, torch.float32)
    self.cls_ref, self.box_ref = self.ref(x)
    self.model = eo.Oracle(config, device_weights(arch, w), torch.float32, store=eo.fp16_store)
    self.cls_model, self.box_model = self.model(x)

  @staticmethod
  def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))

  def endpoint_error(self, name):
    return self.rel_l2(self.model.endpoints[name], self.ref.endpoints[name])

  def cls_error(self, level):
    return self.rel_l2(self.cls_model[level], self.cls_ref[level])

  def box_error(self, level):
    return self.rel_l2(self.box_model[level], self.box_ref[level])


def bar(model_error, factor=1.5, slack=1e-4):
  """Device error allowed for a tensor whose format-mandated error is `model_error`."""
  return factor * model_error + slack
