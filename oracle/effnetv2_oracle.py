"""CPU oracle for the EfficientNet V1/V2 backbone: the reference's
efficientnetv2/effnetv2_model.py forward pass restated in PyTorch (CPU, fp32 / fp64).

TEST INFRASTRUCTURE ONLY (same rule as efficientdet_oracle.py): nothing under automl_b200/
imports this module; tests/ use it as the checker.  It imports nothing from automl_b200 either:
the network it walks is its own (oracle/effnetv2_structure.py), built from the model NAME and the
model_config override only.

Parity status: "parity unpinned" for the convolution numerics (TensorFlow is not installable
here, Appendix C of SURVEY.md).  The structure is pinned to the REAL reference constructor for all
18 registered names and structure-changing overrides (tests/golden/effnetv2_structure.json.gz:
every block's resolved block args, every layer's kind, filters, kernel, stride, bias, name and BN
epsilon; tests/test_effnetv2_structure_pins.py), and by `count_params()` of 15 models
(effnetv2_model_test.py:25-48).  Functions cite /root/reference/efficientnetv2/effnetv2_model.py
lines.
"""
import torch

from oracle import efficientdet_oracle as eo
from oracle import effnetv2_structure


def structure_of(arch, model_config=None):
  """The oracle's own Structure for `arch`: a model name, or any object with a `model_name` (e.g.
  the product's EffNetV2Arch).  Of such an object only `model_name` and the override it was built
  with (`model_config`, the caller's dict as given, never a resolved value) are read.  An override
  passed here must equal the arch's: a model_config is never dropped, and never silently replaced."""
  if isinstance(arch, str):
    name, built_with = arch, None
  else:
    name, built_with = arch.model_name, getattr(arch, 'model_config', None)
  if built_with and model_config and built_with != model_config:
    raise ValueError('%s was built with model_config %r, the oracle was given %r'
                     % (name, built_with, model_config))
  return effnetv2_structure.Structure(name, model_config or built_with)


class EffNetV2Oracle(object):
  """call(images NHWC float) -> dict of endpoints (NCHW tensors): 'stem', 'block_i',
  'reduction_i', 'features', 'head_1x1' (EffNetV2Model.call :595-658)."""

  def __init__(self, arch, weights, dtype=torch.float32, store=None, model_config=None):
    """arch, model_config: see structure_of."""
    self.s = structure_of(arch, model_config)
    self.arch = arch            # for callers' own bookkeeping; the forward walk reads only self.s
    self.model_name = self.s.model_name
    self.dtype = dtype
    self.w = {k: torch.as_tensor(v).to(dtype) for k, v in weights.items()}
    self.store = store or (lambda t: t)     # e.g. eo.fp16_store to model fp16 activations
    self.act = lambda t: eo.activation_fn(t, self.s.act_fn)

  def _bn(self, x, scope):
    return eo.batch_norm_inference(x, self.w, scope, self.s.bn_epsilon)

  def _se(self, x, sc):
    """SE.call :135-147: reduce_mean -> conv(+bias) -> act -> conv(+bias) -> sigmoid * x."""
    w = self.w
    s = x.mean((2, 3), keepdim=True)
    s = eo.conv2d_same(s, w[sc + '/se/conv2d/kernel']) + w[sc + '/se/conv2d/bias'].view(1, -1, 1, 1)
    s = self.act(s)
    s = eo.conv2d_same(s, w[sc + '/se/conv2d_1/kernel']) + w[sc + '/se/conv2d_1/bias'].view(1, -1, 1, 1)
    return torch.sigmoid(s) * x

  def _block(self, b, x):
    """b: one block dict of effnetv2_structure.Structure."""
    w, sc = self.w, '%s/%s' % (self.model_name, b['name'])

    def conv(x, name, stride=1):
      return eo.conv2d_same(x, w['%s/%s/kernel' % (sc, name)], stride)

    def bn(x, name):
      return self._bn(x, '%s/%s' % (sc, name))

    inputs = x
    if b['conv_type'] == 0:   # MBConvBlock.call :279-311
      if b['expand_name']:
        x = self.store(self.act(bn(conv(x, b['expand_name']), b['expand_bn'])))
      x = self.act(bn(eo.depthwise_conv2d_same(x, w[sc + '/depthwise_conv2d/depthwise_kernel'],
                                               b['strides']), b['dw_bn']))
      if b['has_se']:
        # the device folds the gate into the project weights: the depthwise output is stored,
        # the gated tensor is not
        x = self._se(self.store(x), sc)
      else:
        x = self.store(x)
      x = bn(conv(x, b['project_name']), b['project_bn'])
    else:                     # FusedMBConvBlock.call :375-406
      if b['expand_name']:
        x = self.store(self.act(bn(conv(x, b['expand_name'], b['strides']), b['expand_bn'])))
      if b['has_se']:
        x = self._se(x, sc)
      stride = 1 if b['expand_name'] else b['strides']
      x = bn(conv(x, b['project_name'], stride), b['project_bn'])
      if not b['expand_name']:
        x = self.act(x)       # add act if no expansion (:401-402)
    if b['has_skip']:         # residual :266-273 (drop_connect is the identity at inference)
      x = x + inputs
    return self.store(x)

  def __call__(self, images):
    s, w, mn = self.s, self.w, self.model_name
    x = torch.as_tensor(images).to(self.dtype).permute(0, 3, 1, 2)
    ep = {}
    x = self.store(self.act(self._bn(eo.conv2d_same(x, w[mn + '/stem/conv2d/kernel'], 2),
                                     mn + '/stem/tpu_batch_normalization')))  # Stem :409-432
    ep['stem'] = x
    red = 0
    for i, b in enumerate(s.blocks):
      x = self._block(b, x)
      ep['block_%d' % i] = x
      if i in s.reductions:
        red += 1
        ep['reduction_%d' % red] = x
    ep['features'] = x
    x = self.store(self.act(self._bn(eo.conv2d_same(x, w[mn + '/head/conv2d/kernel']),
                                     mn + '/head/tpu_batch_normalization')))  # Head :472-474
    ep['head_1x1'] = x
    return ep
