"""`EfficientDetNet`: the H100 twin of tf2/efficientdet_keras.py:787-915 (inference only).

`EfficientDetNet(model_name=None, config=None, name='', feature_only=False)` resolves the config as
the reference does (:798, a dict is wrapped in hparams_config.Config); calling the network with
`(images, training=False)` returns the reference's output tuple (:906-915):

  * `[class logits per level], [box logits per level]` when config.heads has 'object_detection';
  * then the segmentation logits [N, 2H_min, 2W_min, seg_num_classes] when it has 'segmentation'
    (SegmentationHead, :644-706);

as float32 tensors on the device, NHWC (NCHW for channels_first detection outputs, like the
reference).  Not supported, with NotImplementedError: training=True, feature_only=True, and
channels_first together with the segmentation head (the reference concatenates on axis -1 there,
a width concat rather than a channel concat).

Differences forced by the runtime: images are a float32 tensor or array (copied to the device),
and variables are not created by the layers: pass them with `weights=` (dict keyed by reference
variable names, Keras layouts); without it seeded synthetic weights are used.
"""
import torch

from automl_b200 import efficientdet_arch
from automl_b200 import hparams_config
from automl_b200.arch import DetArch


class EfficientDetNet(object):
  """EfficientDet network without pre / post-processing, on one H100."""

  def __init__(self, model_name=None, config=None, name='', feature_only=False, weights=None,
               device='cuda:0'):
    if feature_only:
      raise NotImplementedError('feature_only=True: the class / box nets return their tower '
                                'features only in training graphs, which this runtime does not build')
    config = config or hparams_config.get_efficientdet_config(model_name)
    if isinstance(config, dict):
      config = hparams_config.Config(config)
    self.config = config
    self.name = name
    self.arch = DetArch(config)   # validates heads, sizes and the data format up front
    self.weights = weights
    self.device = device

  def __call__(self, inputs, training=False):
    if training:
      raise NotImplementedError('training=True: this runtime is inference only')
    x = torch.as_tensor(inputs)
    channels_first = self.config.data_format == 'channels_first'
    if channels_first:
      x = x.permute(0, 2, 3, 1)
    eng = efficientdet_arch.get_engine(self.config, x.shape[0], weights=self.weights,
                                       device=self.device)
    cls_out, box_out = eng.forward(x.contiguous())
    outputs = []
    if self.arch.has_detection:
      levels = self.arch.levels
      cls_l = [cls_out[l].float() for l in levels]
      box_l = [box_out[l].float() for l in levels]
      if channels_first:
        cls_l = [t.permute(0, 3, 1, 2) for t in cls_l]
        box_l = [t.permute(0, 3, 1, 2) for t in box_l]
      outputs.extend([cls_l, box_l])
    if self.arch.has_segmentation:
      outputs.append(eng.seg_logits.float())
    return tuple(outputs)
