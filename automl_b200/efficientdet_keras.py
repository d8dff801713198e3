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

`EfficientDetModel(EfficientDetNet)`, the twin of :918-1003, adds the pre- and post-processing:
calling it with `(inputs, training=False, pre_mode='infer', post_mode='global')` pre-processes
channels-last uint8 or float32 images of any size on the device (edet_preprocess /
edet_preprocess_float), runs the network once and returns postprocess_global's
`(boxes, scores, classes, valid_len)` from the engine's NMS-V5 stage, followed by the segmentation
logits when config.heads has 'segmentation'.
"""
import numpy as np
import torch

from automl_b200 import efficientdet_arch
from automl_b200 import hparams_config
from automl_b200 import inference
from automl_b200 import ops
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
    return tuple(self._network_outputs(eng, cls_out, box_out))

  def _network_outputs(self, eng, cls_out, box_out):
    """The reference's output list of one forward of `eng` (:906-915), as owned float32 tensors."""
    outputs = []
    if self.arch.has_detection:
      channels_first = self.config.data_format == 'channels_first'
      levels = self.arch.levels
      cls_l = [cls_out[l].float() for l in levels]
      box_l = [box_out[l].float() for l in levels]
      if channels_first:
        cls_l = [t.permute(0, 3, 1, 2) for t in cls_l]
        box_l = [t.permute(0, 3, 1, 2) for t in box_l]
      outputs.extend([cls_l, box_l])
    if self.arch.has_segmentation:
      outputs.append(eng.seg_logits.float())
    return outputs


_UNBUILT_POST_MODES = ('per_class', 'combined', 'tflite')


class EfficientDetModel(EfficientDetNet):
  """EfficientDet with pre- and post-processing (tf2/efficientdet_keras.py:918-1003), on one H100.

  `model(inputs, training=False, pre_mode='infer', post_mode='global')`:

    * inputs: channels-last [N, h, w, 3] images, uint8 or float32, a numpy array or a torch tensor
      on the host or on the model's device (read in order on the current stream).  channels_first
      configs take NHWC input too: the reference pre-processes NHWC and transposes afterwards.
    * pre_mode='infer': images of any h x w, normalised, resized to fit config.image_size and zero
      padded on the device; each image's scale back to the original goes to the post-process.
      pre_mode=None: inputs are the float32 network input [N, H, W, 3], scales 1.
    * post_mode='global' (config.heads has 'object_detection'): postprocess_global's
      boxes float32 [N, M, 4] (ymin, xmin, ymax, xmax, clipped to image_size, times the scale),
      scores float32 [N, M], classes float32 [N, M] (CLASS_OFFSET added) and valid_len int32 [N],
      M = nms_configs.max_output_size; rows past valid_len hold anchor 0's box and class with
      score 0, as tf.gather of the zero-padded NMS indices gives.  post_mode=None: the per-level
      class and box logits, as EfficientDetNet returns them.
    * the segmentation logits follow when config.heads has 'segmentation', from the same pass.

  One engine per batch size (efficientdet_arch.get_engine).  The returned tensors live on the
  device, belong to the caller (a later call does not overwrite them) and are ready on the current
  stream.  Raised before anything is enqueued: ValueError for another pre_mode, an unknown
  post_mode, or inputs of another dtype or shape; NotImplementedError for training=True and the
  post modes 'per_class', 'combined' and 'tflite', which are not built."""

  def __call__(self, inputs, training=False, pre_mode='infer', post_mode='global'):
    if training:
      raise NotImplementedError('training=True: this runtime is inference only')
    if pre_mode and pre_mode != 'infer':
      raise ValueError('preprocessing must be infer or empty')
    detect = self.arch.has_detection and bool(post_mode)
    if detect and post_mode != 'global':
      if post_mode in _UNBUILT_POST_MODES:
        raise NotImplementedError("post_mode=%r: only 'global' and None are built" % (post_mode,))
      raise ValueError('Unsupported postprocess mode {}'.format(post_mode))
    x = self._images(inputs, pre_mode).to(self.device).contiguous()
    with torch.cuda.device(self.device):
      eng = efficientdet_arch.get_engine(self.config, x.shape[0], weights=self.weights,
                                         device=self.device)
      scale = 1.0
      if not pre_mode:
        eng.input.copy_(x)
      else:
        mean, std = inference._rgb3(self.config.mean_rgb), inference._rgb3(self.config.stddev_rgb)
        pre = ops.preprocess if x.dtype == torch.uint8 else ops.preprocess_float
        scale = pre(x, eng.input, mean, std)
      if not detect:
        return tuple(self._network_outputs(eng, *eng.forward()))
      det = eng.detect(image_scales=np.full(x.shape[0], scale, np.float32))
      own = lambda t: t.clone(memory_format=torch.contiguous_format)
      outputs = [own(det[..., 1:5]), own(det[..., 5]), own(det[..., 6]), own(eng.valid)]
      if self.arch.has_segmentation:
        outputs.append(eng.seg_logits.float())
    return tuple(outputs)

  def _images(self, inputs, pre_mode):
    """`inputs` as a [N, h, w, 3] uint8 or float32 tensor, where it is; ValueError for anything
    the call does not take."""
    if isinstance(inputs, torch.Tensor):
      x = inputs
      dtype_ok = x.dtype in (torch.uint8, torch.float32)
    else:
      a = np.asarray(inputs)
      dtype_ok = a.dtype in (np.uint8, np.float32)
      x = torch.from_numpy(np.ascontiguousarray(a)) if dtype_ok else None
    if not dtype_ok:
      raise ValueError('images must be uint8 or float32, got %s' % getattr(inputs, 'dtype', type(inputs)))
    if x.dim() != 4 or x.shape[3] != 3 or 0 in x.shape:
      raise ValueError('images must be channels-last [N, h, w, 3], got %s' % (tuple(x.shape),))
    if x.shape[0] > 65535:
      raise ValueError('a batch of %d images: at most 65535 per call' % x.shape[0])
    if x.is_cuda:
      want = torch.device(self.device)
      if want.index is None:
        want = torch.device('cuda', torch.cuda.current_device())
      if x.device != want:
        raise ValueError('images are on %s, the model runs on %s' % (x.device, want))
    hw = tuple(int(v) for v in x.shape[1:3])
    if not pre_mode:
      if x.dtype != torch.float32 or hw != tuple(self.arch.image_hw):
        raise ValueError('pre_mode=None takes the float32 network input [N, %d, %d, 3], got %s %s'
                         % (self.arch.image_hw + (x.dtype, tuple(x.shape))))
    else:
      inference.preprocess_table([hw], self.arch.image_hw)   # ValueError if it collapses to 0 rows
    return x
