"""Weighted box fusion for test-time augmentation on the H100 path: the call surface of the
reference's /root/reference/efficientdet/tf2/wbf.py.

  ensemble_detections(params, detections, num_models)
      wbf.py:70-95 for one image: detections [R, 7] rows [image_id, x1, y1, x2, y2, score, class]
      (the concatenated rows of num_models "models") -> float32 [k, 7] device tensor of clusters,
      sorted by score.  One edet_wbf launch.
  ensemble_detections_batch(params, detections, num_models, image_scales=None, mirrored_mask=0)
      every image of a batch in one launch: detections [num_models * N, rows, 7] (model m of image i
      at block m * N + i, what edet_per_class_nms writes for num_models * N images) ->
      (clusters float32 [N, num_models * rows, 7], counts int32 [N]) device tensors.

Bit-identical to wbf.py run in float32, including its class range: only classes 0 .. num_classes-1
are fused, so with nms_np's 1-based classes the last class is dropped and nms_np's dummy rows
(class 0, score -1e5) form one cluster (include/automl_b200.h, edet_wbf).
"""
import torch

from automl_b200 import ops
from automl_b200 import utils


def ensemble_detections_batch(params, detections, num_models, image_scales=None, mirrored_mask=0):
  """(clusters [N, num_models * rows, 7], counts [N]) for detections [num_models * N, rows, 7];
  models whose bit is set in mirrored_mask are un-mirrored first about image_scales [N] * the
  network input width, as tf2/postprocess.py:560-573 does it."""
  det = torch.as_tensor(detections, dtype=torch.float32)
  dev = det.device if det.is_cuda else torch.device('cuda')
  det = det.to(dev).contiguous()
  if det.dim() != 3 or det.shape[2] != 7 or det.shape[0] % num_models:
    raise ValueError('detections %s must be [num_models * N, rows, 7], num_models = %d'
                     % (tuple(det.shape), num_models))
  if num_models * det.shape[1] > ops.WBF_MAX_ROWS:
    raise ValueError('num_models * rows = %d exceeds %d' % (num_models * det.shape[1], ops.WBF_MAX_ROWS))
  n = det.shape[0] // num_models
  _, width = utils.parse_image_size(params['image_size'])
  if image_scales is not None:
    image_scales = torch.as_tensor(image_scales, dtype=torch.float32).to(dev).reshape(n).contiguous()
  clusters = torch.empty(n, num_models * det.shape[1], 7, dtype=torch.float32, device=dev)
  counts = torch.empty(n, dtype=torch.int32, device=dev)
  with torch.cuda.device(dev):
    ops.wbf(det, num_models, params['num_classes'], clusters, counts, mirrored_mask, image_scales,
            width)
  return clusters, counts


def ensemble_detections(params, detections, num_models):
  """wbf.py:70-95: the clusters of one image's rows [R, 7], float32 [k, 7] on the device.  Rows of
  a class outside [0, num_classes) (here: appended to make R a multiple of num_models) are never
  fused.  With no row of a fused class the result is [0, 7] (the reference's tf.stack raises).
  Unlike the reference, R is limited: R rounded up to a multiple of num_models may be at most
  ops.WBF_MAX_ROWS = 1024 (two models at the largest max_output_size of any registered config
  need 200); more raises ValueError."""
  det = torch.as_tensor(detections, dtype=torch.float32)
  if det.dim() != 2 or det.shape[1] != 7:
    raise ValueError('detections %s must be [R, 7]' % (tuple(det.shape),))
  pad = -det.shape[0] % num_models
  if pad:
    filler = torch.zeros(pad, 7, dtype=torch.float32, device=det.device)
    filler[:, 6] = -1
    det = torch.cat([det, filler])
  rows = max(det.shape[0] // num_models, 1)
  if det.shape[0] == 0:
    det = torch.zeros(num_models, 7, dtype=torch.float32)
    det[:, 6] = -1
  clusters, counts = ensemble_detections_batch(params, det.reshape(num_models, rows, 7), num_models)
  return clusters[0, :int(counts[0].item())]
