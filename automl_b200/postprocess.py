"""Post-processing call surface of the reference's tf2/postprocess.py on the H100 path.

  generate_detections(params, engine, image_scales, image_ids, flip=False)
      /root/reference/efficientdet/tf2/postprocess.py:530-575, the `nms_configs.pyfunc` branch:
      pre_nms (postprocess.py:119-156) followed, per image, by nms_np.per_class_nms
      (nms_np.py:220-264) -- here ONE CUDA launch for the whole batch (edet_per_class_nms).
      Returns float32 [N, max_output_size, 7] rows [image_id, xmin, ymin, xmax, ymax, score,
      class] (the layout of nms_np, NOT the [id, y, x, y, x, ...] layout of det_post_process).
  transform_detections(detections)   postprocess.py:589-601 -> [id, x, y, w, h, score, class]

All four methods of nms_np run on the device (`hard`, `diou`: rows bit-identical to NumPy;
`linear`: bit-identical; `gaussian`: identical selections, scores within a few float32 ulp because
NumPy's SIMD exp is not correctly rounded).  The default serving path (NMS-V5) is Engine.detect().
"""
import torch

from automl_b200 import ops
from automl_b200 import utils


def per_class_nms(boxes, scores, classes, image_ids, image_scales, num_classes, max_boxes_to_draw,
                  nms_configs):
  """Batched nms_np.per_class_nms on device tensors; returns (detections, keep_index, num_valid)."""
  method = nms_configs['method']
  n = scores.shape[0]
  dev = scores.device
  det = torch.empty(n, max_boxes_to_draw, 7, dtype=torch.float32, device=dev)
  keep = torch.empty(n, max_boxes_to_draw, dtype=torch.int32, device=dev)
  valid = torch.empty(n, dtype=torch.int32, device=dev)
  as_f32 = lambda v: None if v is None else torch.as_tensor(v, dtype=torch.float32).to(dev).contiguous()
  ops.per_class_nms(boxes, scores, classes, as_f32(image_ids), as_f32(image_scales), num_classes,
                    max_boxes_to_draw, method, nms_configs.get('iou_thresh'), det, keep, valid,
                    sigma=nms_configs.get('sigma'), score_thresh=nms_configs.get('score_thresh'))
  return det, keep, valid


def generate_detections(params, engine, image_scales, image_ids, flip=False):
  """The reference's legacy [id, x1, y1, x2, y2, score, class] interface on an Engine whose
  forward pass has run (engine.run / engine.forward): pre-NMS + per-class NMS on the device."""
  nms_configs = params['nms_configs']
  ps = engine.pre_nms_only()
  det, _, _ = per_class_nms(ps['boxes'], ps['scores'], ps['classes'], image_ids, image_scales,
                            params['num_classes'], nms_configs['max_output_size'], nms_configs)
  if flip:
    _, width = utils.parse_image_size(params['image_size'])
    ow = (torch.as_tensor(image_scales, dtype=torch.float32).to(det.device) * width)[:, None]
    det = torch.stack([det[..., 0], ow - det[..., 3], det[..., 2], ow - det[..., 1], det[..., 4],
                       det[..., 5], det[..., 6]], dim=-1)
  return det


def transform_detections(detections):
  """[id, x1, y1, x2, y2, score, class] -> [id, x, y, w, h, score, class] (postprocess.py:589)."""
  d = detections
  return torch.stack([d[..., 0], d[..., 1], d[..., 2], d[..., 3] - d[..., 1], d[..., 4] - d[..., 2],
                      d[..., 5], d[..., 6]], dim=-1)
