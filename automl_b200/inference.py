"""`ServingDriver` on the H100 path: same call surface as the reference's
/root/reference/efficientdet/inference.py:340-554.

  driver = inference.ServingDriver('efficientdet-d0', ckpt_path, batch_size=len(imgs))
  driver.build()
  predictions = driver.serve_images(imgs)        # float32 [N, max_output_size, 7]
                                                 # rows [image_id, ymin, xmin, ymax, xmax, score, class]

Mirrored behaviour: constructor arguments and defaults (:389-427), `params` = registry config +
`model_params` + `is_training_bn=False`, lazy `build()` on first serve (:493-494, :549-550),
`build(params_override)` returning the {'image_files','image_arrays','prediction'} dict
(:440-474), `serve_files` (decodes with PIL instead of tf.io.decode_image), `serve_images`,
`benchmark` (1 warm run + 10 timed runs, prints the same two lines, :500-524).  Out of scope and
raising NotImplementedError: `visualize`, `load`, `freeze`, `export` (SavedModel / TFLite /
TensorRT — SURVEY.md section 2 row 8).

`ckpt_path`: '_' (the reference's "don't load a checkpoint" sentinel, inference.py:218-220)
gives seeded synthetic weights; a path to an .npz whose keys are the reference variable names
(Keras layouts, see weights.py) loads real weights.

The whole request runs on the device.  Every request kind is checked and staged the same way
(staging.py): the uint8 images, behind the request's int32 tables, in one H2D copy from a pinned
buffer of the request's slot, MAX_IN_FLIGHT slots per engine.  Then edet_preprocess (images of one
size) or edet_preprocess_ragged (sizes differ; one launch either way) -> network -> pre-NMS -> NMS
-> D2H copy of the [N, max_output_size, 7] detections.  With 'segmentation' in the config's heads,
segment_images / segment_stream run the same staging and pre-process, the network without NMS,
then edet_seg_masks -> one D2H copy of a uint8 mask per image at the image's own size.
serve_images_with_masks / serve_stream_with_masks (both heads) return the detections and the masks
of the same images from one pipelined pass: edet_seg_masks runs on the engine's head stream right
after the step's head stage, and the masks are copied to the host behind the detections.
serve_images_tta / serve_stream_tta (flip test-time augmentation) pre-process each image and its
mirror in one launch (edet_preprocess_mirrored), run the network on the 2N batch, per-class NMS
(edet_per_class_nms) over all 2N, then weighted box fusion (edet_wbf) -> one D2H copy of the
clusters.
"""
import copy
import io
import time

import numpy as np
import torch

from automl_b200 import hparams_config
from automl_b200 import ops
from automl_b200 import parallel
from automl_b200 import staging
from automl_b200 import weights as weights_lib
from automl_b200.arch import DetArch
from automl_b200.engine import Engine


EMA_SUFFIX = '/ExponentialMovingAverage'


def resolve_checkpoint_names(ckpt_keys, wanted, ema_decay=0.9998):
  """Maps model variable names to the keys of a checkpoint dump, the way the reference restores
  (inference.restore_ckpt inference.py:193-230, tf2/util_keras.restore_ckpt util_keras.py:108-203):
  with ema_decay > 0 every variable is read from its shadow `<name>/ExponentialMovingAverage` when
  the checkpoint has one (trainable variables and the BN moving statistics all get shadows,
  utils.get_ema_vars utils.py:78-87), else from `<name>`; a trailing ':0' on checkpoint keys is
  ignored.  Returns {wanted name: checkpoint key}; missing variables are simply absent."""
  norm = {}
  for k in ckpt_keys:
    norm.setdefault(k[:-2] if k.endswith(':0') else k, k)
  out = {}
  for name in wanted:
    if ema_decay and ema_decay > 0 and name + EMA_SUFFIX in norm:
      out[name] = norm[name + EMA_SUFFIX]
    elif name in norm:
      out[name] = norm[name]
  return out


def load_weights(ckpt_path, arch, seed=0, ema_decay=0.9998):
  """'_' / None: seeded synthetic weights (the reference's "don't load a checkpoint" sentinel).
  Otherwise an .npz whose keys are the reference's checkpoint variable names (Keras layouts):
  either written directly, or dumped from a TF checkpoint with
  scripts/export_tf_checkpoint_to_npz.py; EMA shadow variables are preferred like in the
  reference (resolve_checkpoint_names)."""
  if ckpt_path == '_' or ckpt_path is None:
    return weights_lib.synthetic_weights(arch, seed)
  data = np.load(ckpt_path)
  specs = weights_lib.variable_specs(arch)
  names = resolve_checkpoint_names(list(data.keys()), specs, ema_decay)
  missing = [k for k in specs if k not in names]
  if missing:
    raise ValueError('checkpoint %s lacks %d variables, e.g. %s' % (ckpt_path, len(missing), missing[:3]))
  out = {}
  for k, spec in specs.items():
    v = np.asarray(data[names[k]], np.float32)
    if tuple(v.shape) != tuple(spec.shape):
      raise ValueError('variable %s has shape %s, expected %s' % (k, v.shape, spec.shape))
    out[k] = v
  return out


def image_preprocess(image, image_size, mean_rgb, stddev_rgb, device='cuda:0'):
  """inference.py:37-56 for one uint8 HxWx3 image: (float32 [H,W,3] device tensor, scale)."""
  from automl_b200 import utils
  oh, ow = utils.parse_image_size(image_size)
  raw = torch.as_tensor(np.ascontiguousarray(image), dtype=torch.uint8).to(device)[None]
  out = torch.empty(1, oh, ow, 3, dtype=torch.float32, device=device)
  scale = ops.preprocess(raw, out, _rgb3(mean_rgb), _rgb3(stddev_rgb))
  return out[0], scale


def preprocess_table(shapes, image_size):
  """The table of a ragged pre-process (ops.preprocess_ragged) for images of sizes `shapes`
  [(h, w), ...], packed in this order, each at a 16-byte aligned offset: (int32 [N, 6]
  edet_preprocess_image rows, packed byte count, float32 [N] image_scale_to_original).

  Scale-to-fit in float32 as edet_preprocess computes it (dataloader.py:115-127, inference.py:68-109
  runs image_preprocess per image): s = min(H / h, W / w), scaled = int(h * s), w likewise, and
  1 / s.  Raises ValueError for an empty image or one whose scaled size is 0."""
  from automl_b200 import utils
  oh, ow = utils.parse_image_size(image_size)
  hw = np.asarray(shapes, np.int64).reshape(-1, 2)
  if len(hw) == 0 or (hw < 1).any():
    raise ValueError('empty image or request: sizes %s' % hw.tolist())
  h, w = hw[:, 0].astype(np.float32), hw[:, 1].astype(np.float32)
  sy, sx = np.float32(oh) / h, np.float32(ow) / w
  scale = np.where(sx < sy, sx, sy)
  scaled_h, scaled_w = (h * scale).astype(np.int64), (w * scale).astype(np.int64)
  bad = np.flatnonzero((scaled_h < 1) | (scaled_w < 1))
  if len(bad):
    i = bad[0]
    raise ValueError('a %dx%d image collapses to %dx%d at %dx%d'
                     % (hw[i, 0], hw[i, 1], scaled_h[i], scaled_w[i], oh, ow))
  nbytes = 3 * hw[:, 0] * hw[:, 1]
  offsets = np.zeros(len(hw), np.int64)
  offsets[1:] = np.cumsum((nbytes[:-1] + 15) // 16 * 16)
  desc = np.zeros((len(hw), ops.PRE_DESC_WORDS), np.int32)
  desc[:, :2] = offsets.view(np.int32).reshape(-1, 2)
  desc[:, 2:] = np.stack([hw[:, 0], hw[:, 1], scaled_h, scaled_w], axis=1)
  return desc, int(offsets[-1] + nbytes[-1]), np.float32(1.0) / scale


def seg_mask_table(shapes, image_size):
  """The table of ops.seg_masks for images of sizes `shapes` [(h, w), ...] pre-processed to
  `image_size`: (int32 [N, 6] edet_seg_mask_image rows, packed byte count).  Mask i is the h x w
  uint8 block at byte offset sum_{j<i} h_j * w_j; scaled_h, scaled_w are the image's size in the
  letterboxed input, as preprocess_table computes it.  Raises ValueError like preprocess_table."""
  desc, _, _ = preprocess_table(shapes, image_size)
  hw = desc[:, 2:4].astype(np.int64)
  nbytes = hw[:, 0] * hw[:, 1]
  offsets = np.zeros(len(hw), np.int64)
  offsets[1:] = np.cumsum(nbytes[:-1])
  table = np.zeros((len(hw), ops.SEG_MASK_WORDS), np.int32)
  table[:, :2] = offsets.view(np.int32).reshape(-1, 2)
  table[:, 2:] = desc[:, 2:]
  return table, int(offsets[-1] + nbytes[-1])


def _mask_classes(num_classes):
  """`num_classes` if uint8 masks hold that many classes, else ValueError."""
  if not 1 <= num_classes <= ops.SEG_MAX_CLASSES:
    raise ValueError('seg_num_classes = %d: uint8 masks hold 1..%d classes'
                     % (num_classes, ops.SEG_MAX_CLASSES))
  return int(num_classes)


def segment_request(image_arrays, image_size, num_classes):
  """The host checks submit_segment runs on one request before anything is enqueued, without a
  GPU: (shapes [(h, w), ...], mask table, packed byte count).  Raises ValueError as
  staging.decoded_images and seg_mask_table do, and for more than 256 classes (uint8 masks)."""
  _mask_classes(num_classes)
  shapes = staging.decoded_images(image_arrays).shapes
  return (shapes,) + seg_mask_table(shapes, image_size)


def _unpack_masks(packed, shapes):
  """The uint8 [h, w] numpy masks of images of sizes `shapes` [(h, w), ...] from the pinned buffer
  `packed`, where they lie back to back as seg_mask_table lays them out."""
  offsets = np.cumsum([0] + [h * w for h, w in shapes])
  host = packed[:offsets[-1]].numpy().copy()
  return [host[o:o + h * w].reshape(h, w) for o, (h, w) in zip(offsets, shapes)]


def _rgb3(v):
  if isinstance(v, (int, float)):
    return [float(v)] * 3
  return [float(x) for x in v]


class _Request(object):
  """Handle of one in-flight request (ServingDriver.submit, submit_segment, submit_tta,
  submit_with_masks): `result()` blocks until the request's results are in its slot's pinned memory
  and returns `collect(slot)`."""

  def __init__(self, slot, collect):
    self._slot, self._collect = slot, collect
    self._out = None
    slot.pending = self

  def done(self):
    return self._out is not None or self._slot.ev_done.query()

  def result(self):
    if self._out is None:
      self._slot.ev_done.synchronize()
      self._out = self._collect(self._slot)
      if self._slot.pending is self:
        self._slot.pending = None
    return self._out


class _TTABuffers(object):
  """The device buffers of a flip TTA request of n images on an engine of 2n: the per-class NMS rows
  of both views `rows` [2n, max_output_size, 7] with that NMS's `keep`, `valid` and `work` buffers,
  the image ids and scales of both views, and the fused clusters [n, cap, 7] followed by their int32
  counts [n] in `fused` (pinned twin `fused_host`)."""

  def __init__(self, eng, image_id_base, device):
    n, max_out = eng.n // 2, eng.max_output_size
    self.cap = 2 * max_out
    k = eng.total_anchors if not eng.max_nms_inputs else eng.max_nms_inputs
    ids = np.float32(image_id_base) + np.arange(n, dtype=np.float32)
    size = n * self.cap * 7 + n
    self.rows = torch.empty(2 * n, max_out, 7, device=device)
    self.keep = torch.empty(2 * n, max_out, dtype=torch.int32, device=device)
    self.valid = torch.empty(2 * n, dtype=torch.int32, device=device)
    self.work = torch.empty(2 * n, k, device=device)
    self.ids = torch.from_numpy(np.concatenate([ids, ids])).to(device)
    self.scales = torch.empty(2 * n, device=device)
    self.fused = torch.empty(size, device=device)
    self.fused_host = torch.empty(size).pin_memory()


class _Slot(object):
  """One of an engine's MAX_IN_FLIGHT request slots: the request's staging and image scales, its
  result buffers and the events that order their reuse.  Under batch_size=None, a slot of engine
  size 2n serves both detection requests of 2n images and TTA requests of n images, so each kind
  of request keeps result buffers of its own; mask and TTA buffers are allocated on first use."""

  def __init__(self, eng, world, device):
    self.staging = staging.StagingSlot(device)
    self.scales = torch.empty(eng.n, dtype=torch.float32).pin_memory()
    self.host_det = torch.empty(world * eng.n, eng.max_output_size, 7).pin_memory()
    self.gathered = (torch.empty(world * eng.n, eng.max_output_size, 7, device=device)
                     if world > 1 else None)
    self.masks_dev = self.masks_host = None    # segmentation: the packed uint8 masks
    self.tta = None                            # flip TTA: _TTABuffers
    # before the D2H stream's copy: after the request's last kernel (masks, TTA), or after the
    # detection copy of a request with masks
    self.ev_out = torch.cuda.Event()
    self.ev_done = torch.cuda.Event()          # its results are in pinned memory
    self.pending = None                        # its handle, until the results are collected


class ServingDriver(object):
  """A driver for serving single or batch images (reference inference.py:340)."""

  MAX_IN_FLIGHT = 3   # submit(): requests whose results have not been collected yet

  def __init__(self, model_name, ckpt_path, batch_size=1, use_xla=False, min_score_thresh=None,
               max_boxes_to_draw=None, line_thickness=None, model_params=None, device='cuda:0',
               image_id_base=0):
    self.model_name = model_name
    self.ckpt_path = ckpt_path
    self.batch_size = batch_size
    self.params = hparams_config.get_detection_config(model_name).as_dict()
    if model_params:
      self.params.update(model_params)
    self.params.update(dict(is_training_bn=False))
    self.label_map = self.params.get('label_map', None)
    self.signitures = None   # (sic) the reference's spelling
    self.engine = None
    self.use_xla = use_xla    # accepted for signature compatibility; there is no XLA here
    self.min_score_thresh = min_score_thresh
    self.max_boxes_to_draw = max_boxes_to_draw
    self.line_thickness = line_thickness
    self.device = device
    self.image_id_base = image_id_base
    self._engines = None

  # ---- build ---------------------------------------------------------------------------------
  def build(self, params_override=None):
    """Builds the engine (weights, buffers, launch list) and returns the signature dict.

    batch_size=None (the reference's dynamic batch, inference.py:68-109, where `map_fn` runs the
    per-image pre-process over however many images arrive): the weights are loaded here and one
    engine per distinct batch size is built on first use and kept."""
    params = copy.deepcopy(self.params)
    if params_override:
      params.update(params_override)
    config = hparams_config.Config(params)
    arch = DetArch(config)
    self._weights = load_weights(self.ckpt_path, arch)
    self.config = config
    self.mean_rgb = _rgb3(params['mean_rgb'])
    self.stddev_rgb = _rgb3(params['stddev_rgb'])
    self._engines = {}
    self._slots = {}
    self._copy_stream = torch.cuda.Stream(device=self.device)
    self._d2h_stream = torch.cuda.Stream(device=self.device)   # mask and TTA results to the host
    self._seq = 0
    self.engine = self._engine_for(self.batch_size) if self.batch_size else None
    self.signitures = {
        'image_files': 'image_files',     # bytes of encoded images (serve_files)
        'image_arrays': 'image_arrays',   # uint8 HxWx3 arrays (serve_images)
        'prediction': (self.engine.detections if self.engine is not None and
                       self.engine.arch.has_detection else 'detections'),
    }
    return self.signitures

  def _engine_for(self, n):
    eng = self._engines.get(n)
    if eng is None:
      eng = self._engines[n] = Engine(self.config, self._weights, n, device=self.device,
                                      image_id_base=self.image_id_base)
      world = 1
      if torch.distributed.is_available() and torch.distributed.is_initialized():
        world = torch.distributed.get_world_size()
      self._slots[n] = [_Slot(eng, world, self.device) for _ in range(self.MAX_IN_FLIGHT)]
    return eng

  # ---- serving -------------------------------------------------------------------------------
  def _acquire(self, image_arrays, views=1):
    """Checks one request (staging.decoded_images, against batch_size) and takes the next slot of
    the engine of `views` x N images, building the driver on first use: (the decoded request, the
    engine, the slot).  The slot's previous request is completed first, as its buffers are about to
    be reused.  Nothing is enqueued.  A request that is already a staging.Decoded is not checked
    again."""
    request = image_arrays
    if not isinstance(request, staging.Decoded):
      request = staging.decoded_images(image_arrays, self.batch_size or None, self.device)
    if self._engines is None:
      self.build()
    n = views * len(request.shapes)
    eng = self._engine_for(n)
    slot = self._slots[n][self._seq % self.MAX_IN_FLIGHT]
    self._seq += 1
    if slot.pending is not None:
      slot.pending.result()
    return request, eng, slot

  def _stage(self, eng, slot, request, table=None, mirrored=False):
    """Stages a decoded request in the slot (one H2D on the copy stream) and enqueues its
    pre-process into the engine input on the current stream:
      * images of one size: edet_preprocess of the image region viewed [N, h, w, 3];
      * images of different sizes: edet_preprocess_ragged over the preprocess_table rows;
      * mirrored (the engine holds 2N images), either kind: edet_preprocess_mirrored into input[:N]
        and, flipped on width, input[N:]; images of one size take a table of equal rows.
    Every image's scale goes to the engine, for both halves of a mirrored request.  An image that
    collapses to zero size raises ValueError from preprocess_table before anything is enqueued; a
    request of one size that is not mirrored takes no table, and edet_preprocess refuses it.

    table: None, or an int32 [N, k] table that travels with the images for a later kernel.  Returns
    its device view, and the caller releases the slot's staging after that kernel; without a table
    the staging is released after the pre-process."""
    n = len(request.shapes)
    h, w = request.shapes[0]
    offsets = np.arange(n, dtype=np.int64) * (h * w * 3)   # one size: an [N, h, w, 3] batch
    tables = [] if table is None else [table]
    if mirrored or not request.uniform:
      desc, _, scales = preprocess_table(request.shapes, tuple(eng.input.shape[1:3]))
      if request.uniform:
        desc[:, :2] = offsets.view(np.int32).reshape(-1, 2)
      offsets = desc[:, :2].copy().view(np.int64)[:, 0]
      tables.insert(0, desc)
    views, images = slot.staging.stage(self._copy_stream, tables, request, offsets)
    if mirrored:
      ops.preprocess_mirrored(images, views[0], eng.input, self.mean_rgb, self.stddev_rgb)
      slot.scales.numpy()[:] = np.concatenate([scales, scales])
    elif request.uniform:
      slot.scales.fill_(ops.preprocess(images.view(n, h, w, 3), eng.input, self.mean_rgb,
                                       self.stddev_rgb))
    else:
      ops.preprocess_ragged(images, views[0], eng.input, self.mean_rgb, self.stddev_rgb)
      slot.scales.numpy()[:] = scales
    if table is None:
      slot.staging.release()
    eng.image_scales.copy_(slot.scales, non_blocking=True)
    return views[-1] if table is not None else None

  def _download(self, slot, dev, host):
    """After the request's last kernel on the current stream: `dev` to the pinned `host` on the
    D2H stream, which records the slot's ev_done."""
    slot.ev_out.record(torch.cuda.current_stream())
    with torch.cuda.stream(self._d2h_stream):
      self._d2h_stream.wait_event(slot.ev_out)
      host.copy_(dev, non_blocking=True)
      slot.ev_done.record(self._d2h_stream)

  def submit(self, image_arrays):
    """Enqueues one request and returns a handle; `handle.result()` blocks until its detections
    are in host memory.  Up to MAX_IN_FLIGHT (3) requests are in flight: the H2D copy and
    pre-process of request i+1, the backbone of request i, the feature network / heads of request
    i-1 and the NMS + D2H copy of request i-1 / i-2 overlap (copy stream, main stream, the engine's
    head and NMS streams).  Submitting one more request first completes the oldest one.

    image_arrays: a list of uint8 [h, w, 3] images (sizes may differ), a uint8 [N, h, w, 3] numpy
    array or tensor, pinned or not, or such a tensor on the driver's device, which is read in place
    on the current stream.  Anything else raises ValueError before anything is enqueued."""
    with torch.cuda.device(self.device):
      request, eng, slot = self._acquire(image_arrays)
      self._stage(eng, slot, request)

      def after_nms(det, slot=slot):
        """On the engine's NMS stream right after NMS: all-gather (multi-GPU) + D2H copy."""
        det = parallel.gather_detections(det, slot.gathered)
        slot.host_det.copy_(det, non_blocking=True)
        slot.ev_done.record(torch.cuda.current_stream())
      eng.run(postprocess=True, after_nms=after_nms)
    # float32 [N (x world), max_output_size, 7]: [image_id, ymin, xmin, ymax, xmax, score, class]
    return _Request(slot, lambda s: s.host_det.numpy().copy())

  def serve_images(self, image_arrays):
    """image_arrays: list (or array) of HxWx3 uint8 images -> float32 [N, max_output_size, 7].

    Under torch.distributed (one process per GPU, batch sharded over the ranks) the per-rank
    detection blocks are all-gathered on the device first, so every rank returns the global
    [world * N, max_output_size, 7] result (the single collective of the path)."""
    return self.submit(image_arrays).result()

  def serve_stream(self, batches):
    """Generator over an iterable of requests: yields the detections of each, in order, keeping
    MAX_IN_FLIGHT requests in flight."""
    return staging.pipelined(self.submit, batches, self.MAX_IN_FLIGHT)

  # ---- segmentation --------------------------------------------------------------------------
  def _check_masks(self, resize):
    """The refusals every mask request shares, raised before anything is built or enqueued."""
    if resize != 'nearest':
      raise NotImplementedError('mask resize %r: only nearest sampling is built' % (resize,))
    if torch.distributed.is_available() and torch.distributed.is_initialized():
      raise NotImplementedError('segmentation masks under torch.distributed are not built')

  def _stage_masks(self, eng, slot, request):
    """Stages a mask request in the slot with its mask table riding in the same H2D copy (_stage)
    and grows the slot's mask buffers to its packed masks: (device view of the table, packed byte
    count).  The slot's previous request has completed (_acquire), so neither buffer is in use."""
    table, total = seg_mask_table(request.shapes, tuple(eng.input.shape[1:3]))
    dev_table = self._stage(eng, slot, request, table=table)
    slot.masks_dev = staging.grow(slot.masks_dev, total, device=self.device)
    slot.masks_host = staging.grow(slot.masks_host, total, pin_memory=True)
    return dev_table, total

  def _launch_masks(self, eng, slot, request, num_classes, dev_table):
    """edet_seg_masks from the engine's segmentation logits into the slot's mask buffer, on the
    current stream, which then releases the slot's staging: the kernel has read the table."""
    hs, ws = eng.seg_out.shape[1:3]
    f = 2 ** (self.config.min_level - 1)
    assert (hs * f, ws * f) == tuple(eng.input.shape[1:3]), 'logits grid is not input / f'
    ops.seg_masks(eng.seg_out, num_classes, f, dev_table,
                  tuple(int(v) for v in np.max(request.shapes, axis=0)), slot.masks_dev)
    slot.staging.release()

  def submit_segment(self, image_arrays, resize='nearest'):
    """Enqueues one segmentation request and returns a handle; `handle.result()` blocks until the
    masks are in host memory: a list of uint8 [h_i, w_i] numpy arrays, the class of every pixel of
    each image at its own size.  Needs a config whose `heads` include 'segmentation' and at most 256
    classes (uint8 masks).

    The images are staged and pre-processed as in submit() (the mask table rides in the same H2D
    copy), the network runs without the NMS stage, then one edet_seg_masks launch samples the
    segmentation logits at the nearest cell of each image's region of the letterboxed input and
    takes the arg-max over the classes (first class on ties, like tf.argmax in the reference's
    segmentation demo).  The packed masks reach pinned host memory in one D2H copy on a stream of
    their own, so up to MAX_IN_FLIGHT requests overlap like detection requests do."""
    self._check_masks(resize)
    heads = self.params.get('heads') or []
    if 'segmentation' not in heads:
      raise ValueError("segmentation masks need 'segmentation' in heads; heads = %s" % (heads,))
    with torch.cuda.device(self.device):
      request, eng, slot = self._acquire(image_arrays)
      num_classes = _mask_classes(self.config.seg_num_classes)
      dev_table, total = self._stage_masks(eng, slot, request)
      eng.run(postprocess=False)
      self._launch_masks(eng, slot, request, num_classes, dev_table)
      self._download(slot, slot.masks_dev[:total], slot.masks_host[:total])
    shapes = request.shapes
    return _Request(slot, lambda s: _unpack_masks(s.masks_host, shapes))

  def segment_images(self, image_arrays, resize='nearest'):
    """image_arrays: list of HxWx3 uint8 images (sizes may differ) or a uint8 [N, h, w, 3] tensor
    -> list of uint8 [h_i, w_i] numpy masks, one per image (see submit_segment)."""
    return self.submit_segment(image_arrays, resize).result()

  def segment_stream(self, batches, resize='nearest'):
    """Generator over an iterable of requests: yields the masks of each, in order, keeping
    MAX_IN_FLIGHT requests in flight."""
    return staging.pipelined(lambda b: self.submit_segment(b, resize), batches, self.MAX_IN_FLIGHT)

  # ---- detections and masks from one pass ------------------------------------------------------
  def submit_with_masks(self, image_arrays, resize='nearest'):
    """Enqueues one request for detections and segmentation masks of the same images and returns a
    handle; `handle.result()` blocks until both are in host memory and returns (detections, masks):
    what submit() and submit_segment() return for the request, from one network pass.  Needs a
    config whose `heads` hold both 'object_detection' and 'segmentation', and at most 256 classes.

    The request is staged as in submit_segment() and runs the pipelined step of submit(): the
    step's head stage computes the segmentation logits with the class and box outputs, and the
    edet_seg_masks launch follows it on the engine's head stream (Engine.run's after_heads), so the
    backbone of the next request still overlaps this one's heads.  The detections are copied to
    pinned memory on the NMS stream, the masks behind them on the D2H stream.  Combined requests
    share the slots of every other request kind.  The checks of submit() and submit_segment() are
    raised before anything is built or enqueued."""
    self._check_masks(resize)
    heads = self.params.get('heads') or []
    if 'object_detection' not in heads or 'segmentation' not in heads:
      raise ValueError("detections with masks need 'object_detection' and 'segmentation' in heads; "
                       "heads = %s" % (heads,))
    num_classes = _mask_classes(self.config.seg_num_classes if self._engines is not None
                                else self.params['seg_num_classes'])
    request = staging.decoded_images(image_arrays, self.batch_size or None, self.device)
    with torch.cuda.device(self.device):
      request, eng, slot = self._acquire(request)
      dev_table, total = self._stage_masks(eng, slot, request)

      def after_heads(seg_out, slot=slot):
        """On the engine's head stream, before the next request's head stage rewrites seg_out: the
        masks, and the staging release after the one kernel that reads the table."""
        self._launch_masks(eng, slot, request, num_classes, dev_table)

      def after_nms(det, slot=slot):
        """On the engine's NMS stream, which waits for the head stage and after_heads: the
        detections, then the masks on the D2H stream behind that copy (_download records ev_out
        here), so the slot's ev_done follows both copies."""
        slot.host_det.copy_(det, non_blocking=True)
        self._download(slot, slot.masks_dev[:total], slot.masks_host[:total])
      eng.run(postprocess=True, after_nms=after_nms, after_heads=after_heads)
    shapes = request.shapes
    return _Request(slot, lambda s: (s.host_det.numpy().copy(), _unpack_masks(s.masks_host, shapes)))

  def serve_images_with_masks(self, image_arrays):
    """image_arrays: list of HxWx3 uint8 images (sizes may differ) or a uint8 [N, h, w, 3] tensor
    -> (float32 [N, max_output_size, 7] detections, list of uint8 [h_i, w_i] masks), see
    submit_with_masks."""
    return self.submit_with_masks(image_arrays).result()

  def serve_stream_with_masks(self, batches):
    """Generator over an iterable of requests: yields (detections, masks) of each, in order,
    keeping MAX_IN_FLIGHT requests in flight."""
    return staging.pipelined(self.submit_with_masks, batches, self.MAX_IN_FLIGHT)

  # ---- flip test-time augmentation --------------------------------------------------------------
  def submit_tta(self, image_arrays):
    """Enqueues one horizontal-flip test-time-augmented request and returns a handle;
    `handle.result()` blocks until the fused detections are in host memory: a list of float32
    [k_i, 7] numpy arrays [image_id, x1, y1, x2, y2, score, class], sorted by score -- the layout
    of nms_np / postprocess.generate_detections, not serve_images' [id, y, x, y, x, ...].

    The reference's recipe (tf2/postprocess.py:530-586 with flip=True, tf2/wbf.py:70-95), all on
    the device: the images are staged as in submit() and edet_preprocess_mirrored writes each
    letterboxed input and its left-right mirror into the engine of 2N images; the network runs
    without the NMS stage; pre-NMS and one edet_per_class_nms over all 2N images (nms_configs,
    image id image_id_base + i and the image's scale for both halves) give nms_np's rows; one
    edet_wbf launch un-mirrors the second half about image_scale * width and fuses the two models
    per image.  Only the nms_np branch (nms_configs.pyfunc) is built, as for generate_detections;
    the TF per-class NMS branch is not.  WBF fuses classes 0 .. num_classes-1 of nms_np's 1-based
    rows, as the reference does: the last class is dropped and the dummy rows form one class-0
    cluster at score -1e5.  The clusters reach pinned host memory in one D2H copy on a stream of
    their own, so up to MAX_IN_FLIGHT requests overlap."""
    if torch.distributed.is_available() and torch.distributed.is_initialized():
      raise NotImplementedError('test-time augmentation under torch.distributed is not built')
    heads = self.params.get('heads')
    heads = ['object_detection'] if heads is None else list(heads)
    if 'object_detection' not in heads:
      raise ValueError("test-time augmentation needs 'object_detection' in heads; heads = %s"
                       % (heads,))
    with torch.cuda.device(self.device):
      request, eng, slot = self._acquire(image_arrays, views=2)
      n = len(request.shapes)
      self._stage(eng, slot, request, mirrored=True)
      if slot.tta is None:
        slot.tta = _TTABuffers(eng, self.image_id_base, self.device)
      t = slot.tta
      nms = self.config.as_dict()['nms_configs']
      max_out, cap = eng.max_output_size, t.cap
      t.scales.copy_(slot.scales, non_blocking=True)
      eng.run(postprocess=False)
      ps = eng.pre_nms_only()
      ops.per_class_nms(ps['boxes'], ps['scores'], ps['classes'], t.ids, t.scales,
                        self.config.num_classes, max_out, nms['method'], nms.get('iou_thresh'),
                        t.rows, t.keep, t.valid, sigma=nms.get('sigma'),
                        score_thresh=nms.get('score_thresh'), work=t.work)
      ops.wbf(t.rows, 2, self.config.num_classes, t.fused[:n * cap * 7].view(n, cap, 7),
              t.fused[n * cap * 7:].view(torch.int32), mirrored_mask=0b10,
              image_scales=t.scales[:n], width=eng.input.shape[2])
      self._download(slot, t.fused, t.fused_host)

    def fused(s):
      host = s.tta.fused_host.numpy()
      clusters = host[:n * cap * 7].reshape(n, cap, 7)
      counts = host[n * cap * 7:].view(np.int32)
      return [clusters[i, :counts[i]].copy() for i in range(n)]
    return _Request(slot, fused)

  def serve_images_tta(self, image_arrays):
    """image_arrays: list of HxWx3 uint8 images (sizes may differ) or a uint8 [N, h, w, 3] tensor
    -> list of float32 [k_i, 7] numpy arrays of fused detections, one per image (see submit_tta)."""
    return self.submit_tta(image_arrays).result()

  def serve_stream_tta(self, batches):
    """Generator over an iterable of requests: yields the fused detections of each, in order,
    keeping MAX_IN_FLIGHT requests in flight."""
    return staging.pipelined(self.submit_tta, batches, self.MAX_IN_FLIGHT)

  def serve_files(self, image_files):
    """image_files: list of encoded image bytes (jpeg/png)."""
    from PIL import Image  # pylint: disable=g-import-not-at-top
    arrays = [np.asarray(Image.open(io.BytesIO(b)).convert('RGB')) for b in image_files]
    return self.serve_images(arrays)

  def benchmark(self, image_arrays, trace_filename=None):
    """1 warm-up run then the mean of 10 runs, printed like the reference (:500-524)."""
    if self._engines is None:
      self.build()
    self.serve_images(image_arrays)
    start = time.perf_counter()
    for _ in range(10):
      self.serve_images(image_arrays)
    end = time.perf_counter()
    inference_time = (end - start) / 10
    print('Per batch inference time: ', inference_time)
    print('FPS: ', len(image_arrays) / inference_time)
    if trace_filename:
      raise NotImplementedError('chrome traces are replaced by ncu / CUDA events (see bench.py)')
    return inference_time

  # ---- out of scope ----------------------------------------------------------------------------
  def visualize(self, image, prediction, **kwargs):
    raise NotImplementedError('visualisation is out of scope (SURVEY.md section 2 row 18)')

  def load(self, saved_model_dir_or_frozen_graph):
    raise NotImplementedError('SavedModel / frozen-graph loading is out of scope')

  def freeze(self):
    raise NotImplementedError('graph freezing is out of scope')

  def export(self, *args, **kwargs):
    raise NotImplementedError('SavedModel / TFLite / TensorRT export is out of scope')
