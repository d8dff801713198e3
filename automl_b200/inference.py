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

The whole request runs on the device: H2D copy of the uint8 images -> edet_preprocess (images of
one size) or edet_preprocess_ragged (sizes differ; one launch either way) -> network -> pre-NMS ->
NMS -> D2H copy of the [N, max_output_size, 7] detections.  With 'segmentation' in the config's
heads, segment_images / segment_stream run the same staging and pre-process, the network without
NMS, then edet_seg_masks -> one D2H copy of a uint8 mask per image at the image's own size.
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


def segment_request(image_arrays, image_size, num_classes):
  """Checks one segment_images request before anything is enqueued: (shapes [(h, w), ...], mask
  table, packed byte count).  Raises ValueError for an empty request, an image that is not uint8
  [h, w, 3] or collapses to zero size, and for more than 256 classes (uint8 masks)."""
  if not 1 <= num_classes <= ops.SEG_MAX_CLASSES:
    raise ValueError('seg_num_classes = %d: uint8 masks hold 1..%d classes'
                     % (num_classes, ops.SEG_MAX_CLASSES))
  if isinstance(image_arrays, torch.Tensor):
    if image_arrays.dtype != torch.uint8 or image_arrays.dim() != 4 or image_arrays.shape[3] != 3:
      raise ValueError('expected a uint8 [N, h, w, 3] tensor, got %s %s'
                       % (image_arrays.dtype, tuple(image_arrays.shape)))
    shapes = [tuple(image_arrays.shape[1:3])] * image_arrays.shape[0]
  else:
    shapes = []
    for im in image_arrays:
      im = np.asarray(im)
      if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
        raise ValueError('expected uint8 [h, w, 3] images, got %s %s' % (im.dtype, im.shape))
      shapes.append(im.shape[:2])
  if not shapes:
    raise ValueError('empty request')
  table, total = seg_mask_table(shapes, image_size)
  return shapes, table, total


def _grow(buf, nbytes, **kw):
  """`buf` if it holds `nbytes`, else a new uint8 buffer of at least twice its size."""
  if buf is not None and buf.numel() >= nbytes:
    return buf
  return torch.empty(max(nbytes, 2 * buf.numel() if buf is not None else 0), dtype=torch.uint8, **kw)


def _rgb3(v):
  if isinstance(v, (int, float)):
    return [float(v)] * 3
  return [float(x) for x in v]


class _Request(object):
  """Handle of one in-flight serving request (ServingDriver.submit)."""

  def __init__(self, slot):
    self._slot = slot
    self._out = None

  def _finish(self):
    if self._out is None:
      self._slot['engine'].flush()        # a head / NMS stage the engine may still be holding back
      self._slot['ev_done'].synchronize()
      self._out = self._slot['host_det'].numpy().copy()
      if self._slot['pending'] is self:
        self._slot['pending'] = None
    return self._out

  def done(self):
    if self._out is None:
      self._slot['engine'].flush()
    return self._out is not None or self._slot['ev_done'].query()

  def result(self):
    """float32 [N (x world), max_output_size, 7] numpy array
    [image_id, ymin, xmin, ymax, xmax, score, class]."""
    return self._finish()


class _SegmentRequest(_Request):
  """Handle of one in-flight segmentation request (ServingDriver.submit_segment)."""

  def __init__(self, slot, shapes, total):
    super().__init__(slot)
    self._shapes, self._total = shapes, total

  def _finish(self):
    if self._out is None:
      self._slot['ev_done'].synchronize()
      packed = self._slot['mask_host'][:self._total].numpy().copy()
      self._out, off = [], 0
      for h, w in self._shapes:
        self._out.append(packed[off:off + h * w].reshape(h, w))
        off += h * w
      if self._slot['pending'] is self:
        self._slot['pending'] = None
    return self._out

  def done(self):
    return self._out is not None or self._slot['ev_done'].query()

  def result(self):
    """List of uint8 [h_i, w_i] numpy masks, one per image: the class of each pixel."""
    return self._finish()


class _TTARequest(_Request):
  """Handle of one in-flight test-time-augmented request (ServingDriver.submit_tta)."""

  def __init__(self, slot, n, cap):
    super().__init__(slot)
    self._n, self._cap = n, cap

  def _finish(self):
    if self._out is None:
      self._slot['ev_done'].synchronize()
      host = self._slot['tta_host'].numpy()
      size = self._n * self._cap * 7
      clusters = host[:size].reshape(self._n, self._cap, 7)
      counts = host[size:size + self._n].view(np.int32)
      self._out = [clusters[i, :counts[i]].copy() for i in range(self._n)]
      if self._slot['pending'] is self:
        self._slot['pending'] = None
    return self._out

  def done(self):
    return self._out is not None or self._slot['ev_done'].query()

  def result(self):
    """List of float32 [k_i, 7] numpy arrays, one per image: [image_id, x1, y1, x2, y2, score,
    class] rows sorted by score."""
    return self._finish()


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
    self._d2h_stream = torch.cuda.Stream(device=self.device)   # segmentation masks to the host
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
      # MAX_IN_FLIGHT requests per batch size: pinned host staging / result buffers, device raw
      # buffers and the events that order their reuse
      self._slots[n] = [{
          'engine': eng,
          'host_det': torch.empty(world * n, eng.max_output_size, 7).pin_memory(),
          'scales': torch.empty(n, dtype=torch.float32).pin_memory(),
          'gathered': (torch.empty(world * n, eng.max_output_size, 7, device=self.device)
                       if world > 1 else None),
          'raw_host': None, 'raw_dev': None, 'packed_host': None, 'packed_dev': None,
          'extra_host': None, 'extra_dev': None, 'mask_host': None, 'mask_dev': None,
          'ev_h2d': torch.cuda.Event(), 'ev_raw_free': torch.cuda.Event(),
          'ev_masks': torch.cuda.Event(), 'ev_done': torch.cuda.Event(), 'pending': None,
      } for _ in range(self.MAX_IN_FLIGHT)]
    return eng

  # ---- serving -------------------------------------------------------------------------------
  def _stage_raw(self, eng, slot, image_arrays, extra=None, mirrored=False):
    """Uploads the uint8 images (copy stream, from pinned memory) and runs the device pre-process
    into the engine input (current stream): images of one size as one [N, h, w, 3] batch, images
    of different sizes packed behind a descriptor table (preprocess_table), checked before anything
    is enqueued: an image that is not uint8 [h, w, 3] or collapses to zero size raises ValueError.

    extra: None, or an int32 [N, k] table (k even) that travels with the request -- behind the
    descriptor rows in the same H2D copy for a ragged request, in its own small copy on the copy
    stream otherwise.  Returns its 8-byte aligned device view (None without it); it stays valid
    until the slot's next request.

    mirrored: the engine holds 2N images; the N images go through edet_preprocess_mirrored into
    input[:N] and, flipped on width, input[N:] (a uniform batch through a table of equal rows, in
    place of `extra`, so a mirrored request takes none), and both halves get the images' scales."""
    if mirrored and extra is not None:
      raise ValueError('a mirrored request carries its own descriptor table, not an extra one')
    n = eng.n // 2 if mirrored else eng.n
    extra_dev = None
    main = torch.cuda.current_stream()
    if isinstance(image_arrays, torch.Tensor):   # [N,h,w,3] uint8 (e.g. pinned host memory)
      shapes = {tuple(image_arrays.shape[1:])}
    else:
      shapes = {tuple(np.shape(im)) for im in image_arrays}
    if len(shapes) == 1:
      shape = (n,) + next(iter(shapes))
      if isinstance(image_arrays, torch.Tensor) and image_arrays.dtype == torch.uint8 and \
          (image_arrays.is_cuda or image_arrays.is_pinned()):
        batch = image_arrays
      else:
        # stack into this slot's pinned staging buffer (reused; its last H2D must have finished)
        if slot['raw_host'] is None or tuple(slot['raw_host'].shape) != shape:
          slot['raw_host'] = torch.empty(shape, dtype=torch.uint8).pin_memory()
        slot['ev_h2d'].synchronize()
        host = slot['raw_host'].numpy()
        if isinstance(image_arrays, torch.Tensor):
          host[...] = image_arrays.to(torch.uint8).numpy()
        else:
          for i, im in enumerate(image_arrays):
            host[i] = im
        batch = slot['raw_host']
      if slot['raw_dev'] is None or tuple(slot['raw_dev'].shape) != shape:
        slot['raw_dev'] = torch.empty(shape, dtype=torch.uint8, device=self.device)
      if mirrored:                          # image i at byte i * h * w * 3 of raw_dev
        extra, _, scales = preprocess_table([shape[1:3]] * n, tuple(eng.input.shape[1:3]))
        extra[:, :2] = (np.arange(n, dtype=np.int64) * int(np.prod(shape[1:]))).view(np.int32).reshape(-1, 2)
      if extra is not None:
        slot['ev_h2d'].synchronize()        # the slot's previous H2D has read the staging buffer
        slot['extra_host'] = _grow(slot['extra_host'], extra.nbytes, pin_memory=True)
        slot['extra_dev'] = _grow(slot['extra_dev'], extra.nbytes, device=self.device)
        slot['extra_host'].numpy()[:extra.nbytes] = extra.view(np.uint8).ravel()
        extra_dev = slot['extra_dev'][:extra.nbytes].view(torch.int32).view(extra.shape)
      with torch.cuda.stream(self._copy_stream):
        self._copy_stream.wait_event(slot['ev_raw_free'])   # pre-process of the request before last
        slot['raw_dev'].copy_(batch, non_blocking=True)
        if extra is not None:
          slot['extra_dev'][:extra.nbytes].copy_(slot['extra_host'][:extra.nbytes], non_blocking=True)
        slot['ev_h2d'].record(self._copy_stream)
      main.wait_event(slot['ev_h2d'])
      if mirrored:
        ops.preprocess_mirrored(slot['raw_dev'].view(-1), extra_dev, eng.input, self.mean_rgb,
                                self.stddev_rgb)
        slot['scales'].numpy()[:] = np.concatenate([scales, scales])
      else:
        scale = ops.preprocess(slot['raw_dev'], eng.input, self.mean_rgb, self.stddev_rgb)
        slot['scales'].fill_(scale)
      slot['ev_raw_free'].record(main)
    else:  # ragged batch: descriptor rows, then the packed images; one H2D, one launch
      images = [np.asarray(im) for im in image_arrays]
      if len(images) != n:
        raise ValueError('expected %d images, got %d' % (n, len(images)))
      for im in images:
        if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
          raise ValueError('expected uint8 [h, w, 3] images, got %s %s' % (im.dtype, im.shape))
      desc, total, scales = preprocess_table([im.shape[:2] for im in images],
                                             tuple(eng.input.shape[1:3]))
      rows = desc.nbytes + (extra.nbytes if extra is not None else 0)   # desc.nbytes: 24 N
      head = (rows + 15) // 16 * 16
      staged = head + total
      slot['ev_h2d'].synchronize()          # the slot's previous H2D has read the staging buffer
      slot['packed_host'] = _grow(slot['packed_host'], staged, pin_memory=True)
      if slot['packed_dev'] is None or slot['packed_dev'].numel() < staged:
        main.synchronize()                  # no queued pre-process still reads the old buffer
        slot['packed_dev'] = _grow(slot['packed_dev'], staged, device=self.device)
      host, dev = slot['packed_host'].numpy(), slot['packed_dev']
      host[:desc.nbytes] = desc.view(np.uint8).ravel()
      if extra is not None:
        host[desc.nbytes:rows] = extra.view(np.uint8).ravel()
        extra_dev = dev[desc.nbytes:rows].view(torch.int32).view(extra.shape)
      for im, off in zip(images, desc[:, :2].copy().view(np.int64)[:, 0]):
        host[head + off:head + off + im.size] = np.ascontiguousarray(im).reshape(-1)
      with torch.cuda.stream(self._copy_stream):
        self._copy_stream.wait_event(slot['ev_raw_free'])   # pre-process of the request before last
        dev[:staged].copy_(slot['packed_host'][:staged], non_blocking=True)
        slot['ev_h2d'].record(self._copy_stream)
      main.wait_event(slot['ev_h2d'])
      (ops.preprocess_mirrored if mirrored else ops.preprocess_ragged)(
          dev[head:staged], dev[:desc.nbytes].view(torch.int32).view(desc.shape), eng.input,
          self.mean_rgb, self.stddev_rgb)
      slot['ev_raw_free'].record(main)
      slot['scales'].numpy()[:] = np.concatenate([scales, scales]) if mirrored else scales
    eng.image_scales.copy_(slot['scales'], non_blocking=True)
    return extra_dev

  def submit(self, image_arrays):
    """Enqueues one request and returns a handle; `handle.result()` blocks until its detections
    are in host memory.  Up to MAX_IN_FLIGHT (3) requests are in flight: the H2D copy and
    pre-process of request i+1, the backbone of request i, the feature network / heads of request
    i-1 and the NMS + D2H copy of request i-1 / i-2 overlap (copy stream, main stream, the engine's
    head and NMS streams).  Submitting one more request first completes the oldest one."""
    if getattr(self, '_engines', None) is None:
      self.build()
    n = len(image_arrays)
    if self.batch_size and n != self.batch_size:
      raise ValueError('expected %d images, got %d' % (self.batch_size, n))
    if n < 1:
      raise ValueError('empty request')
    with torch.cuda.device(self.device):
      eng = self._engine_for(n)
      slot = self._slots[n][self._seq % self.MAX_IN_FLIGHT]
      self._seq += 1
      if slot['pending'] is not None:
        slot['pending']._finish()          # its host buffer is about to be reused
      self._stage_raw(eng, slot, image_arrays)

      def after_nms(det, slot=slot):
        """On the engine's NMS stream right after NMS: all-gather (multi-GPU) + D2H copy."""
        det = parallel.gather_detections(det, slot['gathered'])
        slot['host_det'].copy_(det, non_blocking=True)
        slot['ev_done'].record(torch.cuda.current_stream())
      eng.run(postprocess=True, after_nms=after_nms)
    handle = _Request(slot)
    slot['pending'] = handle
    return handle

  def serve_images(self, image_arrays):
    """image_arrays: list (or array) of HxWx3 uint8 images -> float32 [N, max_output_size, 7].

    Under torch.distributed (one process per GPU, batch sharded over the ranks) the per-rank
    detection blocks are all-gathered on the device first, so every rank returns the global
    [world * N, max_output_size, 7] result (the single collective of the path)."""
    return self.submit(image_arrays).result()

  def serve_stream(self, batches):
    """Generator over an iterable of requests: yields the detections of each, in order, keeping
    MAX_IN_FLIGHT requests in flight."""
    import collections  # pylint: disable=g-import-not-at-top
    pending = collections.deque()
    for batch in batches:
      pending.append(self.submit(batch))
      if len(pending) >= self.MAX_IN_FLIGHT:
        yield pending.popleft().result()
    while pending:
      yield pending.popleft().result()

  # ---- segmentation --------------------------------------------------------------------------
  def submit_segment(self, image_arrays, resize='nearest'):
    """Enqueues one segmentation request and returns a handle; `handle.result()` blocks until the
    masks are in host memory: a list of uint8 [h_i, w_i] numpy arrays, the class of every pixel of
    each image at its own size.  Needs a config whose `heads` include 'segmentation'.

    The images are staged and pre-processed as in submit() (the mask table rides in the same H2D
    copy), the network runs without the NMS stage, then one edet_seg_masks launch samples the
    segmentation logits at the nearest cell of each image's region of the letterboxed input and
    takes the arg-max over the classes (first class on ties, like tf.argmax in the reference's
    segmentation demo).  The packed masks reach pinned host memory in one D2H copy on a stream of
    their own, so up to MAX_IN_FLIGHT requests overlap like detection requests do."""
    if resize != 'nearest':
      raise NotImplementedError('mask resize %r: only nearest sampling is built' % (resize,))
    if torch.distributed.is_available() and torch.distributed.is_initialized():
      raise NotImplementedError('segmentation masks under torch.distributed are not built')
    heads = self.params.get('heads') or []
    if 'segmentation' not in heads:
      raise ValueError("segmentation masks need 'segmentation' in heads; heads = %s" % (heads,))
    n = len(image_arrays)
    if self.batch_size and n != self.batch_size:
      raise ValueError('expected %d images, got %d' % (self.batch_size, n))
    if n < 1:
      raise ValueError('empty request')
    if getattr(self, '_engines', None) is None:
      self.build()
    with torch.cuda.device(self.device):
      eng = self._engine_for(n)
      shapes, table, total = segment_request(image_arrays, tuple(eng.input.shape[1:3]),
                                             int(self.config.seg_num_classes))
      slot = self._slots[n][self._seq % self.MAX_IN_FLIGHT]
      self._seq += 1
      if slot['pending'] is not None:
        slot['pending']._finish()          # its host buffer is about to be reused
      dev_table = self._stage_raw(eng, slot, image_arrays, extra=table)
      main = torch.cuda.current_stream()
      eng.run(postprocess=False)
      # the slot's previous request has completed (above), so neither buffer is still in use
      slot['mask_dev'] = _grow(slot['mask_dev'], total, device=self.device)
      slot['mask_host'] = _grow(slot['mask_host'], total, pin_memory=True)
      hs, ws = eng.seg_out.shape[1:3]
      f = 2 ** (self.config.min_level - 1)
      assert (hs * f, ws * f) == tuple(eng.input.shape[1:3]), 'logits grid is not input / f'
      ops.seg_masks(eng.seg_out, self.config.seg_num_classes, f, dev_table,
                    tuple(int(v) for v in np.max(np.asarray(shapes), axis=0)), slot['mask_dev'])
      slot['ev_raw_free'].record(main)     # the mask kernel has read the table
      slot['ev_masks'].record(main)
      with torch.cuda.stream(self._d2h_stream):
        self._d2h_stream.wait_event(slot['ev_masks'])
        slot['mask_host'][:total].copy_(slot['mask_dev'][:total], non_blocking=True)
        slot['ev_done'].record(self._d2h_stream)
    handle = _SegmentRequest(slot, [tuple(int(v) for v in s) for s in shapes], total)
    slot['pending'] = handle
    return handle

  def segment_images(self, image_arrays, resize='nearest'):
    """image_arrays: list of HxWx3 uint8 images (sizes may differ) or a uint8 [N, h, w, 3] tensor
    -> list of uint8 [h_i, w_i] numpy masks, one per image (see submit_segment)."""
    return self.submit_segment(image_arrays, resize).result()

  def segment_stream(self, batches, resize='nearest'):
    """Generator over an iterable of requests: yields the masks of each, in order, keeping
    MAX_IN_FLIGHT requests in flight."""
    import collections  # pylint: disable=g-import-not-at-top
    pending = collections.deque()
    for batch in batches:
      pending.append(self.submit_segment(batch, resize))
      if len(pending) >= self.MAX_IN_FLIGHT:
        yield pending.popleft().result()
    while pending:
      yield pending.popleft().result()

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
    n = len(image_arrays)
    if self.batch_size and n != self.batch_size:
      raise ValueError('expected %d images, got %d' % (self.batch_size, n))
    if n < 1:
      raise ValueError('empty request')
    if getattr(self, '_engines', None) is None:
      self.build()
    with torch.cuda.device(self.device):
      eng = self._engine_for(2 * n)
      slot = self._slots[2 * n][self._seq % self.MAX_IN_FLIGHT]
      self._seq += 1
      if slot['pending'] is not None:
        slot['pending']._finish()          # its buffers are about to be reused
      self._stage_raw(eng, slot, image_arrays, mirrored=True)
      nms = self.config.as_dict()['nms_configs']
      max_out = eng.max_output_size
      cap = 2 * max_out
      if slot.get('tta_det') is None:       # the slot's own buffers, reused by its later requests
        k = eng.total_anchors if not eng.max_nms_inputs else eng.max_nms_inputs
        ids = np.float32(self.image_id_base) + np.arange(n, dtype=np.float32)
        size = n * cap * 7 + n
        slot.update(
            tta_det=torch.empty(2 * n, max_out, 7, device=self.device),
            tta_keep=torch.empty(2 * n, max_out, dtype=torch.int32, device=self.device),
            tta_valid=torch.empty(2 * n, dtype=torch.int32, device=self.device),
            tta_work=torch.empty(2 * n, k, device=self.device),
            tta_ids=torch.from_numpy(np.concatenate([ids, ids])).to(self.device),
            tta_scales=torch.empty(2 * n, device=self.device),
            tta_out=torch.empty(size, device=self.device),
            tta_host=torch.empty(size).pin_memory())
      main = torch.cuda.current_stream()
      slot['tta_scales'].copy_(slot['scales'], non_blocking=True)
      eng.run(postprocess=False)
      ps = eng.pre_nms_only()
      ops.per_class_nms(ps['boxes'], ps['scores'], ps['classes'], slot['tta_ids'],
                        slot['tta_scales'], self.config.num_classes, max_out, nms['method'],
                        nms.get('iou_thresh'), slot['tta_det'], slot['tta_keep'], slot['tta_valid'],
                        sigma=nms.get('sigma'), score_thresh=nms.get('score_thresh'),
                        work=slot['tta_work'])
      out = slot['tta_out']
      ops.wbf(slot['tta_det'], 2, self.config.num_classes, out[:n * cap * 7].view(n, cap, 7),
              out[n * cap * 7:].view(torch.int32), mirrored_mask=0b10,
              image_scales=slot['tta_scales'][:n], width=eng.input.shape[2])
      slot['ev_masks'].record(main)
      with torch.cuda.stream(self._d2h_stream):
        self._d2h_stream.wait_event(slot['ev_masks'])
        slot['tta_host'].copy_(out, non_blocking=True)
        slot['ev_done'].record(self._d2h_stream)
    handle = _TTARequest(slot, n, cap)
    slot['pending'] = handle
    return handle

  def serve_images_tta(self, image_arrays):
    """image_arrays: list of HxWx3 uint8 images (sizes may differ) or a uint8 [N, h, w, 3] tensor
    -> list of float32 [k_i, 7] numpy arrays of fused detections, one per image (see submit_tta)."""
    return self.submit_tta(image_arrays).result()

  def serve_stream_tta(self, batches):
    """Generator over an iterable of requests: yields the fused detections of each, in order,
    keeping MAX_IN_FLIGHT requests in flight."""
    import collections  # pylint: disable=g-import-not-at-top
    pending = collections.deque()
    for batch in batches:
      pending.append(self.submit_tta(batch))
      if len(pending) >= self.MAX_IN_FLIGHT:
        yield pending.popleft().result()
    while pending:
      yield pending.popleft().result()

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
