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

The whole request runs on the device: H2D copy of the uint8 images -> edet_preprocess ->
network -> pre-NMS -> NMS -> D2H copy of the [N, max_output_size, 7] detections.
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
    self._seq = 0
    self.engine = self._engine_for(self.batch_size) if self.batch_size else None
    self.signitures = {
        'image_files': 'image_files',     # bytes of encoded images (serve_files)
        'image_arrays': 'image_arrays',   # uint8 HxWx3 arrays (serve_images)
        'prediction': self.engine.detections if self.engine is not None else 'detections',
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
          'raw_host': None, 'raw_dev': None,
          'ev_h2d': torch.cuda.Event(), 'ev_raw_free': torch.cuda.Event(),
          'ev_done': torch.cuda.Event(), 'pending': None,
      } for _ in range(self.MAX_IN_FLIGHT)]
    return eng

  # ---- serving -------------------------------------------------------------------------------
  def _stage_raw(self, eng, slot, image_arrays):
    """Uploads the uint8 images (copy stream, from pinned memory) and runs the device pre-process
    into the engine input (current stream)."""
    n = eng.n
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
      with torch.cuda.stream(self._copy_stream):
        self._copy_stream.wait_event(slot['ev_raw_free'])   # pre-process of the request before last
        slot['raw_dev'].copy_(batch, non_blocking=True)
        slot['ev_h2d'].record(self._copy_stream)
      main.wait_event(slot['ev_h2d'])
      scale = ops.preprocess(slot['raw_dev'], eng.input, self.mean_rgb, self.stddev_rgb)
      slot['ev_raw_free'].record(main)
      slot['scales'].fill_(scale)
    else:  # ragged batch: one pre-process launch per image (like the reference's python loop)
      for i, im in enumerate(image_arrays):
        raw = torch.as_tensor(np.ascontiguousarray(im), dtype=torch.uint8).to(self.device)[None]
        slot['scales'][i] = ops.preprocess(raw, eng.input[i:i + 1], self.mean_rgb, self.stddev_rgb)
    eng.image_scales.copy_(slot['scales'], non_blocking=True)

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
