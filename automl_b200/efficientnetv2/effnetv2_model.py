"""EfficientNet V1 / V2 backbone on the H100 path: the forward pass of the reference's
efficientnetv2/effnetv2_model.py (`EffNetV2Model.call` :595-658) lowered to the C-ABI kernels.

  model = effnetv2_model.get_model('efficientnetv2-s', include_top=True, weights=None,
                                   batch_size=128, image_size=384)
  logits = model(images)                         # float32 [N, 1000]
  outs = model(images, with_endpoints=True)      # [logits, reduction_1, ..., reduction_5]
  probs, classes = model.classify(uint8_images, top_k=5)   # decoded images of any size -> top-5

  model = effnetv2_model.get_model('efficientnetv2-s', weights=None, batch_size=128, image_size=384)
  features = model(images)                       # head_1x1 feature map, fp16 [N, h, w, 1280]

Mirrored: block-string configs, `round_filters` (:84-95, no 0.9 rule) / `round_repeats` (:98-102),
block expansion (:541-566), `MBConvBlock` (:150-311), `FusedMBConvBlock` (:313-406, no SE in any
registered model; expand_ratio == 1 blocks are ONE k x k conv followed by the activation),
`SE` (:105-147), `Stem` (:409-432), the 1x1 head conv + BN + act (`Head` :435-470, endpoint
'head_1x1'), residual rule (:270-277), endpoints 'reduction_i' (:616-637) and, with
include_top=True, the classification top: global average pooling (`Head.call` :477-496, endpoints
'pooled_features' and 'head', float32; dropout is the identity at inference) and the Dense `_fc`
(:571-578, :644-646), float32 from the pooled mean to the logits.  Out of scope: pretrained-weight
download, training (dropout, survival_prob / drop_connect are identities at inference).

Variable names follow the Keras layer names of the reference: <model>/stem/conv2d/kernel,
<model>/blocks_<i>/{conv2d, conv2d_1, depthwise_conv2d, se/conv2d, se/conv2d_1,
tpu_batch_normalization[_n]}, <model>/head/conv2d/kernel; the un-named BN layers of Stem / Head are
named 'tpu_batch_normalization' by the reference's utils.BatchNormalization (utils.py:209-215), the
un-named Dense layer gets Keras' default 'dense' (<model>/dense/kernel [head_filters, num_classes],
<model>/dense/bias).
"""
import collections
import math

import numpy as np
import torch

from automl_b200 import ops
from automl_b200 import staging
from automl_b200 import utils
from automl_b200.backbone.efficientnet_builder import _layer_namer
from automl_b200.efficientnetv2 import effnetv2_configs
from automl_b200.efficientnetv2 import preprocessing
from automl_b200.lowering import LaunchList, bn_fold, capture_graph
from automl_b200.weights import VarSpec, _bn

Block = collections.namedtuple('Block', [
    'name', 'conv_type', 'kernel_size', 'strides', 'expand_ratio', 'input_filters',
    'output_filters', 'mid_filters', 'se_filters', 'has_skip',
    'expand_name', 'expand_bn',    # None when expand_ratio == 1
    'dw_bn',                       # None for Fused-MBConv (conv_type 1)
    'project_name', 'project_bn'])


def round_filters(filters, mconfig, skip=False):
  """effnetv2_model.py:84-95."""
  multiplier = mconfig.width_coefficient
  divisor = mconfig.depth_divisor
  min_depth = mconfig.min_depth
  if skip or not multiplier:
    return filters
  filters *= multiplier
  min_depth = min_depth or divisor
  new_filters = max(min_depth, int(filters + divisor / 2) // divisor * divisor)
  return int(new_filters)


def round_repeats(repeats, multiplier, skip=False):
  """effnetv2_model.py:98-102."""
  if skip or not multiplier:
    return repeats
  return int(math.ceil(multiplier * repeats))


class EffNetV2Arch(object):
  """The resolved network: stem width, flat block list, head width, reduction endpoints."""

  def __init__(self, model_name='efficientnetv2-s', model_config=None):
    cfg = effnetv2_configs.get_model_config(model_name)
    if model_config:
      cfg.model.override(model_config)    # the model section, as the reference does (:525)
    self.cfg = cfg
    m = self.mconfig = cfg.model
    self.model_name = model_name
    self.model_config = model_config    # the override as given, for checkers that re-resolve it
    if m.act_fn not in ('silu', 'swish', 'relu6'):
      raise NotImplementedError('act_fn %s' % m.act_fn)
    self.act = utils.ACT_RELU6 if m.act_fn == 'relu6' else utils.ACT_SWISH
    self.bn_eps = m.bn_epsilon
    self.stem_filters = round_filters(m.blocks_args[0].input_filters, m)
    self.blocks = []
    for ba in m.blocks_args:
      assert ba.num_repeat > 0
      cin, cout = round_filters(ba.input_filters, m), round_filters(ba.output_filters, m)
      stride = ba.strides
      for _ in range(round_repeats(ba.num_repeat, m.depth_coefficient)):
        has_se = ba.se_ratio is not None and 0 < ba.se_ratio <= 1
        # the reference sizes the SE bottleneck from the block's (rounded) input filters
        se = max(1, int(cin * ba.se_ratio)) if has_se else 0
        # Keras layer names in creation order: expand conv + BN, depthwise BN, project conv + BN
        conv, bn = _layer_namer('conv2d'), _layer_namer('tpu_batch_normalization')
        expand_name, expand_bn = (conv(), bn()) if ba.expand_ratio != 1 else (None, None)
        dw_bn = bn() if ba.conv_type == 0 else None
        self.blocks.append(Block(
            name='blocks_%d' % len(self.blocks), conv_type=ba.conv_type,
            kernel_size=ba.kernel_size, strides=stride, expand_ratio=ba.expand_ratio,
            input_filters=cin, output_filters=cout, mid_filters=cin * ba.expand_ratio,
            se_filters=se, has_skip=(stride == 1 and cin == cout),
            expand_name=expand_name, expand_bn=expand_bn, dw_bn=dw_bn,
            project_name=conv(), project_bn=bn()))
        cin, stride = cout, 1
    self.head_filters = round_filters(m.feature_size or 1280, m)
    # a block is a reduction endpoint when it is last or the next block strides (:616-621)
    self.reductions = [i for i, b in enumerate(self.blocks)
                       if i == len(self.blocks) - 1 or self.blocks[i + 1].strides > 1]


def variable_specs(arch, include_top=False):
  """OrderedDict name -> VarSpec (Keras layouts) for the backbone + head conv and, with include_top
  and a non-zero num_classes (:572), the Dense classifier after them."""
  s = collections.OrderedDict()
  mn = arch.model_name
  s['%s/stem/conv2d/kernel' % mn] = VarSpec((3, 3, 3, arch.stem_filters), 'conv', True)
  _bn(s, '%s/stem/tpu_batch_normalization' % mn, arch.stem_filters)
  for b in arch.blocks:
    sc = '%s/%s' % (mn, b.name)
    if b.expand_name:
      ek = 1 if b.conv_type == 0 else b.kernel_size
      s['%s/%s/kernel' % (sc, b.expand_name)] = VarSpec((ek, ek, b.input_filters, b.mid_filters), 'conv', True)
      _bn(s, '%s/%s' % (sc, b.expand_bn), b.mid_filters)
    if b.dw_bn:
      s['%s/depthwise_conv2d/depthwise_kernel' % sc] = VarSpec(
          (b.kernel_size, b.kernel_size, b.mid_filters, 1), 'dw', True)
      _bn(s, '%s/%s' % (sc, b.dw_bn), b.mid_filters)
    if b.se_filters:
      s['%s/se/conv2d/kernel' % sc] = VarSpec((1, 1, b.mid_filters, b.se_filters), 'conv', True)
      s['%s/se/conv2d/bias' % sc] = VarSpec((b.se_filters,), 'se_bias', True)
      s['%s/se/conv2d_1/kernel' % sc] = VarSpec((1, 1, b.se_filters, b.mid_filters), 'conv', True)
      s['%s/se/conv2d_1/bias' % sc] = VarSpec((b.mid_filters,), 'se_bias', True)
    pk = b.kernel_size if (b.conv_type == 1 and b.expand_ratio == 1) else 1
    s['%s/%s/kernel' % (sc, b.project_name)] = VarSpec((pk, pk, b.mid_filters, b.output_filters), 'conv', True)
    last_bn = '%s/%s' % (sc, b.project_bn)
    _bn(s, last_bn, b.output_filters)
    # synthetic init only: a small gain on the residual branch keeps 40-100 stacked blocks O(1)
    s[last_bn + '/gamma'] = VarSpec((b.output_filters,), 'gamma_res' if b.has_skip else 'gamma', True)
  s['%s/head/conv2d/kernel' % mn] = VarSpec((1, 1, arch.blocks[-1].output_filters, arch.head_filters),
                                            'conv', True)
  _bn(s, '%s/head/tpu_batch_normalization' % mn, arch.head_filters)
  if include_top and arch.mconfig.num_classes:
    s['%s/dense/kernel' % mn] = VarSpec((arch.head_filters, arch.mconfig.num_classes), 'dense', True)
    s['%s/dense/bias' % mn] = VarSpec((arch.mconfig.num_classes,), 'dense_bias', True)
  return s


def count_params(arch, include_top=True):
  """Keras `model.count_params()` of the reference model: every variable above (BN moving
  statistics included) and, with include_top, the Dense classifier (effnetv2_model_test.py:25-48)."""
  return sum(int(np.prod(v.shape)) for v in variable_specs(arch, include_top).values())


def synthetic_weights(arch, seed=0, include_top=False):
  """Seeded float32 weights keyed by variable name (no checkpoints offline).  The Dense tensors
  are drawn last, so the backbone of a seed has the same bits with and without the top."""
  rng = np.random.default_rng(seed)
  out = collections.OrderedDict()
  for name, spec in variable_specs(arch, include_top).items():
    shape, kind = spec.shape, spec.kind
    if kind == 'conv':
      kh, kw, cin, _ = shape
      w = rng.normal(0.0, math.sqrt(2.0 / (kh * kw * cin)), size=shape)
    elif kind == 'dw':
      w = rng.normal(0.0, math.sqrt(2.0 / (shape[0] * shape[1])) * 0.7, size=shape)
    elif kind == 'gamma':
      w = rng.uniform(0.8, 1.2, size=shape)
    elif kind == 'gamma_res':
      w = rng.uniform(0.2, 0.4, size=shape)
    elif kind in ('beta', 'mean', 'se_bias'):
      w = rng.normal(0.0, 0.1, size=shape)
    elif kind == 'var':
      w = rng.uniform(0.5, 1.5, size=shape)
    elif kind == 'dense':          # N(0, 1/K): logits of O(1)
      w = rng.normal(0.0, math.sqrt(1.0 / shape[0]), size=shape)
    elif kind == 'dense_bias':     # the reference's constant (:576), perturbed so a wrong bias shows
      w = (arch.mconfig.headbias or 0) + rng.normal(0.0, 0.1, size=shape)
    else:
      raise AssertionError(kind)
    out[name] = np.asarray(w, np.float32)
  return out


class EffNetV2Model(LaunchList):
  """One network instance bound to a device, a batch size and an image size (static buffers, the
  forward pass is one CUDA graph).  There is no CPU fallback.

  include_top=True adds the pooling and, when num_classes is non-zero, the Dense classifier: the
  model returns float32 logits [N, num_classes] (the pooled features [N, C] when num_classes is 0).
  include_top=False returns the fp16 'head_1x1' map; the reference returns the pooled tensor there,
  which this path has never done and callers of the feature map rely on."""

  def __init__(self, model_name='efficientnetv2-s', model_config=None, include_top=False,
               weights=None, batch_size=1, image_size=None, device='cuda:0', use_cuda_graph=True,
               seed=0):
    if not torch.cuda.is_available():
      raise RuntimeError('EffNetV2Model needs a CUDA device; there is no CPU fallback')
    self.arch = a = EffNetV2Arch(model_name, model_config)
    self.cfg = a.cfg
    self.n = int(batch_size)
    size = image_size or a.cfg.eval.isize
    self.image_size = utils.parse_image_size(size)
    super().__init__(device)
    self.act = a.act
    self.use_cuda_graph = use_cuda_graph
    self.include_top = bool(include_top)
    if weights is None:
      weights = synthetic_weights(a, seed, self.include_top)
    elif isinstance(weights, str):
      data = np.load(weights)
      names = list(variable_specs(a, self.include_top))
      missing = [k for k in names if k not in data.files]
      if missing:
        raise ValueError('%s lacks %d variables of %s%s: %s' % (
            weights, len(missing), a.model_name, ' (include_top=True)' if self.include_top else '',
            ', '.join(missing[:8]) + (', ...' if len(missing) > 8 else '')))
      weights = {k: np.asarray(data[k], np.float32) for k in names}
    self.endpoints = {}
    self._graph = None
    with torch.cuda.device(self.device):
      self._build(weights)

  # ---- lowering -----------------------------------------------------------------------------
  def _build(self, w):
    a, n, act, eps = self.arch, self.n, self.act, self.arch.bn_eps
    f16, f32 = torch.float16, torch.float32
    mn = a.model_name
    h, wd = self.image_size
    self.input = self._buf('input', (n, h, wd, 3), f32)
    for c in [a.stem_filters, a.head_filters] + [v for b in a.blocks for v in
                                                  (b.input_filters, b.mid_filters, b.output_filters)]:
      if c % 8:
        raise ValueError('channel count %d is not a multiple of 8' % c)

    def conv_w(name, scope_bn):
      """Conv2D kernel [kh,kw,Cin,Cout] with its BN folded -> ([taps, Cout, Cin] fp16, bias fp32)."""
      s, sh = bn_fold(w, scope_bn, eps)
      k = np.asarray(w[name], np.float64) * s
      kh, kw, cin, cout = k.shape
      return self._dev(k.transpose(0, 1, 3, 2).reshape(kh * kw, cout, cin), f16), self._dev(sh, f32)

    # stem: conv3x3 s2 3 -> C + BN + act (Stem :409-432)
    h, wd = -(-h // 2), -(-wd // 2)
    x = self._stem(w, mn + '/stem/conv2d', mn + '/stem/tpu_batch_normalization', (h, wd))
    self.endpoints['stem'] = x
    self._se_accumulators(a.blocks)
    red = 0
    for bi, b in enumerate(a.blocks):
      sc = '%s/%s' % (mn, b.name)
      if b.conv_type == 0:
        y, (ho, wo) = self._mbconv(w, sc, b, x, (h, wd), b.strides)
      else:
        if b.se_filters:
          raise NotImplementedError('Fused-MBConv with SE (no registered model has it)')
        x_in, s_ = x, b.strides
        ho, wo = -(-h // s_), -(-wd // s_)
        res = x_in if b.has_skip else None
        y = self._buf(b.name + '/out', (n, ho, wo, b.output_filters))
        if b.expand_name:
          ew, eb = conv_w('%s/%s/kernel' % (sc, b.expand_name), '%s/%s' % (sc, b.expand_bn))
          mid = self._buf(b.name + '/expand_kxk', (n, ho, wo, b.mid_filters))
          self._add(b.name + '/expand_kxk',
                    lambda x_in=x_in, ew=ew, eb=eb, mid=mid, b=b:
                    ops.conv2d(x_in, ew, eb, mid, act, b.kernel_size, b.strides), 'conv_tc',
                    nbytes=2 * (x_in.numel() + mid.numel() + ew.numel()),
                    flops=2 * b.kernel_size**2 * b.input_filters * mid.numel())
          pw, pb = conv_w('%s/%s/kernel' % (sc, b.project_name), '%s/%s' % (sc, b.project_bn))
          self._add(b.name + '/project',
                    lambda mid=mid, pw=pw, pb=pb, y=y, res=res:
                    ops.pointwise_conv(mid, pw[0], pb, y, utils.ACT_NONE, residual=res),
                    'pointwise_tc', nbytes=2 * (mid.numel() + y.numel() * (2 if res is not None else 1)),
                    flops=2 * b.mid_filters * y.numel())
        else:   # ONE k x k conv + BN + act (+ skip)   (:355-364, :401-402)
          pw, pb = conv_w('%s/%s/kernel' % (sc, b.project_name), '%s/%s' % (sc, b.project_bn))
          self._add(b.name + '/conv_kxk',
                    lambda x_in=x_in, pw=pw, pb=pb, y=y, res=res, b=b:
                    ops.conv2d(x_in, pw, pb, y, act, b.kernel_size, b.strides, residual=res),
                    'conv_tc', nbytes=2 * (x_in.numel() + y.numel() * (2 if res is not None else 1)),
                    flops=2 * b.kernel_size**2 * b.input_filters * y.numel())
      x, h, wd = y, ho, wo
      self.endpoints['block_%d' % bi] = y
      if bi in a.reductions:
        red += 1
        self.endpoints['reduction_%d' % red] = y
    self.endpoints['features'] = x
    hw_, hb_ = conv_w('%s/head/conv2d/kernel' % mn, '%s/head/tpu_batch_normalization' % mn)
    head = self._buf('head_1x1', (n, h, wd, a.head_filters))
    self._add('head_1x1', lambda x=x, head=head: ops.pointwise_conv(x, hw_[0], hb_, head, act),
              'pointwise_tc', nbytes=2 * (x.numel() + head.numel()),
              flops=2 * a.blocks[-1].output_filters * head.numel())
    self.endpoints['head_1x1'] = self.output = head
    if not self.include_top:
      return
    # Head.call :477-496: global average pooling; dropout is the identity at inference, so 'head'
    # is the pooled tensor.  local_pooling keeps the [N,1,1,C] shape of avg_pool until the Dense.
    pooled = self._buf('avg_pool', (n, a.head_filters), f32)
    self._add('avg_pool', lambda: ops.global_avg_pool(head, pooled), 'global_avg_pool',
              nbytes=2 * head.numel() + 4 * pooled.numel(), flops=head.numel())
    view = pooled.view(n, 1, 1, -1) if a.mconfig.local_pooling else pooled
    self.endpoints['pooled_features'] = self.endpoints['head'] = view
    self.output = pooled
    nc = a.mconfig.num_classes
    if nc:                      # _build :571-578, call :644-646
      fc_w = self._dev(np.asarray(w['%s/dense/kernel' % mn], np.float64).T, f16)   # [classes, K]
      fc_b = self._dev(w['%s/dense/bias' % mn], f32)
      logits = self._buf('dense', (n, nc), f32)
      self._add('dense', lambda: ops.dense(pooled, fc_w, fc_b, logits), 'dense',
                nbytes=2 * fc_w.numel() + 4 * (pooled.numel() + fc_b.numel() + logits.numel()),
                flops=2 * fc_w.numel() * n)
      self.output = logits

  # ---- execution ----------------------------------------------------------------------------
  def _run_ops(self):
    for _, fn in self._ops:
      fn()

  def run(self):
    with torch.cuda.device(self.device):
      if not self.use_cuda_graph:
        self._run_ops()
        return
      if self._graph is None:
        self._run_ops()                      # warm-up (loads kernels, sets attributes)
        torch.cuda.synchronize()
        self._graph = capture_graph(self._run_ops)
      self._graph.replay()

  def __call__(self, images=None, training=False, with_endpoints=False):
    """images float32 [N,H,W,3] (already scaled to [-1,1], preprocessing.py:82-83) -> the model
    output `out`: float32 logits [N, num_classes] with include_top (pooled features [N, C] when
    num_classes is 0), else the fp16 'head_1x1' feature map; with_endpoints [out, reduction_1,
    ...] (:648-657)."""
    if training:
      raise NotImplementedError('inference only')
    if images is not None:
      t = torch.as_tensor(images)
      if tuple(t.shape) != tuple(self.input.shape):
        raise ValueError('expected input shape %s, got %s' % (tuple(self.input.shape), tuple(t.shape)))
      self.input.copy_(t.to(torch.float32), non_blocking=True)
    self.run()
    out = self.output
    if with_endpoints:
      return [out] + [self.endpoints['reduction_%d' % i] for i in range(1, 6)
                      if 'reduction_%d' % i in self.endpoints]
    return out


  def serve_stream(self, batches):
    """Pipelined __call__ over an iterable of host batches (float32 [N,H,W,3], ideally pinned):
    the H2D copy of batch i+1 and the D2H copy of the output of batch i-1 overlap the network
    of batch i (two copy streams for the two PCIe directions, device staging buffers on both
    sides).  Yields the model output of each batch (what __call__ returns: float32 logits with
    include_top, else the float16 'head_1x1' feature map), in order, as a pinned host tensor
    that stays valid until two further results have been yielded.

    The D2H copy of result k is enqueued before result k-1 is yielded, so the pinned results form a
    ring of three: result k is rewritten by the copy of result k+3, which starts while the caller
    asks for result k+2."""
    with torch.cuda.device(self.device):
      if getattr(self, '_pipe', None) is None:
        result = self.output
        self._pipe = {
            'in': [torch.empty_like(self.input) for _ in range(2)],
            'out': [torch.empty_like(result) for _ in range(2)],
            'host': [torch.empty(tuple(result.shape), dtype=result.dtype).pin_memory() for _ in range(3)],
            'h2d': torch.cuda.Stream(device=self.device), 'd2h': torch.cuda.Stream(device=self.device),
            'ev_h2d': [torch.cuda.Event() for _ in range(2)],
            'ev_in_free': [torch.cuda.Event() for _ in range(2)],
            'ev_out': [torch.cuda.Event() for _ in range(2)],
            'ev_d2h': [torch.cuda.Event() for _ in range(3)],    # one per pinned result
        }
      p = self._pipe
      main = torch.cuda.current_stream(self.device)
      result = self.output
      prev = None
      for k, batch in enumerate(batches):
        s, h = k % 2, k % 3         # device staging ring of two, pinned results of three
        t = torch.as_tensor(batch)
        if tuple(t.shape) != tuple(self.input.shape):
          raise ValueError('expected input shape %s, got %s' % (tuple(self.input.shape), tuple(t.shape)))
        with torch.cuda.stream(p['h2d']):
          p['h2d'].wait_event(p['ev_in_free'][s])        # batch k-2 has left this staging buffer
          p['in'][s].copy_(t.to(torch.float32), non_blocking=True)
          p['ev_h2d'][s].record(p['h2d'])
        main.wait_event(p['ev_h2d'][s])
        self.input.copy_(p['in'][s], non_blocking=True)
        p['ev_in_free'][s].record(main)
        self.run()
        main.wait_event(p['ev_d2h'][(k - 2) % 3])        # result k-2 has left this staging buffer
        p['out'][s].copy_(result, non_blocking=True)
        p['ev_out'][s].record(main)
        with torch.cuda.stream(p['d2h']):
          p['d2h'].wait_event(p['ev_out'][s])
          p['host'][h].copy_(p['out'][s], non_blocking=True)
          p['ev_d2h'][h].record(p['d2h'])
        if prev is not None:
          p['ev_d2h'][prev].synchronize()
          yield p['host'][prev]
        prev = h
      if prev is not None:
        p['ev_d2h'][prev].synchronize()
        yield p['host'][prev]

  # ---- classification from decoded images -------------------------------------------------------
  def _cls_slot(self):
    """The next of two request slots (_ClassifySlot) and the copy and D2H streams they share."""
    if getattr(self, '_cls', None) is None:
      self._cls = {
          'seq': 0, 'copy': torch.cuda.Stream(device=self.device),
          'd2h': torch.cuda.Stream(device=self.device),
          'slots': [_ClassifySlot(self.n, self.device) for _ in range(2)],
      }
    c = self._cls
    slot = c['slots'][c['seq'] % 2]
    c['seq'] += 1
    return slot

  def _preprocess_into(self, slot, image_arrays):
    """Stages one request in `slot` (staging.StagingSlot.stage: the descriptor rows and the images
    in one H2D on the copy stream) and enqueues its pre-process into self.input on the current
    stream."""
    h, w = self.image_size
    if h != w:
      raise ValueError('the classification pre-process needs a square image_size, got %dx%d' % (h, w))
    legacy = preprocessing.is_legacy(self.cfg.data.augname)
    request = staging.decoded_images(image_arrays, self.n, self.input.device)
    desc, _ = preprocessing.image_table(request.shapes, h, legacy)
    (table,), images = slot.staging.stage(self._cls['copy'], [desc], request,
                                          desc[:, :2].copy().view(np.int64)[:, 0])
    ops.cls_preprocess(images, table, self.input, ops.CLS_BICUBIC if legacy else ops.CLS_BILINEAR,
                       preprocessing.device_table(self.device) if legacy else None)
    slot.staging.release()

  def preprocess(self, image_arrays):
    """Fills self.input from decoded images -- a list of uint8 [h, w, 3] arrays (sizes may differ)
    or a uint8 [N, h, w, 3] tensor (pinned host or CUDA) -- with the model's eval recipe
    (cfg.data.augname, see preprocessing.py) at its square image_size, in one launch on the
    current stream.  Returns self.input."""
    with torch.cuda.device(self.device):
      self._preprocess_into(self._cls_slot(), image_arrays)
    return self.input

  def _check_top_k(self, top_k):
    nc = self.arch.mconfig.num_classes if self.include_top else 0
    if not nc:
      raise ValueError('classify needs include_top=True and num_classes > 0')
    if not 1 <= int(top_k) <= min(nc, ops.SOFTMAX_TOPK_MAX_K):
      raise ValueError('top_k=%s must be in [1, %d]' % (top_k, min(nc, ops.SOFTMAX_TOPK_MAX_K)))
    return int(top_k)

  def _classify_enqueue(self, image_arrays, k):
    """Pre-process, graph replay and softmax top-k on the current stream, then the D2H of the
    [N, k] results on the d2h stream.  Returns the slot."""
    slot = self._cls_slot()
    self._preprocess_into(slot, image_arrays)
    self.run()
    main = torch.cuda.current_stream(self.device)
    n = self.n
    main.wait_event(slot.ev_d2h)              # the slot's previous results have left the device
    ops.softmax_topk(self.output, slot.probs[:n * k].view(n, k), slot.classes[:n * k].view(n, k))
    slot.ev_out.record(main)
    d2h = self._cls['d2h']
    with torch.cuda.stream(d2h):
      d2h.wait_event(slot.ev_out)
      slot.host_probs[:n * k].copy_(slot.probs[:n * k], non_blocking=True)
      slot.host_classes[:n * k].copy_(slot.classes[:n * k], non_blocking=True)
      slot.ev_d2h.record(d2h)
    slot.k = k
    return slot

  def classify(self, image_arrays, top_k=5):
    """Decoded uint8 images (as `preprocess` takes them) -> (probs float32 [N, top_k], classes
    int32 [N, top_k]) numpy arrays: the top_k classes by logit (ties: lower class first) and their
    softmax probabilities.  Needs include_top=True and num_classes > 0; 1 <= top_k <=
    min(num_classes, 32)."""
    k = self._check_top_k(top_k)
    with torch.cuda.device(self.device):
      return self._classify_enqueue(image_arrays, k).result()

  def classify_stream(self, batches, top_k=5):
    """Pipelined `classify` over an iterable of requests, two in flight: the H2D copy of request
    i+1 and the D2H copy of the results of request i-1 overlap the network of request i.  Yields
    (probs, classes) numpy arrays per request, in order."""
    k = self._check_top_k(top_k)
    with torch.cuda.device(self.device):
      yield from staging.pipelined(lambda batch: self._classify_enqueue(batch, k), batches, 2)


class _ClassifySlot(object):
  """One of the classifier's two request slots: its staging, the top-k outputs on the device and in
  pinned memory, and the events ordering their reuse."""

  def __init__(self, n, device):
    size = n * ops.SOFTMAX_TOPK_MAX_K
    self.n, self.k = n, None
    self.staging = staging.StagingSlot(device)
    self.probs = torch.empty(size, dtype=torch.float32, device=device)
    self.classes = torch.empty(size, dtype=torch.int32, device=device)
    self.host_probs = torch.empty(size, dtype=torch.float32).pin_memory()
    self.host_classes = torch.empty(size, dtype=torch.int32).pin_memory()
    self.ev_out, self.ev_d2h = torch.cuda.Event(), torch.cuda.Event()

  def result(self):
    """(probs, classes) numpy [N, k] of the slot's latest request, once they are in host memory."""
    self.ev_d2h.synchronize()
    n, k = self.n, self.k
    return (self.host_probs[:n * k].numpy().reshape(n, k).copy(),
            self.host_classes[:n * k].numpy().reshape(n, k).copy())


def get_model(model_name, model_config=None, include_top=False, weights=None, training=False,
              with_endpoints=False, **kwargs):
  """effnetv2_model.get_model (:661-722) for inference: returns the bound model instance
  (pretrained-weight download is out of scope: weights is None / a dict / an .npz path)."""
  if training:
    raise NotImplementedError('inference only')
  if weights in ('imagenet', 'imagenet21k', 'imagenet21k-ft1k', 'jft'):
    raise NotImplementedError('pretrained weight download is out of scope (no network)')
  del with_endpoints  # chosen per call
  return EffNetV2Model(model_name, model_config, include_top, weights=weights, **kwargs)
