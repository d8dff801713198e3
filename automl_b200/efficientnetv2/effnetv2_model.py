"""EfficientNet V1 / V2 backbone on the H100 path: the forward pass of the reference's
efficientnetv2/effnetv2_model.py (`EffNetV2Model.call` :595-658) lowered to the C-ABI kernels.

  model = effnetv2_model.get_model('efficientnetv2-s', weights=None, batch_size=128, image_size=384)
  features = model(images)                       # head_1x1 feature map, fp16 [N, h, w, 1280]
  outs = model(images, with_endpoints=True)      # [head_1x1, reduction_1, ..., reduction_5]

Mirrored: block-string configs, `round_filters` (:84-95, no 0.9 rule) / `round_repeats` (:98-102),
block expansion (:541-566), `MBConvBlock` (:150-311), `FusedMBConvBlock` (:313-406, no SE in any
registered model; expand_ratio == 1 blocks are ONE k x k conv followed by the activation),
`SE` (:105-147), `Stem` (:409-432), the 1x1 head conv + BN + act (`Head` :435-470, endpoint
'head_1x1'), residual rule (:270-277), endpoints 'reduction_i' (:616-637).  Out of scope (SURVEY.md
row 21): global pooling + dropout + the classification `_fc`, pretrained-weight download,
training (survival_prob / drop_connect are identities at inference).

Variable names follow the Keras layer names of the reference: <model>/stem/conv2d/kernel,
<model>/blocks_<i>/{conv2d, conv2d_1, depthwise_conv2d, se/conv2d, se/conv2d_1,
tpu_batch_normalization[_n]}, <model>/head/conv2d/kernel; the un-named BN layers of Stem / Head get
Keras' default 'batch_normalization'.
"""
import collections
import math

import numpy as np
import torch

from automl_b200 import ops
from automl_b200 import utils
from automl_b200.efficientnetv2 import effnetv2_configs
from automl_b200.weights import VarSpec, _bn

Block = collections.namedtuple('Block', [
    'name', 'conv_type', 'kernel_size', 'strides', 'expand_ratio', 'input_filters',
    'output_filters', 'mid_filters', 'se_filters', 'has_skip'])


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
      cfg.override(model_config)
    self.cfg = cfg
    m = self.mconfig = cfg.model
    self.model_name = model_name
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
        self.blocks.append(Block(
            name='blocks_%d' % len(self.blocks), conv_type=ba.conv_type,
            kernel_size=ba.kernel_size, strides=stride, expand_ratio=ba.expand_ratio,
            input_filters=cin, output_filters=cout, mid_filters=cin * ba.expand_ratio,
            se_filters=se, has_skip=(stride == 1 and cin == cout)))
        cin, stride = cout, 1
    self.head_filters = round_filters(m.feature_size or 1280, m)
    # a block is a reduction endpoint when it is last or the next block strides (:616-621)
    self.reductions = [i for i, b in enumerate(self.blocks)
                       if i == len(self.blocks) - 1 or self.blocks[i + 1].strides > 1]


def variable_specs(arch):
  """OrderedDict name -> VarSpec (Keras layouts) for the backbone + head conv."""
  s = collections.OrderedDict()
  mn = arch.model_name
  s['%s/stem/conv2d/kernel' % mn] = VarSpec((3, 3, 3, arch.stem_filters), 'conv', True)
  _bn(s, '%s/stem/batch_normalization' % mn, arch.stem_filters)
  for b in arch.blocks:
    sc = '%s/%s' % (mn, b.name)
    convs = iter(['conv2d', 'conv2d_1'])
    bns = iter(['tpu_batch_normalization', 'tpu_batch_normalization_1', 'tpu_batch_normalization_2'])
    if b.conv_type == 0:
      if b.expand_ratio != 1:
        s['%s/%s/kernel' % (sc, next(convs))] = VarSpec((1, 1, b.input_filters, b.mid_filters), 'conv', True)
        _bn(s, '%s/%s' % (sc, next(bns)), b.mid_filters)
      s['%s/depthwise_conv2d/depthwise_kernel' % sc] = VarSpec(
          (b.kernel_size, b.kernel_size, b.mid_filters, 1), 'dw', True)
      _bn(s, '%s/%s' % (sc, next(bns)), b.mid_filters)
    else:
      if b.expand_ratio != 1:
        s['%s/%s/kernel' % (sc, next(convs))] = VarSpec(
            (b.kernel_size, b.kernel_size, b.input_filters, b.mid_filters), 'conv', True)
        _bn(s, '%s/%s' % (sc, next(bns)), b.mid_filters)
    if b.se_filters:
      s['%s/se/conv2d/kernel' % sc] = VarSpec((1, 1, b.mid_filters, b.se_filters), 'conv', True)
      s['%s/se/conv2d/bias' % sc] = VarSpec((b.se_filters,), 'se_bias', True)
      s['%s/se/conv2d_1/kernel' % sc] = VarSpec((1, 1, b.se_filters, b.mid_filters), 'conv', True)
      s['%s/se/conv2d_1/bias' % sc] = VarSpec((b.mid_filters,), 'se_bias', True)
    pk = b.kernel_size if (b.conv_type == 1 and b.expand_ratio == 1) else 1
    s['%s/%s/kernel' % (sc, next(convs))] = VarSpec((pk, pk, b.mid_filters, b.output_filters), 'conv', True)
    last_bn = '%s/%s' % (sc, next(bns))
    _bn(s, last_bn, b.output_filters)
    # synthetic init only: a small gain on the residual branch keeps 40-100 stacked blocks O(1)
    s[last_bn + '/gamma'] = VarSpec((b.output_filters,), 'gamma_res' if b.has_skip else 'gamma', True)
  s['%s/head/conv2d/kernel' % mn] = VarSpec((1, 1, arch.blocks[-1].output_filters, arch.head_filters),
                                            'conv', True)
  _bn(s, '%s/head/batch_normalization' % mn, arch.head_filters)
  return s


def count_params(arch, include_top=True):
  """Keras `model.count_params()` of the reference model: every variable above (BN moving
  statistics included) plus, with include_top, the Dense classifier (effnetv2_model_test.py:25-48)."""
  total = sum(int(np.prod(v.shape)) for v in variable_specs(arch).values())
  if include_top and arch.mconfig.num_classes:
    total += arch.head_filters * arch.mconfig.num_classes + arch.mconfig.num_classes
  return total


def synthetic_weights(arch, seed=0):
  """Seeded float32 weights keyed by variable name (no checkpoints offline)."""
  rng = np.random.default_rng(seed)
  out = collections.OrderedDict()
  for name, spec in variable_specs(arch).items():
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
    else:
      raise AssertionError(kind)
    out[name] = np.asarray(w, np.float32)
  return out


def _bn_fold(w, scope, eps):
  g, b = np.asarray(w[scope + '/gamma'], np.float64), np.asarray(w[scope + '/beta'], np.float64)
  m, v = np.asarray(w[scope + '/moving_mean'], np.float64), np.asarray(w[scope + '/moving_variance'], np.float64)
  scale = g / np.sqrt(v + eps)
  return scale, b - m * scale


class EffNetV2Model(object):
  """One network instance bound to a device, a batch size and an image size (static buffers, the
  forward pass is one CUDA graph).  There is no CPU fallback."""

  def __init__(self, model_name='efficientnetv2-s', model_config=None, include_top=False,
               weights=None, batch_size=1, image_size=None, device='cuda:0', use_cuda_graph=True,
               seed=0):
    if include_top:
      raise NotImplementedError('the classification head (pooling + Dense) is out of scope')
    if not torch.cuda.is_available():
      raise RuntimeError('EffNetV2Model needs a CUDA device; there is no CPU fallback')
    self.arch = a = EffNetV2Arch(model_name, model_config)
    self.cfg = a.cfg
    self.n = int(batch_size)
    size = image_size or a.cfg.eval.isize
    self.image_size = utils.parse_image_size(size)
    self.device = torch.device(device)
    self.use_cuda_graph = use_cuda_graph
    if weights is None:
      weights = synthetic_weights(a, seed)
    elif isinstance(weights, str):
      data = np.load(weights)
      weights = {k: np.asarray(data[k], np.float32) for k in variable_specs(a)}
    self.endpoints = {}
    self._ops, self.op_info, self._keep, self._graph = [], [], [], None
    with torch.cuda.device(self.device):
      self._build(weights)

  # ---- lowering -----------------------------------------------------------------------------
  def _dev(self, arr, dtype):
    t = torch.as_tensor(np.ascontiguousarray(arr)).to(dtype).to(self.device).contiguous()
    self._keep.append(t)
    return t

  def _add(self, name, fn, kind, nbytes=0, flops=0):
    self._ops.append((name, fn))
    self.op_info.append({'name': name, 'kind': kind, 'bytes': int(nbytes), 'flops': int(flops)})

  def _build(self, w):
    a, n, act, eps = self.arch, self.n, self.arch.act, self.arch.bn_eps
    f16, f32 = torch.float16, torch.float32
    mn = a.model_name
    h, wd = self.image_size
    buf = lambda shape, dt=f16: torch.empty(shape, dtype=dt, device=self.device)
    self.input = buf((n, h, wd, 3), f32)
    for c in [a.stem_filters, a.head_filters] + [v for b in a.blocks for v in
                                                  (b.input_filters, b.mid_filters, b.output_filters)]:
      if c % 8:
        raise ValueError('channel count %d is not a multiple of 8' % c)

    def conv_w(name, scope_bn):
      """Conv2D kernel [kh,kw,Cin,Cout] with its BN folded -> ([taps, Cout, Cin] fp16, bias fp32)."""
      s, sh = _bn_fold(w, scope_bn, eps)
      k = np.asarray(w[name], np.float64) * s
      kh, kw, cin, cout = k.shape
      return self._dev(k.transpose(0, 1, 3, 2).reshape(kh * kw, cout, cin), f16), self._dev(sh, f32)

    # stem: conv3x3 s2 3 -> C + BN + act (Stem :409-432)
    s, sh = _bn_fold(w, '%s/stem/batch_normalization' % mn, eps)
    ks = np.asarray(w['%s/stem/conv2d/kernel' % mn], np.float64) * s
    stem_w, stem_b = self._dev(ks.reshape(27, a.stem_filters), f16), self._dev(sh, f32)
    h, wd = -(-h // 2), -(-wd // 2)
    x = buf((n, h, wd, a.stem_filters))
    self._add('stem', lambda x=x: ops.stem_conv(self.input, x, stem_w, stem_b, act), 'stem',
              nbytes=self.input.numel() * 4 + x.numel() * 2, flops=2 * 27 * x.numel())
    self.endpoints['stem'] = x

    max_mid = max(b.mid_filters for b in a.blocks)
    se_acc = [torch.zeros((n, max_mid), dtype=torch.int64, device=self.device) for _ in range(2)]
    se_index = 0
    if any(b.se_filters for b in a.blocks):
      self._add('se_clear', lambda t=se_acc[0]: t.zero_(), 'memset')
    red = 0
    for bi, b in enumerate(a.blocks):
      sc = '%s/%s' % (mn, b.name)
      x_in, s_ = x, b.strides
      ho, wo = -(-h // s_), -(-wd // s_)
      res = x_in if b.has_skip else None
      y = buf((n, ho, wo, b.output_filters))
      convs = iter(['conv2d', 'conv2d_1'])
      bns = iter(['tpu_batch_normalization', 'tpu_batch_normalization_1', 'tpu_batch_normalization_2'])
      if b.conv_type == 1:
        if b.se_filters:
          raise NotImplementedError('Fused-MBConv with SE (no registered model has it)')
        if b.expand_ratio != 1:
          ew, eb = conv_w('%s/%s/kernel' % (sc, next(convs)), '%s/%s' % (sc, next(bns)))
          mid = buf((n, ho, wo, b.mid_filters))
          self._add(b.name + '/expand_kxk',
                    lambda x_in=x_in, ew=ew, eb=eb, mid=mid, b=b:
                    ops.conv2d(x_in, ew, eb, mid, act, b.kernel_size, b.strides), 'conv_tc',
                    nbytes=2 * (x_in.numel() + mid.numel() + ew.numel()),
                    flops=2 * b.kernel_size**2 * b.input_filters * mid.numel())
          pw, pb = conv_w('%s/%s/kernel' % (sc, next(convs)), '%s/%s' % (sc, next(bns)))
          self._add(b.name + '/project',
                    lambda mid=mid, pw=pw, pb=pb, y=y, res=res:
                    ops.pointwise_conv(mid, pw[0], pb, y, utils.ACT_NONE, residual=res),
                    'pointwise_tc', nbytes=2 * (mid.numel() + y.numel() * (2 if res is not None else 1)),
                    flops=2 * b.mid_filters * y.numel())
        else:   # ONE k x k conv + BN + act (+ skip)   (:355-364, :401-402)
          pw, pb = conv_w('%s/%s/kernel' % (sc, next(convs)), '%s/%s' % (sc, next(bns)))
          self._add(b.name + '/conv_kxk',
                    lambda x_in=x_in, pw=pw, pb=pb, y=y, res=res, b=b:
                    ops.conv2d(x_in, pw, pb, y, act, b.kernel_size, b.strides, residual=res),
                    'conv_tc', nbytes=2 * (x_in.numel() + y.numel() * (2 if res is not None else 1)),
                    flops=2 * b.kernel_size**2 * b.input_filters * y.numel())
      else:
        mid = x_in
        if b.expand_ratio != 1:
          ew, eb = conv_w('%s/%s/kernel' % (sc, next(convs)), '%s/%s' % (sc, next(bns)))
          mid = buf((n, h, wd, b.mid_filters))
          self._add(b.name + '/expand',
                    lambda x_in=x_in, ew=ew, eb=eb, mid=mid: ops.pointwise_conv(x_in, ew[0], eb, mid, act),
                    'pointwise_tc', nbytes=2 * (x_in.numel() + mid.numel()),
                    flops=2 * b.input_filters * mid.numel())
        s, sh = _bn_fold(w, '%s/%s' % (sc, next(bns)), eps)
        kd = np.asarray(w[sc + '/depthwise_conv2d/depthwise_kernel'], np.float64)[..., 0] * s
        dw_w, dw_b = self._dev(kd.reshape(b.kernel_size**2, -1), f32), self._dev(sh, f32)   # fp32 taps
        dwo = buf((n, ho, wo, b.mid_filters))
        partial = next_zero = None
        if b.se_filters:
          partial = se_acc[se_index % 2].view(-1)[:n * b.mid_filters].view(n, b.mid_filters)
          next_zero = se_acc[(se_index + 1) % 2]
          se_index += 1
        self._add(b.name + '/dw',
                  lambda mid=mid, dwo=dwo, dw_w=dw_w, dw_b=dw_b, partial=partial, b=b:
                  ops.depthwise_conv(mid, dwo, dw_w, dw_b, act, b.kernel_size, b.strides, partial),
                  'depthwise', nbytes=2 * (mid.numel() + dwo.numel()),
                  flops=2 * b.kernel_size**2 * dwo.numel())
        s, sh = _bn_fold(w, '%s/%s' % (sc, next(bns)), eps)
        kp = np.asarray(w['%s/%s/kernel' % (sc, next(convs))], np.float64)[0, 0] * s   # [Cmid, Cout]
        proj_wt, proj_b = self._dev(kp.T, f16), self._dev(sh, f32)
        if b.se_filters:
          w1 = self._dev(np.asarray(w[sc + '/se/conv2d/kernel'], np.float64)[0, 0].T, f32)
          b1 = self._dev(w[sc + '/se/conv2d/bias'], f32)
          w2 = self._dev(np.asarray(w[sc + '/se/conv2d_1/kernel'], np.float64)[0, 0], f32)
          b2 = self._dev(w[sc + '/se/conv2d_1/bias'], f32)
          gate = buf((n, b.mid_filters), f32)
          hidden = buf((n, b.se_filters), f32)
          wt_scaled = buf((n, b.output_filters, b.mid_filters))
          inv_hw = 1.0 / float(ho * wo)
          self._add(b.name + '/se',
                    lambda partial=partial, inv_hw=inv_hw, w1=w1, b1=b1, w2=w2, b2=b2, gate=gate,
                    proj_wt=proj_wt, wt_scaled=wt_scaled, next_zero=next_zero, hidden=hidden:
                    ops.se_fc(partial, inv_hw, w1, b1, w2, b2, gate, act, proj_wt, wt_scaled,
                              next_zero, hidden), 'se_fc', nbytes=2 * wt_scaled.numel())
          self._add(b.name + '/project',
                    lambda dwo=dwo, wt_scaled=wt_scaled, proj_b=proj_b, y=y, res=res, ho=ho, wo=wo:
                    ops.pointwise_conv(dwo, wt_scaled, proj_b, y, utils.ACT_NONE, residual=res,
                                       batch=n, rows=ho * wo), 'pointwise_tc',
                    nbytes=2 * (dwo.numel() + y.numel() * (2 if res is not None else 1) + wt_scaled.numel()),
                    flops=2 * b.mid_filters * y.numel())
        else:
          self._add(b.name + '/project',
                    lambda dwo=dwo, proj_wt=proj_wt, proj_b=proj_b, y=y, res=res:
                    ops.pointwise_conv(dwo, proj_wt, proj_b, y, utils.ACT_NONE, residual=res),
                    'pointwise_tc', nbytes=2 * (dwo.numel() + y.numel() * (2 if res is not None else 1)),
                    flops=2 * b.mid_filters * y.numel())
      x, h, wd = y, ho, wo
      self.endpoints['block_%d' % bi] = y
      if bi in a.reductions:
        red += 1
        self.endpoints['reduction_%d' % red] = y
    self.endpoints['features'] = x
    hw_, hb_ = conv_w('%s/head/conv2d/kernel' % mn, '%s/head/batch_normalization' % mn)
    head = buf((n, h, wd, a.head_filters))
    self._add('head_1x1', lambda x=x, head=head: ops.pointwise_conv(x, hw_[0], hb_, head, act),
              'pointwise_tc', nbytes=2 * (x.numel() + head.numel()),
              flops=2 * a.blocks[-1].output_filters * head.numel())
    self.endpoints['head_1x1'] = head

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
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
          self._run_ops()
        self._graph = g
      self._graph.replay()

  def __call__(self, images=None, training=False, with_endpoints=False):
    """images float32 [N,H,W,3] (already scaled to [-1,1], preprocessing.py:82-83) -> the
    'head_1x1' feature map, or with_endpoints [head_1x1, reduction_1, ...] (:648-657)."""
    if training:
      raise NotImplementedError('inference only')
    if images is not None:
      t = torch.as_tensor(images)
      if tuple(t.shape) != tuple(self.input.shape):
        raise ValueError('expected input shape %s, got %s' % (tuple(self.input.shape), tuple(t.shape)))
      self.input.copy_(t.to(torch.float32), non_blocking=True)
    self.run()
    out = self.endpoints['head_1x1']
    if with_endpoints:
      return [out] + [self.endpoints['reduction_%d' % i] for i in range(1, 6)
                      if 'reduction_%d' % i in self.endpoints]
    return out


  def serve_stream(self, batches):
    """Pipelined __call__ over an iterable of host batches (float32 [N,H,W,3], ideally pinned):
    the H2D copy of batch i+1 and the D2H copy of the feature map of batch i-1 overlap the network
    of batch i (two copy streams for the two PCIe directions, device staging buffers on both
    sides).  Yields the 'head_1x1' feature map of each batch, in order, as a pinned host float16
    tensor that stays valid until two further results have been yielded."""
    with torch.cuda.device(self.device):
      if getattr(self, '_pipe', None) is None:
        head = self.endpoints['head_1x1']
        self._pipe = {
            'in': [torch.empty_like(self.input) for _ in range(2)],
            'out': [torch.empty_like(head) for _ in range(2)],
            'host': [torch.empty(tuple(head.shape), dtype=head.dtype).pin_memory() for _ in range(2)],
            'h2d': torch.cuda.Stream(device=self.device), 'd2h': torch.cuda.Stream(device=self.device),
            'ev_h2d': [torch.cuda.Event() for _ in range(2)],
            'ev_in_free': [torch.cuda.Event() for _ in range(2)],
            'ev_out': [torch.cuda.Event() for _ in range(2)],
            'ev_d2h': [torch.cuda.Event() for _ in range(2)],
        }
      p = self._pipe
      main = torch.cuda.current_stream(self.device)
      head = self.endpoints['head_1x1']
      prev = None
      for k, batch in enumerate(batches):
        s = k % 2
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
        main.wait_event(p['ev_d2h'][s])                  # result k-2 has left this staging buffer
        p['out'][s].copy_(head, non_blocking=True)
        p['ev_out'][s].record(main)
        with torch.cuda.stream(p['d2h']):
          p['d2h'].wait_event(p['ev_out'][s])
          p['host'][s].copy_(p['out'][s], non_blocking=True)
          p['ev_d2h'][s].record(p['d2h'])
        if prev is not None:
          p['ev_d2h'][prev].synchronize()
          yield p['host'][prev]
        prev = s
      if prev is not None:
        p['ev_d2h'][prev].synchronize()
        yield p['host'][prev]


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
