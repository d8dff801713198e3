"""Lowers a resolved EfficientDet architecture to a static list of kernel launches on one H100.

  * folds inference BatchNorm into the conv weights (reference utils.py:244-326, eps 1e-3),
    casts weights to fp16 / biases to fp32 and uploads them once;
  * allocates every activation buffer once (NHWC fp16, static shapes);
  * records the launch list (stem -> MBConv blocks -> extra levels -> BiFPN cells -> heads ->
    pre-NMS -> NMS) and replays it as CUDA graphs: the whole network as one graph for forward(),
    three overlapping stages on three streams for run(postprocess=True) (backbone of step i+1 over
    feature network + heads + pre-NMS of step i over NMS of step i; Engine._run_pipelined).

The launch list mirrors the call structure of efficientdet_arch.efficientdet
(/root/reference/efficientdet/efficientdet_arch.py:547-577) and inference.det_post_process
(inference.py:233-271).  PyTorch is used for device memory, streams and graph capture only.
"""
import math
import os

import numpy as np
import torch

from automl_b200 import anchors as anchors_lib
from automl_b200 import ops
from automl_b200 import utils
from automl_b200.arch import DetArch


def _round_up(x, m):
  return (x + m - 1) // m * m


def _bn_fold(w, scope, eps):
  """(scale, shift) float64 for y = x*scale + shift."""
  g = np.asarray(w[scope + '/gamma'], np.float64)
  b = np.asarray(w[scope + '/beta'], np.float64)
  m = np.asarray(w[scope + '/moving_mean'], np.float64)
  v = np.asarray(w[scope + '/moving_variance'], np.float64)
  scale = g / np.sqrt(v + eps)
  return scale, b - m * scale


def nms_v5_params(nms_configs):
  """(iou_thresh, score_thresh, tf_sigma) as postprocess.nms passes them to
  NonMaxSuppressionV5 (tf2/postprocess.py:175-199)."""
  method = nms_configs['method']
  if method == 'hard' or not method:
    sigma = 0.0
    iou_thresh = nms_configs['iou_thresh'] or 0.5
    score_thresh = nms_configs['score_thresh'] or float('-inf')
  elif method == 'gaussian':
    sigma = nms_configs['sigma'] or 0.5
    iou_thresh = 0.5
    score_thresh = nms_configs['score_thresh'] or 0.001
  else:
    raise ValueError('Inference has invalid nms method {}'.format(method))
  return iou_thresh, score_thresh, sigma / 2


class Engine(object):
  """One network instance bound to one device, one batch size and one image size."""

  def __init__(self, config, weights, batch_size, device='cuda:0', pw_impl=ops.PW_TCGEN05,
               use_cuda_graph=True, image_id_base=0, fuse_mbconv_front=False,
               fuse_sepconv=True, pipeline=True, defer_heads=False,
               fuse_class_argmax=True):
    if not torch.cuda.is_available():
      raise RuntimeError('automl_b200.Engine needs a CUDA device; there is no CPU fallback')
    self.config = config
    self.arch = a = DetArch(config)
    self.n = int(batch_size)
    self.device = torch.device(device)
    self.pw_impl = pw_impl
    self.use_cuda_graph = use_cuda_graph
    self.image_id_base = image_id_base
    if os.environ.get('EDET_FUSE_FRONT'):     # A/B switch for scripts / bench runs
      fuse_mbconv_front = os.environ['EDET_FUSE_FRONT'] != '0'
    self.fuse_mbconv_front = fuse_mbconv_front
    self.fuse_sepconv = fuse_sepconv              # head tower layers: dw + pw in one kernel
    # pipeline: run(postprocess=True) overlaps the backbone of step i+1 (main stream) with the
    # feature network + heads + pre-NMS of step i (head stream) and the NMS of step i (NMS stream)
    if os.environ.get('EDET_PIPELINE'):        # A/B switch for scripts / bench runs
      pipeline = os.environ['EDET_PIPELINE'] != '0'
    self.pipeline = pipeline
    if os.environ.get('EDET_DEFER_HEADS'):
      defer_heads = os.environ['EDET_DEFER_HEADS'] != '0'
    self.defer_heads = bool(defer_heads and pipeline)   # see _run_pipelined
    self._deferred = None
    # run(postprocess=True): the class-predict 1x1 conv computes max / arg-max / sigmoid over the
    # classes in its epilogue (edet_class_argmax) and never writes the [N,H,W,810] logits;
    # forward() always writes them.  Bit-identical detections either way.
    if os.environ.get('EDET_FUSE_ARGMAX'):
      fuse_class_argmax = os.environ['EDET_FUSE_ARGMAX'] != '0'
    self.fuse_class_argmax = fuse_class_argmax
    self._fused_target = None   # post-processing buffer set the fused class head writes to
    self._logits_current = False   # the head output buffers hold the latest pass (forward())
    self.act = utils.activation_code(a.act_type)
    self._graph = None
    self._bb_split = None
    self._cell0_end = None
    self._ops = []          # (name, callable)
    self.op_info = []       # parallel to _ops: kind / algorithmic bytes / flops
    self._branch = None
    self._branch_streams = {}
    self.buffers = {}       # debug / tests: name -> tensor
    self._keep = []         # keeps weight tensors alive
    self.launches_per_forward = 0
    with torch.cuda.device(self.device):
      self._build(weights)

  # ---- helpers --------------------------------------------------------------------------
  def _dev(self, arr, dtype):
    t = torch.as_tensor(np.ascontiguousarray(arr)).to(dtype).to(self.device).contiguous()
    self._keep.append(t)
    return t

  def _buf(self, name, shape, dtype=torch.float16):
    t = torch.empty(shape, dtype=dtype, device=self.device)
    self.buffers[name] = t
    return t

  def _add(self, name, fn, kind='other', nbytes=0, flops=0, kernels=1, branch=None, needs=None):
    """kind groups launches of the same kernel; nbytes / flops are the ALGORITHMIC HBM bytes
    and floating-point operations of the launch (SURVEY.md 8d formulas), used by bench.py."""
    self._ops.append((name, fn))
    if branch is None:
      branch = self._branch      # set while lowering independent sub-graphs (the head towers)
    self.op_info.append({'name': name, 'kind': kind, 'bytes': int(nbytes), 'flops': int(flops),
                         'kernels': int(kernels), 'branch': branch, 'needs': list(needs or [])})

  def _pw(self, name, a, wt, bias, out, act, residual=None, batch=1, rows=None, nout=None,
          branch=None):
    if rows is None:
      rows = a.numel() // (a.shape[-1] * batch)
    impl = self.pw_impl
    k = wt.shape[-1]
    n_out = nout if nout is not None else wt.shape[-2]
    m = rows * batch
    wbatch = wt.shape[0] if wt.dim() == 3 else 1
    nbytes = 2 * (m * k + m * n_out * (2 if residual is not None else 1)) + 2 * wbatch * n_out * k
    self._add(name, lambda: ops.pointwise_conv(a, wt, bias, out, act, residual=residual,
                                               rows=rows, batch=batch, nout=nout, impl=impl),
              kind='pointwise_tc' if impl == ops.PW_TCGEN05 else 'pointwise_simt',
              nbytes=nbytes, flops=2 * m * k * n_out, branch=branch)

  # ---- network lowering -------------------------------------------------------------------
  def _build(self, w):
    a, n, act = self.arch, self.n, self.act
    eps = a.bn_eps
    f16, f32 = torch.float16, torch.float32
    H, W = a.image_hw
    self.input = self._buf('input', (n, H, W, 3), f32)

    def check_c(c, what):
      if c % 8:
        raise NotImplementedError('%s has %d channels; the kernels need multiples of 8' % (what, c))

    # -- stem ---------------------------------------------------------------------------------
    bb = a.backbone_name
    scale, shift = _bn_fold(w, bb + '/stem/tpu_batch_normalization', eps)
    k = np.asarray(w[bb + '/stem/conv2d/kernel'], np.float64) * scale  # [3,3,3,C]
    stem_w = self._dev(k.reshape(27, -1), f16)
    stem_b = self._dev(shift, f32)
    h, wd = a.level_hw[1]
    x = self._buf('stem', (n, h, wd, a.stem_filters))
    inp = self.input
    self._add('stem', lambda inp=inp, x=x: ops.stem_conv(inp, x, stem_w, stem_b, act),
              kind='stem', nbytes=12 * n * H * W + 2 * n * h * wd * a.stem_filters,
              flops=2 * 27 * n * h * wd * a.stem_filters)
    cur, cur_hw = x, (h, wd)

    # -- MBConv blocks ----------------------------------------------------------------------
    feats = {}
    max_mid = max(b.mid_filters for b in a.blocks)
    se_acc = [self._buf('se_acc%d' % i, (n, max_mid), torch.int64) for i in range(2)]
    for t in se_acc:
      t.zero_()
    se_index = 0
    if any(b.se_filters for b in a.blocks):
      # one explicit clear per forward keeps the ping-pong valid for any number of SE blocks
      self._add('se_clear', lambda t=se_acc[0]: t.zero_(), kind='memset', nbytes=8 * n * max_mid,
                kernels=0)   # torch fill kernel, not one of ours
    for b in a.blocks:
      scope = '%s/%s' % (bb, b.name)
      check_c(b.input_filters, scope); check_c(b.mid_filters, scope); check_c(b.output_filters, scope)
      h, wd = cur_hw
      x_in = cur
      mid = x_in
      # fuse_mbconv_front: blocks whose expanded map is large and whose depthwise is 3x3 stride 2
      # run the fused front half (expand in registers, depthwise from shared memory; the expanded map
      # never reaches HBM).  Off by default since round 2: with the three-team pointwise kernel
      # and the TMA-tiled depthwise the separate pair is 1 % faster on the D0 step (4.165 vs
      # 4.204 ms) although it moves 4x the bytes -- the fused kernel serialises TMA -> MMA ->
      # epilogue -> depthwise inside a CTA at two CTAs per SM (DESIGN.md section 4).
      fuse_front = (self.fuse_mbconv_front and b.expand_name and b.kernel_size == 3 and
                    b.stride == 2 and b.input_filters <= 64 and h * wd >= 1600)
      exp_wt = exp_b = None
      if b.expand_name:
        s, sh = _bn_fold(w, '%s/%s' % (scope, b.expand_bn), eps)
        kw = np.asarray(w['%s/%s/kernel' % (scope, b.expand_name)], np.float64)[0, 0]  # [Cin,Cmid]
        exp_wt = self._dev((kw * s).T, f16)
        exp_b = self._dev(sh, f32)
        if not fuse_front:
          mid = self._buf(b.name + '/expand', (n, h, wd, b.mid_filters))
          self._pw(b.name + '/expand', x_in, exp_wt, exp_b, mid, act)
      # depthwise
      s, sh = _bn_fold(w, '%s/%s' % (scope, b.dw_bn), eps)
      kd = np.asarray(w[scope + '/depthwise_conv2d/depthwise_kernel'], np.float64)[..., 0]  # [k,k,C]
      dw_w = self._dev((kd * s).reshape(b.kernel_size * b.kernel_size, -1), f32)   # fp32 taps
      dw_b = self._dev(sh, f32)
      ho, wo = utils.same_pad(h, b.kernel_size, b.stride)[0], utils.same_pad(wd, b.kernel_size, b.stride)[0]
      dwo = self._buf(b.name + '/dw', (n, ho, wo, b.mid_filters))
      partial = None
      if b.se_filters:
        # int64 fixed-point squeeze accumulator [n, mid]; two buffers alternate between blocks,
        # each block's se_fc launch clears the one the next block will accumulate into.
        partial = se_acc[se_index % 2].view(-1)[:n * b.mid_filters].view(n, b.mid_filters)
        next_zero = se_acc[(se_index + 1) % 2]
        se_index += 1
      if fuse_front:
        self._add(b.name + '/expand_dw',
                  lambda x_in=x_in, exp_wt=exp_wt, exp_b=exp_b, dwo=dwo, dw_w=dw_w, dw_b=dw_b,
                  partial=partial, b=b:
                  ops.mbconv_expand_dw(x_in, exp_wt, exp_b, dw_w, dw_b, dwo, act, b.kernel_size,
                                       b.stride, partial),
                  kind='mbconv_expand_dw',
                  nbytes=2 * n * (h * wd * b.input_filters + ho * wo * b.mid_filters)
                  + 2 * b.mid_filters * (b.input_filters + b.kernel_size**2)
                  + (8 * partial.numel() if partial is not None else 0),
                  flops=2 * n * b.mid_filters * (h * wd * b.input_filters + b.kernel_size**2 * ho * wo))
      else:
        self._add(b.name + '/dw',
                  lambda mid=mid, dwo=dwo, dw_w=dw_w, dw_b=dw_b, partial=partial, b=b:
                  ops.depthwise_conv(mid, dwo, dw_w, dw_b, act, b.kernel_size, b.stride, partial),
                  kind='depthwise_k%ds%d' % (b.kernel_size, b.stride),
                  nbytes=2 * n * b.mid_filters * (h * wd + ho * wo) + 2 * b.kernel_size**2 * b.mid_filters
                  + (8 * partial.numel() if partial is not None else 0),
                  flops=2 * b.kernel_size**2 * n * b.mid_filters * ho * wo)
      # project (+SE folded into per-image weights, + skip)
      s, sh = _bn_fold(w, '%s/%s' % (scope, b.project_bn), eps)
      kp = np.asarray(w['%s/%s/kernel' % (scope, b.project_name)], np.float64)[0, 0]  # [Cmid,Cout]
      proj_wt = self._dev((kp * s).T, f16)  # [Cout, Cmid]
      proj_b = self._dev(sh, f32)
      y = self._buf(b.name + '/out', (n, ho, wo, b.output_filters))
      res = x_in if b.has_skip else None
      if b.reduction and b.reduction >= a.config.min_level and self._bb_split is None:
        # first op that writes a backbone feature the feature network reads (see run())
        self._bb_split = len(self._ops) + (1 if b.se_filters else 0)
      if b.se_filters:
        w1 = self._dev(np.asarray(w[scope + '/se/conv2d/kernel'], np.float64)[0, 0].T, f32)   # [se,C]
        b1 = self._dev(w[scope + '/se/conv2d/bias'], f32)
        w2 = self._dev(np.asarray(w[scope + '/se/conv2d_1/kernel'], np.float64)[0, 0], f32)  # [se,C]
        b2 = self._dev(w[scope + '/se/conv2d_1/bias'], f32)
        gate = self._buf(b.name + '/se_gate', (n, b.mid_filters), f32)
        hidden = self._buf(b.name + '/se_hidden', (n, b.se_filters), f32)
        wt_scaled = self._buf(b.name + '/proj_w', (n, b.output_filters, b.mid_filters))
        inv_hw = 1.0 / float(ho * wo)
        self._add(b.name + '/se',
                  lambda partial=partial, inv_hw=inv_hw, w1=w1, b1=b1, w2=w2, b2=b2, gate=gate,
                  proj_wt=proj_wt, wt_scaled=wt_scaled, next_zero=next_zero, hidden=hidden:
                  ops.se_fc(partial, inv_hw, w1, b1, w2, b2, gate, act, proj_wt, wt_scaled,
                            next_zero, hidden),
                  kind='se_fc', nbytes=8 * partial.numel() + 2 * proj_wt.numel() + 2 * wt_scaled.numel(),
                  kernels=2)
        self._pw(b.name + '/project', dwo, wt_scaled, proj_b, y, utils.ACT_NONE, residual=res,
                 batch=n, rows=ho * wo)
      else:
        self._pw(b.name + '/project', dwo, proj_wt, proj_b, y, utils.ACT_NONE, residual=res)
      cur, cur_hw = y, (ho, wo)
      if b.reduction:
        feats[b.reduction] = y

    self.num_backbone_ops = len(self._ops)
    if self._bb_split is None:
      self._bb_split = self.num_backbone_ops
    if self.defer_heads:
      # the held-back head stage reads copies of P3..P5 (see _run_pipelined); torch's copy kernel
      for level in sorted(feats):
        if level >= a.config.min_level:
          src = feats[level]
          dst = self._buf('P%d_copy' % level, tuple(src.shape))
          self._add('feat_copy/P%d' % level, lambda src=src, dst=dst: dst.copy_(src),
                    kind='memcpy', nbytes=4 * src.numel(), kernels=0)
          feats[level] = dst
    self._heads_start = len(self._ops)

    # -- feature network --------------------------------------------------------------------
    F = a.fpn_filters
    check_c(F, 'fpn_num_filters')

    def resample_conv(r, src):
      """1x1 conv(+bias)+BN of a resample op at the SOURCE resolution (conv_after_downsample
      is False for every registered model)."""
      kw = np.asarray(w[r.scope + '/conv2d/kernel'], np.float64)[0, 0]  # [Cin,F]
      cb = np.asarray(w[r.scope + '/conv2d/bias'], np.float64)
      if a.config.apply_bn_for_resampling:
        s, sh = _bn_fold(w, r.scope + '/bn', eps)
      else:
        s, sh = np.ones(F), np.zeros(F)
      wt = self._dev((kw * s).T, f16)
      bias = self._dev(cb * s + sh, f32)
      out = self._buf(r.scope + '/conv', (n, r.in_hw[0], r.in_hw[1], F))
      # a detached branch ('~' prefix): only the op that consumes `out` joins it
      self._pw(r.scope + '/conv', src, wt, bias, out, utils.ACT_NONE, branch='~' + r.scope)
      return out

    pyramid = []
    for level, _ in a.pyramid_in:
      if level in feats:
        pyramid.append(feats[level])
    # The channel-matching 1x1 convs of the backbone features (P6 creation and the first cell)
    # only depend on the backbone: launch them all now, each on its own branch, so they overlap
    # each other and the start of the BiFPN chain.
    hoisted = {}
    for r in a.extra_levels:
      if r.has_conv:
        hoisted[r.scope] = resample_conv(r, pyramid[r.src])
    if a.cells:
      for node in a.cells[0]['nodes']:
        for r in node.inputs:
          if r.has_conv and r.src < len(pyramid):
            hoisted[r.scope] = resample_conv(r, pyramid[r.src])
    for r in a.extra_levels:
      src = pyramid[r.src]
      needs = []
      if r.has_conv:
        src = hoisted[r.scope]
        needs = ['~' + r.scope]
      if r.mode == 'same':
        # 1x1 maps cannot shrink further: the reference only applies the (optional) 1x1 conv
        # (efficientdet_arch.py:116-117), so the level aliases its source.
        pyramid.append(src)
        continue
      if r.mode != 'down':
        raise NotImplementedError('extra level that is an upsample')
      out = self._buf(r.scope, (n, r.out_hw[0], r.out_hw[1], F))
      self._add(r.scope + '/pool',
                lambda src=src, out=out, r=r: ops.max_pool(src, out, r.pool[:2], r.pool[2:]),
                kind='max_pool', nbytes=2 * (src.numel() + out.numel()), needs=needs)
      pyramid.append(out)

    mode_code = {'same': ops.RS_SAME, 'up': ops.RS_UP, 'down': ops.RS_DOWN}
    # the fused separable-conv kernel covers D0-D2 widths and the swish / relu6 networks; wider
    # feature networks keep the fuse_dw + pointwise pair
    fuse_sep = (self.fuse_sepconv and F <= ops.SEPCONV_MAX_C and
                act in (utils.ACT_SWISH, utils.ACT_RELU6))
    for ci, cell in enumerate(a.cells):
      cell_feats = list(pyramid)
      for node in cell['nodes']:
        specs = []
        # fusion weights (efficientdet_arch.py:439-447), float32 like the reference
        if a.fpn_weight_method == 'fastattn':
          ew = [np.maximum(np.float32(w['%s/WSM%s' % (node.scope, '' if i == 0 else '_%d' % i)]),
                           np.float32(0)) for i in range(len(node.inputs))]
          tot = np.float32(sum(ew)) + np.float32(0.0001)
          fw = [np.float32(e) / tot for e in ew]
        elif a.fpn_weight_method == 'attn':
          ev = np.asarray([np.float32(w['%s/WSM%s' % (node.scope, '' if i == 0 else '_%d' % i)])
                           for i in range(len(node.inputs))], np.float32)
          ex = np.exp(ev - ev.max())
          fw = list(ex / ex.sum())
        elif a.fpn_weight_method == 'sum':
          fw = [1.0] * len(node.inputs)
        else:
          raise NotImplementedError('fpn_weight_method %s' % a.fpn_weight_method)
        needs = []
        for r, wgt in zip(node.inputs, fw):
          src = cell_feats[r.src]
          if r.has_conv:
            if r.scope in hoisted:
              src = hoisted[r.scope]
            else:
              src = resample_conv(r, src)
            needs.append('~' + r.scope)
          specs.append((src, mode_code[r.mode], r.pool, float(wgt)))
        op = node.op_scope
        dw_w = self._dev(np.asarray(w[op + '/conv/depthwise_kernel'], np.float64)[..., 0].reshape(9, F), f32)
        s, sh = _bn_fold(w, op + '/bn', eps)
        kp = np.asarray(w[op + '/conv/pointwise_kernel'], np.float64)[0, 0]
        cb = np.asarray(w[op + '/conv/bias'], np.float64)
        pw_wt = self._dev((kp * s).T, f16)
        pw_b = self._dev(cb * s + sh, f32)
        hh, ww = node.hw
        out = self._buf(node.scope + '/out', (n, hh, ww, F))
        in_bytes = 2 * sum(sp[0].numel() for sp in specs)
        tmp = self._buf(node.scope + '/fused_dw', (n, hh, ww, F))
        self._add(node.scope + '/fuse_dw',
                  lambda specs=specs, dw_w=dw_w, tmp=tmp: ops.fuse_dw(specs, dw_w, tmp, act),
                  kind='bifpn_fuse_dw', nbytes=in_bytes + 2 * tmp.numel() + 18 * F,
                  flops=2 * 9 * tmp.numel(), needs=needs)
        self._pw(node.scope + '/pw', tmp, pw_wt, pw_b, out, utils.ACT_NONE)
        cell_feats.append(out)
      pyramid = [cell_feats[cell['out_index'][l]] for l in a.levels]
      if ci == 0:
        self._cell0_end = len(self._ops)   # nothing after this launch reads a backbone feature
    self.fpn_feats = dict(zip(a.levels, pyramid))

    # -- heads ----------------------------------------------------------------------------------
    A, C = a.num_anchors, a.num_classes
    self.ld_cls, self.ld_box = _round_up(A * C, 8), _round_up(A * 4, 8)
    self.cls_out, self.box_out = {}, {}
    nms_cfg = a.config.nms_configs
    nms_cfg = nms_cfg.as_dict() if hasattr(nms_cfg, 'as_dict') else dict(nms_cfg)
    self.fuse_class_argmax = bool(self.fuse_class_argmax and not int(nms_cfg.get('max_nms_inputs', 0) or 0)
                                  and C <= ops.CLASS_ARGMAX_COLS and self.pw_impl == ops.PW_TCGEN05)
    anchor_begin = 0
    for net, pred_c, ld in (('class', A * C, self.ld_cls), ('box', A * 4, self.ld_box)):
      scope = '%s_net' % net
      dws, pws, pbs = [], [], []
      for i in range(a.head_repeats):
        name = '%s/%s-%d' % (scope, net, i)
        dws.append(self._dev(np.asarray(w[name + '/depthwise_kernel'], np.float64)[..., 0].reshape(9, F), f32))
        pws.append(np.asarray(w[name + '/pointwise_kernel'], np.float64)[0, 0])
        pbs.append(np.asarray(w[name + '/bias'], np.float64))
      name = '%s/%s-predict' % (scope, net)
      pred_dw = self._dev(np.asarray(w[name + '/depthwise_kernel'], np.float64)[..., 0].reshape(9, F), f32)
      pred_wt = self._dev(np.asarray(w[name + '/pointwise_kernel'], np.float64)[0, 0].T, f16)  # [pred_c, F]
      pred_b = self._dev(w[name + '/bias'], f32)
      pad_wt = pad_b = None
      if net == 'class' and self.fuse_class_argmax:
        # one anchor per 96-row block: rows a*96 + c; pad rows: zero weights, -inf bias
        pcols = ops.CLASS_ARGMAX_COLS
        kp = np.asarray(w[name + '/pointwise_kernel'], np.float64)[0, 0].T.reshape(A, C, F)
        wpad = np.zeros((A, pcols, F), np.float64)
        wpad[:, :C] = kp
        bpad = np.full((A, pcols), -np.inf, np.float32)
        bpad[:, :C] = np.asarray(w[name + '/bias'], np.float32).reshape(A, C)
        pad_wt = self._dev(wpad.reshape(A * pcols, F), f16)
        pad_b = self._dev(bpad.reshape(-1), f32)
      for level in a.levels:
        # every (tower, level) chain is independent: it becomes a parallel branch of the graph
        self._branch = '%s/l%d' % (scope, level)
        hh, ww = a.level_hw[level]
        x = self.fpn_feats[level]
        t = self._buf('%s/l%d/t' % (scope, level), (n, hh, ww, F))
        ping = self._buf('%s/l%d/a' % (scope, level), (n, hh, ww, F))
        pong = self._buf('%s/l%d/b' % (scope, level), (n, hh, ww, F))
        for i in range(a.head_repeats):
          s, sh = _bn_fold(w, '%s/%s-%d-bn-%d' % (scope, net, i, level), eps)
          wt = self._dev((pws[i] * s).T, f16)
          bias = self._dev(pbs[i] * s + sh, f32)
          y = ping if i % 2 == 0 else pong
          if fuse_sep and self.fuse_sepconv:
            self._add('%s/l%d/sep%d' % (scope, level, i),
                      lambda x=x, dwk=dws[i], wt=wt, bias=bias, y=y:
                      ops.sepconv([(x, ops.RS_SAME, None, 1.0)], utils.ACT_NONE, dwk, wt, bias, y, act),
                      kind='sepconv_tc', nbytes=4 * y.numel() + 18 * F + 2 * F * F,
                      flops=2 * (9 + F) * y.numel())
          else:
            self._add('%s/l%d/dw%d' % (scope, level, i),
                      lambda x=x, t=t, dwk=dws[i]: ops.depthwise_conv(x, t, dwk, None, utils.ACT_NONE, 3, 1),
                      kind='depthwise_k3s1', nbytes=4 * t.numel() + 18 * F, flops=18 * t.numel())
            self._pw('%s/l%d/pw%d' % (scope, level, i), t, wt, bias, y, act)
          x = y
        out = self._buf('%s/l%d/out' % (scope, level), (n, hh, ww, ld))
        out.zero_()
        self._add('%s/l%d/dwp' % (scope, level),
                  lambda x=x, t=t, pred_dw=pred_dw: ops.depthwise_conv(x, t, pred_dw, None, utils.ACT_NONE, 3, 1),
                  kind='depthwise_k3s1', nbytes=4 * t.numel() + 18 * F, flops=18 * t.numel())
        if pad_wt is None:
          self._pw('%s/l%d/predict' % (scope, level), t, pred_wt, pred_b, out, utils.ACT_NONE,
                   nout=pred_c)
        else:
          def predict(t=t, out=out, begin=anchor_begin, pad_wt=pad_wt, pad_b=pad_b,
                      pred_wt=pred_wt, pred_b=pred_b, impl=self.pw_impl, pred_c=pred_c):
            ps = self._fused_target
            if ps is not None:     # detect path: scores / classes straight into the post buffers
              ops.class_argmax(t, pad_wt, pad_b, ps['scores'], ps['classes'], begin, A)
            else:
              ops.pointwise_conv(t, pred_wt, pred_b, out, utils.ACT_NONE, rows=t.numel() // F,
                                 batch=1, nout=pred_c, impl=impl)
          m = n * hh * ww
          self._add('%s/l%d/predict' % (scope, level), predict, kind='pointwise_tc',
                    nbytes=2 * m * F + 8 * m * A + 2 * pad_wt.numel(),
                    flops=2 * m * F * pad_wt.shape[0])
          anchor_begin += hh * ww * A
        (self.cls_out if net == 'class' else self.box_out)[level] = out
    self._branch = None
    self.num_network_ops = len(self._ops)

    # -- post-processing ----------------------------------------------------------------------
    p = a.config
    self.anchors = anchors_lib.Anchors(p.min_level, p.max_level, p.num_scales,
                                       list(p.aspect_ratios), p.anchor_scale, p.image_size)
    anc = self._dev(self.anchors.boxes, f32)
    self.total_anchors = K = self.anchors.boxes.shape[0]
    # max_nms_inputs > 0: NMS sees the top-k (anchor, class) pairs instead of one arg-max class
    # per anchor (tf2/postprocess.py:88-102)
    self.max_nms_inputs = topk = int(nms_cfg.get('max_nms_inputs', 0) or 0)
    if topk > 0:
      K = topk
    iou_t, score_t, tf_sigma = nms_v5_params(nms_cfg)
    self.max_output_size = int(nms_cfg['max_output_size'])
    # Two sets of post-processing buffers: NMS of step i runs on its own stream while the
    # network of step i+1 (which writes the OTHER set) already runs on the main stream.
    self._post = []
    cls_l = [self.cls_out[l] for l in a.levels]
    box_l = [self.box_out[l] for l in a.levels]
    level_hw = [a.level_hw[l] for l in a.levels]
    self._pre_ops, self._nms_ops, self._pre_ops_full = [], [], []
    for sidx in range(2):
      ps = {
          'boxes': self._buf('boxes%d' % sidx, (n, K, 4), f32),
          'scores': self._buf('scores%d' % sidx, (n, K), f32),
          'classes': self._buf('classes%d' % sidx, (n, K), torch.int32),
          'detections': self._buf('detections%d' % sidx, (n, self.max_output_size, 7), f32),
          'sel_index': self._buf('sel_index%d' % sidx, (n, self.max_output_size), torch.int32),
          'valid': self._buf('valid%d' % sidx, (n,), torch.int32),
          'work': self._buf('nms_work%d' % sidx, (ops.nms_work_bytes(n, K),), torch.uint8),
          # per set: the NMS of step i (own stream) may still read its scales while the caller
          # already stages the scales of step i+1
          'image_scales': self._buf('image_scales%d' % sidx, (n,), f32),
      }
      ps['image_scales'].fill_(1.0)
      self._post.append(ps)
      if topk > 0:
        ps['indices'] = self._buf('indices%d' % sidx, (n, K), torch.int32)
        self._pre_ops.append(lambda ps=ps: ops.pre_nms_topk(
            cls_l, box_l, level_hw, A, C, anc, ps['boxes'], ps['scores'], ps['classes'], ps['indices']))
      else:
        full = lambda ps=ps: ops.pre_nms(cls_l, box_l, level_hw, A, C, anc,
                                         ps['boxes'], ps['scores'], ps['classes'])
        self._pre_ops_full.append(full)
        if self.fuse_class_argmax:    # boxes only: the fused class head wrote scores / classes
          self._pre_ops.append(lambda ps=ps: ops.pre_nms(None, box_l, level_hw, A, C, anc,
                                                         ps['boxes'], None, None))
        else:
          self._pre_ops.append(full)
      self._nms_ops.append(lambda ps=ps: ops.nms_v5(
          ps['boxes'], ps['scores'], ps['classes'], ps['image_scales'], self.image_id_base,
          self.max_output_size, iou_t, score_t, tf_sigma, (float(H), float(W)),
          ps['detections'], ps['sel_index'], ps['valid'], ps['work']))
    self._cur = 0
    self._step = 0
    # image scales of the steps in flight: the caller writes entry step % 4 before run(); the NMS
    # stage copies it into its buffer set on the NMS stream (so staging step i+2 never races the
    # NMS of step i, which uses the same set and may still be queued)
    self._scales_ring = [self._buf('image_scales_ring%d' % i, (n,), f32) for i in range(4)]
    for t in self._scales_ring:
      t.fill_(1.0)
    # Stream priorities of the head and NMS stages (A/B switches).  Measured on the D0 step: a
    # high-priority head stage pushes whole waves of the next backbone out (4.04 ms), equal
    # priorities let it fill the slots the backbone leaves (3.90 ms).
    self._head_priority = -1 if os.environ.get('EDET_HEAD_PRIO', '0') != '0' else 0
    self._nms_priority = -1 if os.environ.get('EDET_NMS_PRIO', '0') != '0' else 0
    self._nms_stream = torch.cuda.Stream(device=self.device, priority=self._nms_priority)
    self._head_stream = torch.cuda.Stream(device=self.device, priority=self._head_priority)
    self._head_capture_stream = torch.cuda.Stream(device=self.device, priority=self._head_priority)
    self._ev_bb = torch.cuda.Event()
    self._ev_early = torch.cuda.Event()
    self._ev_head = torch.cuda.Event()
    self._head_pending = False
    self._ev_pre = [torch.cuda.Event() for _ in range(2)]
    self._ev_nms = [torch.cuda.Event() for _ in range(2)]
    self._nms_pending = [False, False]
    # op list entries (set 0) for profiling / accounting
    if self.fuse_class_argmax and topk == 0:   # boxes only: box logits in, decoded boxes out
      pre_bytes = 2 * sum(t.numel() for t in box_l) + 16 * n * K + 16 * K
    else:
      pre_bytes = 2 * sum(t.numel() for t in cls_l + box_l) + 24 * n * K + 16 * K
    self._add('pre_nms', self._pre_ops[0], kind='pre_nms', nbytes=pre_bytes)
    self._add('nms', self._nms_ops[0], kind='nms_v5', nbytes=28 * n * K, kernels=2)
    self.launches_per_forward = sum(i['kernels'] for i in self.op_info)

  # ---- execution ------------------------------------------------------------------------------
  def _run_ops(self, upto=None, parallel_branches=True, start=0, priority=0):
    """Runs ops [start, upto) of the launch list on the current stream; ops tagged with a branch
    run on side streams forked from / joined back into it (parallel graph branches when
    captured).  priority: CUDA priority of the side streams (the head half of a pipelined step
    runs at high priority so that its short kernels are not queued behind the next backbone)."""
    upto = len(self._ops) if upto is None else upto
    main = torch.cuda.current_stream(self.device)
    open_branches = {}
    for i in range(start, upto):
      fn = self._ops[i][1]
      br = self.op_info[i]['branch'] if parallel_branches else None
      if br is None:
        # join every open branch except the detached ('~...') ones this op does not consume
        needs = self.op_info[i]['needs']
        for name in list(open_branches):
          if not name.startswith('~') or name in needs:
            main.wait_stream(open_branches.pop(name))
        fn()
        continue
      st = open_branches.get(br)
      if st is None:
        st = self._branch_streams.get((br, priority))
        if st is None:
          st = self._branch_streams[(br, priority)] = torch.cuda.Stream(device=self.device,
                                                                        priority=priority)
        st.wait_stream(main)                   # fork
        open_branches[br] = st
      with torch.cuda.stream(st):
        fn()
    for st in open_branches.values():
      main.wait_stream(st)

  @property
  def image_scales(self):
    """float32 [N] image_scale_to_original of the NEXT run(postprocess=True): write it (on the
    current stream) before calling run() / detect().  One buffer per post-processing set, so
    staging step i+1 never races the NMS of step i."""
    return self._scales_ring[self._step % 4]

  # buffers of the most recent post-processed step
  @property
  def boxes(self):
    return self._post[self._cur]['boxes']

  @property
  def scores(self):
    return self._post[self._cur]['scores']

  @property
  def classes(self):
    return self._post[self._cur]['classes']

  @property
  def detections(self):
    return self._post[self._cur]['detections']

  @property
  def sel_index(self):
    return self._post[self._cur]['sel_index']

  @property
  def valid(self):
    return self._post[self._cur]['valid']

  def _graph_for(self, key, fn, capture_stream=None, warm=True):
    if self._graph is None:
      self._graph = {}
    if key not in self._graph:
      if warm:
        fn()                                 # warm-up outside capture (kernel attributes, modules)
      torch.cuda.synchronize(self.device)
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g, stream=capture_stream):
        fn()
      self._graph[key] = g
    return self._graph[key]

  def run(self, postprocess=True, after_nms=None):
    """Enqueues one forward from self.input.

    postprocess=False: network only, on the current stream (writes every head output).
    postprocess=True : backbone on the current stream, feature network + heads + pre-NMS on the
      engine's head stream, NMS (and `after_nms(dets)`, e.g. the all-gather / D2H copy) on its NMS
      stream, so consecutive steps overlap (pipeline=False: network + pre-NMS as one graph on the
      current stream, only the NMS overlaps the next step).  The class logits are not stored on
      this path (fuse_class_argmax).  Call wait_detections() (or detect()) before reading
      `self.detections` from the current stream.
    """
    net_upto = self.num_network_ops
    if not postprocess:
      self.flush()
      self._logits_current = True
      if self._head_pending:   # a pipelined step may still be reading / writing the head buffers
        torch.cuda.current_stream(self.device).wait_event(self._ev_pre[self._cur])
      if self.use_cuda_graph:
        self._graph_for('net', lambda: self._run_ops(net_upto)).replay()
      else:
        self._run_ops(net_upto)
      return
    sidx = self._step % 2
    ring = self._step % 4
    self._step += 1
    self._logits_current = not self.fuse_class_argmax
    main = torch.cuda.current_stream(self.device)
    if self.pipeline:
      self._run_pipelined(sidx, main, after_nms, ring)
    else:
      if self._nms_pending[sidx]:
        main.wait_event(self._ev_nms[sidx])      # the NMS that last read this buffer set is done
      def net_and_pre():
        self._fused_target = self._post[sidx] if self.fuse_class_argmax else None
        try:
          self._run_ops(net_upto)
        finally:
          self._fused_target = None
        self._pre_ops[sidx]()
      if self.use_cuda_graph:
        self._graph_for(('net+pre', sidx), net_and_pre).replay()
      else:
        net_and_pre()
      self._ev_pre[sidx].record(main)
      self._enqueue_nms(sidx, after_nms, ring)
    self._cur = sidx

  def _enqueue_nms(self, sidx, after_nms, ring):
    with torch.cuda.stream(self._nms_stream):
      self._nms_stream.wait_event(self._ev_pre[sidx])
      self._post[sidx]['image_scales'].copy_(self._scales_ring[ring], non_blocking=True)
      if self.use_cuda_graph:
        self._graph_for(('nms', sidx), self._nms_ops[sidx]).replay()
      else:
        self._nms_ops[sidx]()
      if after_nms is not None:
        after_nms(self._post[sidx]['detections'])
      self._ev_nms[sidx].record(self._nms_stream)
    self._nms_pending[sidx] = True

  def _replay(self, key, fn, capture_stream=None):
    if self.use_cuda_graph:
      self._graph_for(key, fn, capture_stream, warm=False).replay()
    else:
      fn()

  def _run_pipelined(self, sidx, main, after_nms, ring):
    """One step as three overlapping stages:

      main stream : stem + MBConv blocks of THIS step (throughput bound: the large maps)
      head stream : feature network + heads + pre-NMS (~100 short dependent launches, mostly on
                    small maps) -- runs under the backbone of the NEXT step
      NMS stream  : NMS-V5 (+ after_nms hook)

    The only tensors the two halves share are the backbone features P3..P5.
    defer_heads=False: the head stage of step i is enqueued right away and overlaps the EARLY
      backbone of step i+1.  No copy of P3..P5 is needed: the backbone is cut in two graphs at the
      first launch that writes one of them (blocks_4/project in D0, 1.6 ms into the backbone) and
      the main stream waits there for the first BiFPN cell of the previous step -- their only
      reader -- which by then has long finished.
    defer_heads=True: the head stage of step i is held back until step i+1 has been submitted and
      starts when its early backbone is done, so that the ~100 short head launches overlap the
      LATE, small-map backbone layers (blocks_5.. in D0) instead of the bandwidth-bound first
      layers.  P3..P5 are then copied (35 MB in D0, ~12 us) at the end of the backbone, and the
      head stage reads the copies.  flush() / wait_detections() submit a held-back head stage."""
    split, nb, nbc, net_upto = self._bb_split, self.num_backbone_ops, self._heads_start, self.num_network_ops
    if self.use_cuda_graph and (self._graph is None or ('heads+pre', sidx) not in self._graph):
      # One eager forward (kernel attributes, module loading), then the captures -- which execute
      # nothing -- so the partial graphs are never run out of order: bb2 alone would add the SE
      # sums of its first block onto a stale accumulator.
      if self._graph is None or 'bb1' not in self._graph:
        self._run_ops(net_upto)
        for sx in (0, 1):
          (self._pre_ops_full[sx] if self._pre_ops_full else self._pre_ops[sx])()
    self._replay('bb1', lambda: self._run_ops(split))
    if self.defer_heads:
      self._ev_early.record(main)
      self.flush(after=self._ev_early)          # head + NMS stages of the previous step
      self._replay('bb2', lambda: self._run_ops(nb, start=split))
      if self._head_pending:
        main.wait_event(self._ev_head)          # first BiFPN cell of the previous step read the copies
      self._replay('featcopy', lambda: self._run_ops(nbc, start=nb))
      self._ev_bb.record(main)
      self._deferred = (sidx, after_nms, ring)
    else:
      if self._head_pending:
        main.wait_event(self._ev_head)          # previous step's first BiFPN cell has read P3..P5
      self._replay('bb2', lambda: self._run_ops(nbc, start=split))
      self._ev_bb.record(main)
      self._enqueue_heads(sidx, None)
      self._enqueue_nms(sidx, after_nms, ring)

  def _enqueue_heads(self, sidx, after):
    nbc, net_upto = self._heads_start, self.num_network_ops
    c0 = self._cell0_end if self._cell0_end is not None else nbc
    hs = self._head_stream
    with torch.cuda.stream(hs):
      hs.wait_event(self._ev_bb)
      if after is not None:
        hs.wait_event(after)
      if self._nms_pending[sidx]:
        hs.wait_event(self._ev_nms[sidx])      # the NMS that last read this buffer set is done
      # first BiFPN cell (+ extra levels): the only reader of P3..P5 (or of their copies)
      self._replay('cell0', lambda: self._run_ops(c0, start=nbc, priority=self._head_priority),
                   self._head_capture_stream)
      self._ev_head.record(hs)
      def heads_and_pre():
        self._fused_target = self._post[sidx] if self.fuse_class_argmax else None
        try:
          self._run_ops(net_upto, start=c0, priority=self._head_priority)
        finally:
          self._fused_target = None
        self._pre_ops[sidx]()
      self._replay(('heads+pre', sidx), heads_and_pre, self._head_capture_stream)
      self._ev_pre[sidx].record(hs)
    self._head_pending = True

  def flush(self, after=None):
    """Submits the head + NMS stages of the latest step if they are being held back
    (defer_heads); `after`: an event they additionally wait for.  No-op otherwise."""
    if self._deferred is not None:
      sidx, after_nms, ring = self._deferred
      self._deferred = None
      with torch.cuda.device(self.device):
        self._enqueue_heads(sidx, after)
        self._enqueue_nms(sidx, after_nms, ring)

  def wait_detections(self):
    """Makes the current stream wait for the NMS (and after_nms hook) of the latest step."""
    self.flush()
    torch.cuda.current_stream(self.device).wait_event(self._ev_nms[self._cur])

  def set_input(self, images):
    """images: float32 [N,H,W,3] tensor (any device) or array; copied into the static input."""
    t = torch.as_tensor(images)
    if tuple(t.shape) != tuple(self.input.shape):
      raise ValueError('expected input shape %s, got %s' % (tuple(self.input.shape), tuple(t.shape)))
    self.input.copy_(t.to(torch.float32), non_blocking=True)

  def forward(self, images=None):
    """Network only: returns (cls_outputs, box_outputs) dicts level -> fp16 views
    [N,H_l,W_l,A*C] / [N,H_l,W_l,4A] (strided views into padded buffers)."""
    with torch.cuda.device(self.device):
      if images is not None:
        self.set_input(images)
      self.run(postprocess=False)
    A, C = self.arch.num_anchors, self.arch.num_classes
    return ({l: t[..., :A * C] for l, t in self.cls_out.items()},
            {l: t[..., :A * 4] for l, t in self.box_out.items()})

  def detect(self, images=None, image_scales=None):
    """Network + post-process: float32 [N, max_output_size, 7] device tensor."""
    with torch.cuda.device(self.device):
      if images is not None:
        self.set_input(images)
      if image_scales is not None:
        self.image_scales.copy_(torch.as_tensor(image_scales, dtype=torch.float32), non_blocking=True)
      self.run(postprocess=True)
      self.wait_detections()
    return self.detections

  def pre_nms_only(self):
    """Pre-NMS (class arg-max, sigmoid, box decode) of the latest forward pass: the buffer set
    {'boxes' [N,K,4], 'scores' [N,K], 'classes' [N,K]} (for the per-class NMS path,
    automl_b200/postprocess.py).  After forward() it is computed here from the head outputs;
    after run(postprocess=True) / detect() it is what that step already produced."""
    with torch.cuda.device(self.device):
      self.flush()
      main = torch.cuda.current_stream(self.device)
      if self._logits_current:
        (self._pre_ops_full if self._pre_ops_full else self._pre_ops)[self._cur]()
      elif self._head_pending or not self.pipeline:
        main.wait_event(self._ev_pre[self._cur])
    return self._post[self._cur]

  def nms_fallback_count(self):
    """Images of the last run that needed the full-queue NMS kernel (fast path not provable)."""
    self.wait_detections()
    flags = self._post[self._cur]['work'][-4 * self.n:].view(torch.int32)
    return int(flags.sum().item())

  def op_names(self):
    return [n for n, _ in self._ops]

  def profile_ops(self, iters=3, postprocess=True):
    """Times every launch of the list individually with CUDA events on the current stream
    (eager launches, not the graph) and returns op_info rows extended with 'ms' (mean)."""
    upto = len(self._ops) if postprocess else self.num_network_ops
    self.flush()
    if postprocess and self.fuse_class_argmax:
      self._fused_target = self._post[0]       # time the launches run(postprocess=True) makes
    try:
      return self._profile_ops(iters, upto)
    finally:
      self._fused_target = None

  def _profile_ops(self, iters, upto):
    with torch.cuda.device(self.device):
      torch.cuda.synchronize()
      self._run_ops(upto, parallel_branches=False)  # warm-up
      torch.cuda.synchronize()
      acc = [0.0] * upto
      for _ in range(iters):
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(upto + 1)]
        evs[0].record()
        for i in range(upto):
          self._ops[i][1]()
          evs[i + 1].record()
        torch.cuda.synchronize()
        for i in range(upto):
          acc[i] += evs[i].elapsed_time(evs[i + 1])
    rows = []
    for i in range(upto):
      r = dict(self.op_info[i])
      r['ms'] = acc[i] / iters
      rows.append(r)
    return rows
