"""Lowers a resolved EfficientDet architecture to a static list of kernel launches on one H100.

  * folds inference BatchNorm into the conv weights (reference utils.py:244-326, eps 1e-3),
    casts weights to fp16 / biases to fp32 and uploads them once;
  * allocates every activation buffer once (NHWC fp16, static shapes);
  * records the launch list (stem -> MBConv blocks -> extra levels -> BiFPN cells -> heads ->
    pre-NMS -> NMS) and replays it as CUDA graphs: the whole network as one graph for forward(),
    one pipelined step of three overlapping stages on three streams for run(postprocess=True)
    (backbone of step i+1 over feature network + heads + pre-NMS of step i over NMS of step i;
    Engine._run_pipelined).

The launch list mirrors the call structure of efficientdet_arch.efficientdet
(/root/reference/efficientdet/efficientdet_arch.py:547-577) and inference.det_post_process
(inference.py:233-271).  PyTorch is used for device memory, streams and graph capture only.
"""
import contextlib
import math
import os

import numpy as np
import torch

from automl_b200 import anchors as anchors_lib
from automl_b200 import ops
from automl_b200 import utils
from automl_b200.arch import DetArch
from automl_b200.lowering import LaunchList, bn_fold, capture_graph


def _round_up(x, m):
  return (x + m - 1) // m * m


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


class Engine(LaunchList):
  """One network instance bound to one device, one batch size and one image size."""

  def __init__(self, config, weights, batch_size, device='cuda:0', pw_impl=ops.PW_TCGEN05,
               use_cuda_graph=True, image_id_base=0, fuse_mbconv_front=False,
               fuse_sepconv=True, pipeline=True, fuse_class_argmax=True):
    if not torch.cuda.is_available():
      raise RuntimeError('automl_b200.Engine needs a CUDA device; there is no CPU fallback')
    self.config = config
    self.arch = a = DetArch(config)
    self.n = int(batch_size)
    super().__init__(device)
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
    self._cell0_end = None
    self._branch_streams = {}
    self.launches_per_forward = 0
    with torch.cuda.device(self.device):
      self._build(weights)

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

    # -- stem and MBConv blocks ----------------------------------------------------------------
    bb = a.backbone_name
    cur = self._stem(w, bb + '/stem/conv2d', bb + '/stem/tpu_batch_normalization', a.level_hw[1])
    cur_hw = a.level_hw[1]
    self._se_accumulators(a.blocks)
    feats = {}
    for b in a.blocks:
      scope = '%s/%s' % (bb, b.name)
      check_c(b.input_filters, scope); check_c(b.mid_filters, scope); check_c(b.output_filters, scope)
      h, wd = cur_hw
      # fuse_mbconv_front: blocks whose expanded map is large and whose depthwise is 3x3 stride 2
      # run the fused front half (expand in registers, depthwise from shared memory; the expanded map
      # never reaches HBM).  Off by default since round 2: with the three-team pointwise kernel
      # and the TMA-tiled depthwise the separate pair is 1 % faster on the D0 step (4.165 vs
      # 4.204 ms) although it moves 4x the bytes -- the fused kernel serialises TMA -> MMA ->
      # epilogue -> depthwise inside a CTA at two CTAs per SM (DESIGN.md section 4).
      fuse_front = bool(self.fuse_mbconv_front and b.expand_name and b.kernel_size == 3 and
                        b.stride == 2 and b.input_filters <= 64 and h * wd >= 1600)
      cur, cur_hw = self._mbconv(w, scope, b, cur, cur_hw, b.stride, fuse_front)
      if b.reduction:
        feats[b.reduction] = cur

    self.num_backbone_ops = len(self._ops)
    # first op that writes a backbone feature the feature network reads (see run())
    first = next((b for b in a.blocks if b.reduction and b.reduction >= a.config.min_level), None)
    self._bb_split = (self.op_names().index(first.name + '/project') if first else
                      self.num_backbone_ops)

    # -- feature network --------------------------------------------------------------------
    F = a.fpn_filters
    check_c(F, 'fpn_num_filters')

    def resample_conv(r, src):
      """1x1 conv(+bias)+BN of a resample op at the SOURCE resolution, or, when
      conv_after_downsample moves it behind the max-pool (a.conv_after_pool), max-pool then
      conv at the TARGET resolution: the result then enters the node as a 'same' input."""
      kw = np.asarray(w[r.scope + '/conv2d/kernel'], np.float64)[0, 0]  # [Cin,F]
      cb = np.asarray(w[r.scope + '/conv2d/bias'], np.float64)
      if a.config.apply_bn_for_resampling:
        s, sh = bn_fold(w, r.scope + '/bn', eps)
      else:
        s, sh = np.ones(F), np.zeros(F)
      wt = self._dev((kw * s).T, f16)
      bias = self._dev(cb * s + sh, f32)
      # a detached branch ('~' prefix): only the op that consumes `out` joins it
      branch = '~' + r.scope
      hh, ww = r.in_hw
      if a.conv_after_pool(r):
        check_c(r.in_channels, r.scope)
        hh, ww = r.out_hw
        pooled = self._buf(r.scope + '/pool', (n, hh, ww, r.in_channels))
        self._add(r.scope + '/pool',
                  lambda src=src, pooled=pooled, r=r: ops.max_pool(src, pooled, r.pool[:2], r.pool[2:]),
                  kind='max_pool', nbytes=2 * (src.numel() + pooled.numel()), branch=branch)
        src = pooled
      out = self._buf(r.scope + '/conv', (n, hh, ww, F))
      self._pw(r.scope + '/conv', src, wt, bias, out, utils.ACT_NONE, branch=branch)
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
    level_needs = {}   # pyramid index -> detached branch that writes the level
    for r in a.extra_levels:
      src = pyramid[r.src]
      needs = list(level_needs.get(r.src, []))
      if r.has_conv:
        src = hoisted[r.scope]
        needs.append('~' + r.scope)
      if r.mode == 'same' or a.conv_after_pool(r):
        # 1x1 maps cannot shrink further: the reference only applies the (optional) 1x1 conv
        # (efficientdet_arch.py:116-117), so the level aliases its source; with
        # conv_after_downsample the hoisted op already pooled before its conv.
        level_needs[len(pyramid)] = needs
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
    # conv_bn_act_pattern: the activation moves from the fusion to the pointwise epilogue
    node_pre_act, node_post_act = (utils.ACT_NONE, act) if a.conv_bn_act_pattern else (act, utils.ACT_NONE)
    for ci, cell in enumerate(a.cells):
      cell_feats = list(pyramid)
      for node in cell['nodes']:
        specs = []
        cw = None     # per-channel weights [inputs, F] of the channel_* methods
        wsm = lambda i, node=node: w['%s/WSM%s' % (node.scope, '' if i == 0 else '_%d' % i)]
        # fusion weights (efficientdet_arch.py:439-468), float32 like the reference
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
        elif a.fpn_weight_method == 'channel_fastattn':
          # per channel: relu(w_i) / (sum_j relu(w_j) + 1e-4), summed in input order like add_n
          ew = [np.maximum(np.asarray(wsm(i), np.float32), np.float32(0)) for i in range(len(node.inputs))]
          tot = ew[0]
          for e in ew[1:]:
            tot = tot + e
          tot = tot + np.float32(0.0001)
          cw = np.stack([e / tot for e in ew])
        elif a.fpn_weight_method == 'channel_attn':
          ev = np.stack([np.asarray(wsm(i), np.float32) for i in range(len(node.inputs))])
          ex = np.exp(ev - ev.max(axis=0))       # softmax over the inputs, per channel
          cw = ex / ex.sum(axis=0)
        else:
          raise NotImplementedError('fpn_weight_method %s' % a.fpn_weight_method)
        if cw is not None:
          fw = [1.0] * len(node.inputs)          # ignored by the per-channel entry point
          cw = self._dev(cw.astype(np.float32), f32)
        needs = []
        for r, wgt in zip(node.inputs, fw):
          src = cell_feats[r.src]
          mode, pool = r.mode, r.pool
          if r.has_conv:
            if r.scope in hoisted:
              src = hoisted[r.scope]
            else:
              src = resample_conv(r, src)
            needs.append('~' + r.scope)
            if a.conv_after_pool(r):
              mode, pool = 'same', None
          elif ci == 0:
            needs.extend(level_needs.get(r.src, []))
          specs.append((src, mode_code[mode], pool, float(wgt)))
        op = node.op_scope
        dw_w = self._dev(np.asarray(w[op + '/conv/depthwise_kernel'], np.float64)[..., 0].reshape(9, F), f32)
        s, sh = bn_fold(w, op + '/bn', eps)
        kp = np.asarray(w[op + '/conv/pointwise_kernel'], np.float64)[0, 0]
        cb = 0.0 if a.conv_bn_act_pattern else np.asarray(w[op + '/conv/bias'], np.float64)
        pw_wt = self._dev((kp * s).T, f16)
        pw_b = self._dev(cb * s + sh, f32)
        hh, ww = node.hw
        out = self._buf(node.scope + '/out', (n, hh, ww, F))
        in_bytes = 2 * sum(sp[0].numel() for sp in specs)
        tmp = self._buf(node.scope + '/fused_dw', (n, hh, ww, F))
        self._add(node.scope + '/fuse_dw',
                  lambda specs=specs, dw_w=dw_w, tmp=tmp, cw=cw:
                  ops.fuse_dw(specs, dw_w, tmp, node_pre_act, channel_weights=cw),
                  kind='bifpn_fuse_dw',
                  nbytes=in_bytes + 2 * tmp.numel() + 18 * F + (cw.numel() * 4 if cw is not None else 0),
                  flops=2 * 9 * tmp.numel(), needs=needs)
        self._pw(node.scope + '/pw', tmp, pw_wt, pw_b, out, node_post_act)
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
    towers = ((('class', A * C, self.ld_cls), ('box', A * 4, self.ld_box))
              if a.has_detection else ())
    for net, pred_c, ld in towers:
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
          s, sh = bn_fold(w, '%s/%s-%d-bn-%d' % (scope, net, i, level), eps)
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
    self._build_segmentation(w)
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
    cls_l = [self.cls_out[l] for l in a.levels if l in self.cls_out]
    box_l = [self.box_out[l] for l in a.levels if l in self.box_out]
    level_hw = [a.level_hw[l] for l in a.levels]
    self._pre_ops, self._nms_ops, self._pre_ops_full = [], [], []
    # no object_detection head: no pre-NMS / NMS buffers or launches (detect() raises)
    for sidx in range(2 if a.has_detection else 0):
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
    # The head and NMS streams keep the default priority.  Measured on a B200 D0 step: a
    # high-priority head stage pushes whole waves of the next backbone out (4.04 ms), equal
    # priorities let it fill the slots the backbone leaves (3.89 ms).
    self._nms_stream = torch.cuda.Stream(device=self.device)
    self._head_stream = torch.cuda.Stream(device=self.device)
    self._head_capture_stream = torch.cuda.Stream(device=self.device)
    self._ev_bb = torch.cuda.Event()
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
    if a.has_detection:
      self._add('pre_nms', self._pre_ops[0], kind='pre_nms', nbytes=pre_bytes)
      self._add('nms', self._nms_ops[0], kind='nms_v5', nbytes=28 * n * K, kernels=2)
    self.launches_per_forward = sum(i['kernels'] for i in self.op_info)

  def _build_segmentation(self, w):
    """SegmentationHead (tf2/efficientdet_keras.py:694-706) after the last BiFPN cell, as one
    graph branch: every stage is one edet_conv2d_transpose with BN folded into its weights, whose
    two K sources are the previous stage's output and the BiFPN level of the reference's concat
    (the concat is never written).  self.seg_out: fp16 [N, 2H_min, 2W_min, round8(C)]."""
    a, n = self.arch, self.n
    self.seg_out = None
    if not a.seg_stages:
      return
    f16, f32 = torch.float16, torch.float32
    F = a.fpn_filters
    self._branch = 'segmentation_head'
    x, skip = self.fpn_feats[a.max_level], None
    for st in a.seg_stages:
      kernel = np.asarray(w[st.kernel_scope + '/kernel'], np.float64)   # [3, 3, out, in]
      if st.bn_scope:
        scale, bias = bn_fold(w, st.bn_scope, a.bn_eps)
        act = self.act
      else:
        scale, bias = None, np.asarray(w[st.kernel_scope + '/bias'], np.float64)
        act = utils.ACT_NONE
      cout = st.out_channels
      wt = self._dev(ops.conv_transpose_weights(kernel, F, scale), f16)
      b = self._dev(bias, f32)
      oh, ow = st.out_hw
      y = self._buf(st.kernel_scope, (n, oh, ow, _round_up(cout, 8)))
      ih, iw = st.in_hw
      self._add(st.kernel_scope,
                lambda x=x, skip=skip, wt=wt, b=b, y=y, act=act, cout=cout:
                ops.conv2d_transpose(x, wt, b, y, act, cout, a1=skip),
                kind='conv_transpose_tc',
                nbytes=2 * n * (ih * iw * st.in_channels + oh * ow * y.shape[-1]) + 2 * wt.numel(),
                flops=18 * n * ih * iw * st.in_channels * cout)
      x, skip = y, (self.fpn_feats[st.skip_level] if st.skip_level is not None else None)
    self.seg_out = x
    self._branch = None

  # ---- execution ------------------------------------------------------------------------------
  def _run_ops(self, upto=None, parallel_branches=True, start=0):
    """Runs ops [start, upto) of the launch list on the current stream; ops tagged with a branch
    run on side streams forked from / joined back into it (parallel graph branches when
    captured)."""
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
        st = self._branch_streams.get(br)
        if st is None:
          st = self._branch_streams[br] = torch.cuda.Stream(device=self.device)
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
      self._graph[key] = capture_graph(fn, capture_stream)
    return self._graph[key]

  def run(self, postprocess=True, after_nms=None, after_heads=None):
    """Enqueues one forward from self.input.

    postprocess=False: network only, on the current stream (writes every head output).
    postprocess=True : one pipelined step (_run_pipelined): backbone on the current stream,
      feature network + heads + pre-NMS on the engine's head stream, NMS (and `after_nms(dets)`,
      e.g. the all-gather / D2H copy) on its NMS stream, so consecutive steps overlap
      (pipeline=False: network + pre-NMS as one graph on the current stream, only the NMS overlaps
      the next step).  The class logits are not stored on this path (fuse_class_argmax).  Call
      wait_detections() (or detect()) before reading `self.detections` from the current stream.

      after_heads(seg_out), with the segmentation head only: called right after the step's head
      stage, on the stream that ran it (the head stream; pipeline=False: the current stream), to
      enqueue work that reads this step's segmentation logits, e.g. the masks.  The step's NMS and
      after_nms, and any later reader of the head outputs, are ordered after it; the next step's
      head stage, which rewrites seg_out, runs after it on the same stream.
    """
    if postprocess and not self.arch.has_detection:
      raise ValueError('post-processing needs the object_detection head; config.heads = %s'
                       % (self.arch.heads,))
    if after_heads is not None and (self.seg_out is None or not postprocess):
      raise ValueError('after_heads needs the segmentation head and postprocess=True; '
                       'config.heads = %s' % (self.arch.heads,))
    if not postprocess:
      self._logits_current = True
      if self._head_pending:   # a pipelined step may still be reading / writing the head buffers
        torch.cuda.current_stream(self.device).wait_event(self._ev_pre[self._cur])
      if self.use_cuda_graph:
        self._graph_for('net', lambda: self._run_ops(self.num_network_ops)).replay()
      else:
        self._run_ops(self.num_network_ops)
      return
    sidx = self._step % 2
    ring = self._step % 4
    self._step += 1
    self._logits_current = not self.fuse_class_argmax
    main = torch.cuda.current_stream(self.device)
    if self.pipeline:
      self._run_pipelined(sidx, main, after_nms, ring, after_heads)
    else:
      if self._nms_pending[sidx]:
        main.wait_event(self._ev_nms[sidx])      # the NMS that last read this buffer set is done
      if self.use_cuda_graph:
        self._graph_for(('net+pre', sidx), lambda: self._net_and_pre(sidx)).replay()
      else:
        self._net_and_pre(sidx)
      if after_heads is not None:
        after_heads(self.seg_out)
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

  def _run_pipelined(self, sidx, main, after_nms, ring, after_heads):
    """One step as three overlapping stages:

      main stream : stem + MBConv blocks of THIS step (throughput bound: the large maps)
      head stream : feature network + heads + pre-NMS (~100 short dependent launches, mostly on
                    small maps) -- runs under the backbone of the NEXT step
      NMS stream  : NMS-V5 (+ after_nms hook)

    The only tensors the two halves share are the backbone features P3..P5.  The head stage of
    step i is enqueued right away and overlaps the early backbone of step i+1.  No copy of P3..P5
    is needed: the backbone is cut in two graphs (bb1, bb2) at the first launch that writes one of
    them (blocks_4/project in D0, 1.6 ms into the backbone) and the main stream waits there for the
    first BiFPN cell of the previous step (cell0) -- their only reader -- which by then has long
    finished."""
    split, nb = self._bb_split, self.num_backbone_ops
    if self.use_cuda_graph and (self._graph is None or ('heads+pre', sidx) not in self._graph):
      # One eager forward (kernel attributes, module loading), then the captures -- which execute
      # nothing -- so the partial graphs are never run out of order: bb2 alone would add the SE
      # sums of its first block onto a stale accumulator.
      if self._graph is None or 'bb1' not in self._graph:
        self._run_ops(self.num_network_ops)
        for sx in (0, 1):
          (self._pre_ops_full[sx] if self._pre_ops_full else self._pre_ops[sx])()
    self._replay('bb1', lambda: self._run_ops(split))
    if self._head_pending:
      main.wait_event(self._ev_head)          # previous step's first BiFPN cell has read P3..P5
    self._replay('bb2', lambda: self._run_ops(nb, start=split))
    self._ev_bb.record(main)
    self._enqueue_heads(sidx, after_heads)
    self._enqueue_nms(sidx, after_nms, ring)

  def _enqueue_heads(self, sidx, after_heads):
    nb = self.num_backbone_ops
    c0 = self._cell0_end if self._cell0_end is not None else nb
    hs = self._head_stream
    with torch.cuda.stream(hs):
      hs.wait_event(self._ev_bb)
      if self._nms_pending[sidx]:
        hs.wait_event(self._ev_nms[sidx])      # the NMS that last read this buffer set is done
      # first BiFPN cell (+ extra levels): the only reader of P3..P5
      self._replay('cell0', lambda: self._run_ops(c0, start=nb), self._head_capture_stream)
      self._ev_head.record(hs)
      self._replay(('heads+pre', sidx), lambda: self._net_and_pre(sidx, start=c0),
                   self._head_capture_stream)
      if after_heads is not None:     # outside the graphs: it changes with every request
        after_heads(self.seg_out)
      self._ev_pre[sidx].record(hs)
    self._head_pending = True

  @contextlib.contextmanager
  def _class_head_into(self, sidx):
    """Inside: the fused class head (fuse_class_argmax) writes scores / classes into
    post-processing set `sidx` instead of logits; sidx None: logits."""
    self._fused_target = self._post[sidx] if sidx is not None and self.fuse_class_argmax else None
    try:
      yield
    finally:
      self._fused_target = None

  def _net_and_pre(self, sidx, start=0):
    """Ops [start, num_network_ops) with the class head writing into post-processing set `sidx`,
    then that set's pre-NMS."""
    with self._class_head_into(sidx):
      self._run_ops(self.num_network_ops, start=start)
    self._pre_ops[sidx]()

  def wait_detections(self):
    """Makes the current stream wait for the NMS (and after_nms hook) of the latest step."""
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

  @property
  def seg_logits(self):
    """fp16 [N, 2H_min, 2W_min, seg_num_classes] view of the segmentation head's output (written
    by every forward / run; None without the head)."""
    if self.seg_out is None:
      return None
    return self.seg_out[..., :self.arch.config.seg_num_classes]

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
    if not self.arch.has_detection:
      raise ValueError('pre-NMS needs the object_detection head; config.heads = %s'
                       % (self.arch.heads,))
    with torch.cuda.device(self.device):
      main = torch.cuda.current_stream(self.device)
      if self._logits_current:
        if self._nms_pending[self._cur]:
          main.wait_event(self._ev_nms[self._cur])   # the NMS that last read this buffer set is done
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
    # postprocess: time the launches run(postprocess=True) makes
    with self._class_head_into(0 if postprocess else None):
      return self._profile_ops(iters, upto)

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
