"""What the detector (engine.Engine) and the EfficientNet V1 / V2 classifier
(efficientnetv2/effnetv2_model.EffNetV2Model) lower the same way: the BatchNorm fold, the recorded
launch list with its per-launch accounting, its capture into a CUDA graph, and the EfficientNet
stem and MBConv blocks."""
import gc

import numpy as np
import torch

from automl_b200 import ops
from automl_b200 import utils


def capture_graph(fn, stream=None):
  """fn() captured into a new torch.cuda.CUDAGraph (on `stream`, else a side stream torch picks).

  Python's cyclic garbage collector is paused for the capture.  A dropped Engine or model lives in
  reference cycles until the collector frees it; freed during a capture, its CUDA graphs and pinned
  buffers are destroyed with CUDA calls that a global-mode capture forbids, and the capture fails at
  capture_end.  Paused, the collector frees them once the capture has ended."""
  g = torch.cuda.CUDAGraph()
  enabled = gc.isenabled()
  gc.disable()
  try:
    with torch.cuda.graph(g, stream=stream):
      fn()
  finally:
    if enabled:
      gc.enable()
  return g


def bn_fold(w, scope, eps):
  """(scale, shift) float64 for y = x*scale + shift."""
  g = np.asarray(w[scope + '/gamma'], np.float64)
  b = np.asarray(w[scope + '/beta'], np.float64)
  m = np.asarray(w[scope + '/moving_mean'], np.float64)
  v = np.asarray(w[scope + '/moving_variance'], np.float64)
  scale = g / np.sqrt(v + eps)
  return scale, b - m * scale


class LaunchList(object):
  """A static list of kernel launches bound to one device, recorded once and replayed.

  Uploaded weights stay alive in `_keep`, activation buffers are allocated once (`buffers`: name
  -> tensor), `_ops` holds (name, callable) and `op_info` the accounting of each launch.  The
  stem / MBConv lowering reads `n`, `act`, `arch.bn_eps` and `input`, which the subclass sets."""

  pw_impl = ops.PW_TCGEN05

  def __init__(self, device):
    self.device = torch.device(device)
    self._ops = []          # (name, callable)
    self.op_info = []       # parallel to _ops: kind / algorithmic bytes / flops
    self._keep = []         # keeps weight tensors alive
    self.buffers = {}       # debug / tests: name -> tensor
    self._branch = None
    self._sched_slots = None   # int32 [ops, 2]: the tile-scheduler slot of each op (_bound)

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
    if self._sched_slots is not None:
      raise RuntimeError('%s: the launch list has run; it takes no more ops' % name)
    i = len(self._ops)
    self._ops.append((name, lambda: self._bound(i, fn)))
    if branch is None:
      branch = self._branch      # set while lowering independent sub-graphs (the head towers)
    self.op_info.append({'name': name, 'kind': kind, 'bytes': int(nbytes), 'flops': int(flops),
                         'kernels': int(kernels), 'branch': branch, 'needs': list(needs or [])})

  def _bound(self, i, fn):
    """Runs op i with its scheduler-slot launch (if it makes one) on the list's slot i
    (edet_sched_bind), not on the global pool, where a slot comes back 4096 launches later.

    Op i then uses the same slot in the eager passes and in every graph that contains it, which
    is safe because one op of one list is never in flight twice: the graphs and eager passes that
    share ops are ordered on one stream (Engine: net, net+pre, bb1 and bb2 on the main
    stream; cell0 and heads+pre on the head stream, over ops the main-stream stages of the
    pipelined step do not run; forward()
    waits for a pending head stage first), and a side stream of a parallel branch forks from and
    joins back into its stream within the pass.  Lists never share slots with each other or
    with standalone ops.* launches."""
    pool = self._sched_slots
    if pool is None:
      if torch.cuda.is_current_stream_capturing():
        raise RuntimeError('a launch list must run eagerly once before it is captured')
      pool = torch.zeros(len(self._ops), 2, dtype=torch.int32, device=self.device)
      torch.cuda.synchronize(self.device)   # zero before any stream of the list uses a slot
      self._sched_slots = pool
    ops.sched_bind(pool.data_ptr() + 8 * i, 1)
    try:
      fn()
    finally:
      ops.sched_bind(None)

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

  def op_names(self):
    return [n for n, _ in self._ops]

  # ---- EfficientNet stem and MBConv blocks ---------------------------------------------------
  def _stem(self, w, scope, bn_scope, out_hw):
    """3x3 stride-2 conv + BN + act of `input` (kernel `<scope>/kernel`) into buffer 'stem'."""
    scale, shift = bn_fold(w, bn_scope, self.arch.bn_eps)
    k = np.asarray(w[scope + '/kernel'], np.float64) * scale  # [3,3,3,C]
    stem_w = self._dev(k.reshape(27, -1), torch.float16)
    stem_b = self._dev(shift, torch.float32)
    x = self._buf('stem', (self.n,) + tuple(out_hw) + (k.shape[-1],))
    inp, act = self.input, self.act
    self._add('stem', lambda: ops.stem_conv(inp, x, stem_w, stem_b, act),
              kind='stem', nbytes=4 * inp.numel() + 2 * x.numel(), flops=2 * 27 * x.numel())
    return x

  def _se_accumulators(self, blocks):
    """int64 fixed-point squeeze accumulators [n, mid] of the SE blocks: two buffers alternate
    between blocks, each block's se_fc launch clears the one the next block will accumulate into.
    One explicit clear per forward keeps the ping-pong valid for any number of SE blocks."""
    n, max_mid = self.n, max(b.mid_filters for b in blocks)
    self._se_acc = [self._buf('se_acc%d' % i, (n, max_mid), torch.int64) for i in range(2)]
    for t in self._se_acc:
      t.zero_()
    self._se_index = 0
    if any(b.se_filters for b in blocks):
      self._add('se_clear', lambda t=self._se_acc[0]: t.zero_(), kind='memset',
                nbytes=8 * n * max_mid, kernels=0)   # torch fill kernel, not one of ours

  def _mbconv(self, w, scope, b, x_in, hw, stride, fuse_front=False):
    """One MBConv block (conv_type 0) from x_in [n, h, w, Cin] at hw = (h, w): expand 1x1 ->
    depthwise (+ SE squeeze sums) -> se_fc -> project 1x1 with the SE gate folded into per-image
    weights (+ skip).  The layer names come from the block (`expand_name`, `dw_bn`, ...).
    fuse_front: expand + depthwise as one launch, the expanded map never reaches HBM.
    Returns (output buffer '<block>/out', (ho, wo))."""
    n, act, eps = self.n, self.act, self.arch.bn_eps
    f16, f32 = torch.float16, torch.float32
    k = b.kernel_size
    h, wd = hw
    mid = x_in
    exp_wt = exp_b = None
    if b.expand_name:
      s, sh = bn_fold(w, '%s/%s' % (scope, b.expand_bn), eps)
      kw = np.asarray(w['%s/%s/kernel' % (scope, b.expand_name)], np.float64)[0, 0]  # [Cin,Cmid]
      exp_wt = self._dev((kw * s).T, f16)
      exp_b = self._dev(sh, f32)
      if not fuse_front:
        mid = self._buf(b.name + '/expand', (n, h, wd, b.mid_filters))
        self._pw(b.name + '/expand', x_in, exp_wt, exp_b, mid, act)
    # depthwise
    s, sh = bn_fold(w, '%s/%s' % (scope, b.dw_bn), eps)
    kd = np.asarray(w[scope + '/depthwise_conv2d/depthwise_kernel'], np.float64)[..., 0]  # [k,k,C]
    dw_w = self._dev((kd * s).reshape(k * k, -1), f32)   # fp32 taps
    dw_b = self._dev(sh, f32)
    ho, wo = utils.same_pad(h, k, stride)[0], utils.same_pad(wd, k, stride)[0]
    dwo = self._buf(b.name + '/dw', (n, ho, wo, b.mid_filters))
    partial = None
    if b.se_filters:
      acc = self._se_acc
      partial = acc[self._se_index % 2].view(-1)[:n * b.mid_filters].view(n, b.mid_filters)
      next_zero = acc[(self._se_index + 1) % 2]
      self._se_index += 1
    se_bytes = 8 * partial.numel() if partial is not None else 0
    if fuse_front:
      self._add(b.name + '/expand_dw',
                lambda: ops.mbconv_expand_dw(x_in, exp_wt, exp_b, dw_w, dw_b, dwo, act, k, stride,
                                             partial),
                kind='mbconv_expand_dw',
                nbytes=2 * n * (h * wd * b.input_filters + ho * wo * b.mid_filters)
                + 2 * b.mid_filters * (b.input_filters + k**2) + se_bytes,
                flops=2 * n * b.mid_filters * (h * wd * b.input_filters + k**2 * ho * wo))
    else:
      self._add(b.name + '/dw',
                lambda: ops.depthwise_conv(mid, dwo, dw_w, dw_b, act, k, stride, partial),
                kind='depthwise_k%ds%d' % (k, stride),
                nbytes=2 * n * b.mid_filters * (h * wd + ho * wo) + 2 * k**2 * b.mid_filters + se_bytes,
                flops=2 * k**2 * n * b.mid_filters * ho * wo)
    # project (+SE folded into per-image weights, + skip)
    s, sh = bn_fold(w, '%s/%s' % (scope, b.project_bn), eps)
    kp = np.asarray(w['%s/%s/kernel' % (scope, b.project_name)], np.float64)[0, 0]  # [Cmid,Cout]
    proj_wt = self._dev((kp * s).T, f16)  # [Cout, Cmid]
    proj_b = self._dev(sh, f32)
    y = self._buf(b.name + '/out', (n, ho, wo, b.output_filters))
    res = x_in if b.has_skip else None
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
                lambda: ops.se_fc(partial, inv_hw, w1, b1, w2, b2, gate, act, proj_wt, wt_scaled,
                                  next_zero, hidden),
                kind='se_fc', nbytes=8 * partial.numel() + 2 * proj_wt.numel() + 2 * wt_scaled.numel(),
                kernels=2)
      self._pw(b.name + '/project', dwo, wt_scaled, proj_b, y, utils.ACT_NONE, residual=res,
               batch=n, rows=ho * wo)
    else:
      self._pw(b.name + '/project', dwo, proj_wt, proj_b, y, utils.ACT_NONE, residual=res)
    return y, (ho, wo)
