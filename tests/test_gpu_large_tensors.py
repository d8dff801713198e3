"""Every batch-scaled kernel on tensors past 2^31 elements, at the batches the registered models
reach: EfficientDet D6-D7x and EfficientNet-L2 at their native sizes and a batch of 32 already
hold one activation of more than 2^31 elements, D5 one of more than 2^31 fp16 bytes (the table in
crossing_batches()), so a per-image or flattened offset formed in 32-bit `int` reads or writes
another image without any error.

Each case tiles random images over the batch on the device: image i is source i % 4, except the
image that straddles element 2^31 of the largest tensor the kernel touches (source 4), the images
holding the further crossings of the pre-process cases (sources 6 and 7: byte 2^32 of the packed
input, element 2^31 of the output) and the last image (source 5), whose content appears nowhere
else.  Then:
  1. every image of the output equals the same kernel run on its source image alone at batch 1,
     bit for bit, compared on the device over the whole output (a write that wrapped onto an early
     image changes it);
  2. those batch-1 results of sources 4 and 5 are within the float64 bound (or equal to the
     oracle) of the family's own test (the references and checks are imported from it);
  3. the canary words after every output are unchanged;
  4. where the kernel adds to SE sums (int64 [N, C]), the rows of every image equal the batch-1
     rows of its source.
Each case states the bytes it allocates and skips, saying so, when the device has less free
memory than that plus MARGIN; everything is freed between cases.

  entry point (variant)         layer                                     batch  crossing tensor           peak
  stem_conv (stem_impl 0 / 1)   D7x stem @1536, 3 -> 64                   58     out 768^2 x 64            6.0 GB
  depthwise_conv k3s1 (+/- SE)  D7x blocks_0 @1536, 768^2 x 64            58     in / out 768^2 x 64       8.8 GB
  depthwise_conv k5s2 (+/- SE)  D7x blocks_11 @1536, 384^2 x 288          52     in 384^2 x 288            5.5 GB
    (both kernels of dw_impl: the tiled kernel and the register kernel)
  mbconv_expand_dw k3s1 + SE    D7x blocks_5 @1536, 48 -> 288 @ 384^2     52     out 384^2 x 288           5.2 GB
  pointwise_conv rows + resid.  D7x blocks_1 project @1536, 32 -> 32      58     out (ldo 64)              8.8 GB
  pointwise_conv per-image W    D7x blocks_1 project (SE-scaled W)        115    a / out 768^2 x 32        8.7 GB
  pointwise_conv SIMT           D7x blocks_1 project, rows, ldo 64        58     out (ldo 64)              6.6 GB
  conv2d k3s1 + residual        V2-L blocks_1 @480, 32 -> 32 @ 240^2      1167   x / out / residual       12.9 GB
  conv2d k3s2                   V2-L blocks_4 @480, 32 -> 128 @ 240^2     1167   x / out                   8.6 GB
  conv2d_transpose + skip       D7x seg stage 96^2 -> 192^2, 384 + 384    153    out 192^2 x 384           6.5 GB
  fuse_dw(_channel) same + up   D7x P3 node, 192^2 x 384 (+ P4 up)        153    out / same in             9.8 GB
  fuse_dw(_channel) down        D7x P4 node, same x 2 + P3 3x3/2 pool     153    P3 in 192^2 x 384         7.6 GB
  sepconv, TMA-staged kernel    lite0 P3 @320, 40^2 x 64 (F <= 64)        20973  in / out                  8.6 GB
  sepconv, global-load kernel   D2 P3 @768, 96^2 x 112 (64 < F <= 128)    2082   in / out                  8.6 GB
  max_pool                      D7x P6 resample, 48^2 x 384, 3x3/2        2429   in                        5.4 GB
  global_avg_pool               L2 head @800, 25^2 x 5504                 626    in                        4.3 GB
  class_argmax                  D7x P3 class head @1536, 192^2 x 384      153    a 192^2 x 384             4.7 GB
  pre_nms, stored logits        D7x P3 @1536, 192^2 x 816 (9 x 90)        73     logits                    5.2 GB
  softmax_topk k = 5            21843 classes (ImageNet-21k)              98316  logits fp32               8.6 GB
  preprocess                    D7x @1536, 1080 x 1920 sources            305    out fp32 1536^2 x 3      10.5 GB
  preprocess_ragged             D7x @1536, 2200 x 2200 sources            305    packed (147); its byte   13.1 GB
                                                                                 2^32 (295); out (303)
  cls_preprocess (bicubic)      L2 @800, 1140 x 1140 sources              1120   packed (550); its byte   13.0 GB
                                                                                 2^32 (1101); out (1118)
(peak: the batched inputs and outputs.  The batch-1 runs and the compare add at most about 0.3 GB.)

Three cases need more than 12 GiB (12.88e9 bytes), and they cannot need less.  The conv2d k3s1
case has three tensors of the same size that cross 2^31 fp16 elements: x, out and the residual.
Each pre-process case holds a float32 output past 2^31 elements (8.6 GB) and a packed uint8 input
past 2^32 bytes (4.3 GB).  The gate skips them on a device with less free memory.

The whole file takes about three minutes on an H100 80GB HBM3 (700 W).

test_checks_catch_misplaced_images feeds doctored outputs through the same check functions and
asserts that each misplacement is reported."""
import collections
import functools

import numpy as np
import pytest
import torch

from automl_b200 import utils
from automl_b200.efficientnetv2 import effnetv2_model
from oracle import efficientdet_oracle as eo
from oracle import postprocess_oracle as po
from test_gpu_memory_bound_kernels import (U, _check_se_sums, _det_arch, _dw_reference,
                                           _node_signature, _pools, dw_partials, dw_tiled)
from test_gpu_persistent_kernels import DEV, act_ref, check_close

pytestmark = pytest.mark.gpu

B31 = 1 << 31
GIB = 1 << 30
BUDGET = 13.2e9               # bytes a case may need (the ragged pre-process: out 8.6 GB, in 4.4 GB)
MARGIN = 2 * GIB              # free memory beyond a case's own need before it runs
GUARD = 1024                  # canary words after every output
SOURCES = 8                   # 0-3 tiled over the batch, 4 the boundary image, 5 the last one,
                              # 6-7 the images holding a case's further crossings
NONE, SWISH, RELU6 = utils.ACT_NONE, utils.ACT_SWISH, utils.ACT_RELU6
CANARY = {torch.float16: 7.0, torch.float32: -12345.5, torch.int64: 0x5A5A5A5A5A5A5A5A,
          torch.int32: -0x5A5A5A5A}
BITS = {torch.float16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64,
        torch.int32: torch.int32, torch.uint8: torch.uint8}


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def _cdiv(a, b):
  return -(-a // b)


# ---------------------------------------------------------------------------------------------
# the registered models' layers (no GPU)
def backbone_maps(blocks, image, stride_of):
  """[(block, input h)] of a square image: the stem halves it, each block divides by its stride."""
  h = _cdiv(image, 2)
  out = []
  for b in blocks:
    out.append((b, h))
    h = _cdiv(h, stride_of(b))
  return out


def largest_tensor(blocks, image, stem, stride_of):
  """(elements, name) of the largest activation of one image: the stem output, each expand
  output and each depthwise output.  An MBConv expand (1 x 1) keeps the block's input size; the
  k x k expand conv of a Fused-MBConv block (conv_type 1) strides, so its output has the block's
  output size."""
  best = (_cdiv(image, 2) ** 2 * stem, 'stem')
  for b, h in backbone_maps(blocks, image, stride_of):
    if b.expand_ratio != 1:
      he = _cdiv(h, stride_of(b)) if getattr(b, 'conv_type', 0) == 1 else h
      best = max(best, (he * he * b.mid_filters, '%s expand' % b.name))
    best = max(best, (_cdiv(h, stride_of(b)) ** 2 * b.mid_filters, '%s depthwise' % b.name))
  return best


TABLE_MODELS = [('efficientdet-d7x', 1536), ('efficientdet-d7', 1536), ('efficientdet-d6', 1280),
                ('efficientdet-d5', 1280), ('efficientnet-l2', 800), ('efficientdet-d4', 1024),
                ('efficientnet-b7', 600), ('efficientnetv2-xl', 512), ('efficientnetv2-l', 480),
                ('efficientnetv2-s', 384)]


def crossing_batches():
  """model -> (native size, largest per-image tensor, the batch at which it reaches 2^31
  elements): D6-D7x and L2 at a batch of 32; D5 at 32 and V2-S at 1024 pass 2^31 fp16 bytes."""
  out = {}
  for name, size in TABLE_MODELS:
    if name.startswith('efficientdet'):
      a = _det_arch(name)
      assert a.image_hw == (size, size)
      p, _ = largest_tensor(a.blocks, size, a.stem_filters, lambda b: b.stride)
    else:
      v = effnetv2_model.EffNetV2Arch(name)
      assert v.cfg.eval.isize == size
      p, _ = largest_tensor(v.blocks, size, v.stem_filters, lambda b: b.strides)
    out[name] = (size, p, _cdiv(B31, p))
  return out


def det_block(name, index):
  """(block, input h) of a detector's backbone block at the native size."""
  a = _det_arch(name)
  return backbone_maps(a.blocks, a.image_hw[0], lambda b: b.stride)[index]


def v2_block(name, index):
  v = effnetv2_model.EffNetV2Arch(name)
  return backbone_maps(v.blocks, v.cfg.eval.isize, lambda b: b.strides)[index]


def fpn_node(name, level, modes):
  """(F, node h, input hs) of the first node of `name` at `level` with signature `modes`."""
  a = _det_arch(name)
  for cell in a.cells:
    for node in cell['nodes']:
      sig, hws = _node_signature(a, node)
      if node.feat_level == level and sig == modes:
        return a.fpn_filters, node.hw[0], [hw[0] for hw in hws]
  raise AssertionError('no %s node at P%d with %s' % (name, level, modes))


SAME, UP, DOWN = ('same', None), ('up', None), ('down', (3, 3, 2, 2))

# extra: (tensor, elements per image, crossing) of the further points a case's batch passes (the
# packed uint8 inputs of the pre-process kernels past 2^32 bytes, their float32 outputs past 2^31)
Case = collections.namedtuple('Case', 'name layer crossing per_image batch need extra')


def _need(batch, *per_image_bytes):
  return batch * sum(per_image_bytes)


def _batch(per_image):
  """The smallest batch whose boundary image (the one holding element 2^31) is not the last."""
  assert B31 % per_image, 'element 2^31 falls on an image edge'
  return B31 // per_image + 2


@functools.lru_cache(maxsize=None)
def case_table():
  """name -> Case: the layer (from the architecture objects), the tensor that crosses 2^31
  elements, its elements per image, the batch and the bytes the batched tensors take."""
  cases = {}

  def add(name, layer, crossing, per_image, need_of_batch, batch=None, extra=()):
    n = batch or _batch(per_image)
    cases[name] = Case(name, layer, crossing, per_image, n, need_of_batch(n), tuple(extra))

  a = _det_arch('efficientdet-d7x')
  s, c = 768, a.stem_filters
  layer = dict(image=1536, cout=c)
  add('stem', layer, 'out', s * s * c, lambda n: _need(n, 1536 * 1536 * 12, s * s * c * 2))

  b, h = det_block('efficientdet-d7x', 0)
  layer = dict(h=h, c=b.mid_filters, k=b.kernel_size, s=b.stride, se=bool(b.se_filters))
  add('dw_k3s1', layer, 'in / out', h * h * b.mid_filters, lambda n: _need(n, 4 * h * h * b.mid_filters))
  b, h = det_block('efficientdet-d7x', 11)
  ho = _cdiv(h, b.stride)
  layer = dict(h=h, c=b.mid_filters, k=b.kernel_size, s=b.stride, se=bool(b.se_filters))
  add('dw_k5s2', layer, 'in', h * h * b.mid_filters,
      lambda n: _need(n, 2 * h * h * b.mid_filters, 2 * ho * ho * b.mid_filters))

  b, h = det_block('efficientdet-d7x', 5)
  layer = dict(h=h, cin=b.input_filters, cmid=b.mid_filters, k=b.kernel_size, s=b.stride,
               se=bool(b.se_filters))
  add('mbconv', layer, 'out', h * h * b.mid_filters,
      lambda n: _need(n, 2 * h * h * (b.input_filters + b.mid_filters)))

  b, h = det_block('efficientdet-d7x', 1)
  rows, k, nout = (h // b.stride) ** 2, b.mid_filters, b.output_filters
  layer = dict(rows=rows, k=k, nout=nout, residual=b.has_skip, se=bool(b.se_filters))
  add('pw_rows', dict(layer, ldo=2 * nout), 'out', rows * 2 * nout,
      lambda n: _need(n, 2 * rows * (k + 2 * nout + nout)))
  add('pw_image_w', dict(layer, ldo=nout), 'a / out', rows * nout,
      lambda n: _need(n, 2 * rows * (k + nout)))
  add('pw_simt', dict(layer, ldo=2 * nout), 'out', rows * 2 * nout,
      lambda n: _need(n, 2 * rows * (k + 2 * nout)))

  b, h = v2_block('efficientnetv2-l', 1)
  layer = dict(h=h, cin=b.input_filters, cout=b.output_filters, k=b.kernel_size, s=b.strides,
               residual=b.has_skip)
  add('conv_s1', layer, 'x / out / residual', h * h * b.output_filters,
      lambda n: _need(n, 2 * h * h * (b.input_filters + 2 * b.output_filters)))
  b, h = v2_block('efficientnetv2-l', 4)
  ho = _cdiv(h, b.strides)
  layer = dict(h=h, cin=b.input_filters, cout=b.mid_filters, k=b.kernel_size, s=b.strides,
               residual=False)
  add('conv_s2', layer, 'x / out', h * h * b.input_filters,
      lambda n: _need(n, 2 * (h * h * b.input_filters + ho * ho * b.mid_filters)))

  a = _det_arch('efficientdet-d7x', None, (('heads', ('object_detection', 'segmentation')),))
  st = [st for st in a.seg_stages if st.in_hw == (96, 96)][0]
  f, cout, h = a.fpn_filters, st.out_channels, st.in_hw[0]
  layer = dict(h=h, c0=f, c1=st.in_channels - f, cout=cout)
  add('convt', layer, 'out', 4 * h * h * cout,
      lambda n: _need(n, 2 * (h * h * st.in_channels + 4 * h * h * cout)))

  f, h, ins = fpn_node('efficientdet-d7x', 3, (SAME, UP))
  layer = dict(f=f, h=h, modes=(SAME, UP), ins=tuple(ins))
  add('fuse_up', layer, 'out / same input', h * h * f,
      lambda n: _need(n, 2 * f * (h * h + sum(i * i for i in ins))))
  f, h, ins = fpn_node('efficientdet-d7x', 4, (SAME, SAME, DOWN))
  layer = dict(f=f, h=h, modes=(SAME, SAME, DOWN), ins=tuple(ins))
  add('fuse_down', layer, 'P3 input', ins[2] ** 2 * f,
      lambda n: _need(n, 2 * f * (h * h + sum(i * i for i in ins))))

  # F <= 64 runs the TMA-staged kernel (sepconv_impl 0), wider inputs the global-load one
  a = _det_arch('efficientdet-lite0')
  f, h = a.fpn_filters, a.level_hw[3][0]
  add('sepconv_tma', dict(f=f, h=h), 'in / out', h * h * f, lambda n: _need(n, 4 * h * h * f))
  a = _det_arch('efficientdet-d2')
  f, h = a.fpn_filters, a.level_hw[3][0]
  add('sepconv', dict(f=f, h=h), 'in / out', h * h * f, lambda n: _need(n, 4 * h * h * f))

  a = _det_arch('efficientdet-d7x')
  c, pool, (h, _) = [p for p in _pools(a) if p[2][0] == 48][0]
  ho = _cdiv(h, pool[2])
  add('max_pool', dict(c=c, pool=pool, h=h), 'in', h * h * c,
      lambda n: _need(n, 2 * (h * h + ho * ho) * c))

  v = effnetv2_model.EffNetV2Arch('efficientnet-l2')
  h, c = _cdiv(v.cfg.eval.isize, 32), v.head_filters
  add('gap', dict(h=h, c=c), 'in', h * h * c, lambda n: _need(n, 2 * h * h * c + 4 * c))

  size = _det_arch('efficientdet-d7x').image_hw[0]
  add('preprocess', dict(size=size, src=(1080, 1920)), 'out', size * size * 3,
      lambda n: _need(n, 12 * size * size + 1080 * 1920 * 3))
  # the packed input (14.5 MB per image) passes element 2^31 first, then 2^32 bytes; the batch
  # takes the float32 output past 2^31 elements too
  packed, out = 2200 * 2200 * 3, size * size * 3
  add('preprocess_ragged', dict(size=size, src=(2200, 2200)), 'packed input', packed,
      lambda n: _need(n, 4 * out + packed), batch=_batch(out),
      extra=[('packed input, byte 2^32', packed, 1 << 32), ('out', out, B31)])

  a = _det_arch('efficientdet-d7x')
  h, na, nc = a.level_hw[3][0], a.num_anchors, a.num_classes
  ld_cls, ld_box = _cdiv(na * nc, 8) * 8, _cdiv(na * 4, 8) * 8
  add('pre_nms', dict(image=size, h=h, na=na, nc=nc, ld_cls=ld_cls, ld_box=ld_box), 'logits',
      h * h * ld_cls, lambda n: _need(n, 2 * h * h * (ld_cls + ld_box) + 24 * h * h * na))

  # L2's eval pre-process at 800: 1140 x 1140 sources pass element 2^31 of the packed input at
  # image 550 and 2^32 bytes at image 1101; the batch takes the float32 output past 2^31 elements
  v = effnetv2_model.EffNetV2Arch('efficientnet-l2')
  s2, packed = v.cfg.eval.isize, 1140 * 1140 * 3
  out = s2 * s2 * 3
  add('cls_preprocess', dict(size=s2, src=(1140, 1140)), 'packed input', packed,
      lambda n: _need(n, 4 * out + packed), batch=_batch(out),
      extra=[('packed input, byte 2^32', packed, 1 << 32), ('out', out, B31)])

  a = _det_arch('efficientdet-d7x')
  f, h, na, nc = a.fpn_filters, a.level_hw[3][0], a.num_anchors, a.num_classes
  add('class_argmax', dict(f=f, h=h, na=na, nc=nc), 'a', h * h * f,
      lambda n: _need(n, 2 * h * h * f + 8 * h * h * na))

  classes = 21843
  add('softmax_topk', dict(c=classes, k=5), 'logits', classes, lambda n: _need(n, 4 * classes + 40))
  return cases


# ---------------------------------------------------------------------------------------------
# the harness
def gate(case):
  free, _ = torch.cuda.mem_get_info()
  if free < case.need + MARGIN:
    pytest.skip('%s needs %.2f GB free (+ %.1f GB margin), the device has %.2f GB'
                % (case.name, case.need / 1e9, MARGIN / 1e9, free / 1e9))


def free_all():
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


def boundary_image(case):
  return B31 // case.per_image


def extra_images(case):
  """The images holding the further crossings of case.extra."""
  return [limit // per_image for _, per_image, limit in case.extra]


def sources(n, b, extra=()):
  """Source index of each of n images: i % 4, 4 at the boundary image b, 6, 7 at the images
  `extra`, 5 at the last."""
  src = torch.arange(n, device=DEV) % 4
  src[b] = 4
  for j, e in enumerate(extra):
    src[e] = 6 + j
  src[n - 1] = 5
  return src


class Canaried(object):
  """A device tensor of `shape` filled with `init`, followed by GUARD canary words."""

  def __init__(self, shape, dtype, init=None):
    self.numel = int(np.prod(shape))
    self.canary = CANARY[dtype]
    self.buf = torch.full((self.numel + GUARD,), self.canary, dtype=dtype, device=DEV)
    self.buf[:self.numel] = self.canary if init is None else init
    self.t = self.buf[:self.numel].view(shape)


def check_canary(out, what=''):
  torch.cuda.synchronize()
  tail = out.buf[out.numel:]
  assert bool((tail == out.canary).all()), '%s: %d canary words after the output changed' % (
      what, int((tail != out.canary).sum()))


def _bits(t):
  return t.view(BITS[t.dtype])


def mismatched_images(out, singles, src):
  """Indices of the images of out [N, ...] whose bits differ from singles[src[i]], compared on the
  device in chunks of about 256 MB."""
  n = out.shape[0]
  o = _bits(out).reshape(n, -1)
  s = _bits(singles).reshape(singles.shape[0], -1)
  step = max(1, (256 << 20) // (o.shape[1] * o.element_size()))
  bad = []
  for i in range(0, n, step):
    j = min(n, i + step)
    diff = (o[i:j] != s[src[i:j]]).any(1)
    bad += (diff.nonzero().flatten() + i).tolist()
  return bad


def check_images(out, singles, src, what=''):
  bad = mismatched_images(out, singles, src)
  assert not bad, '%s: %d images differ from their source run alone, first %s' % (
      what, len(bad), bad[:8])


def run_case(case, stacks, out_specs, launch):
  """stacks: per-image inputs [SOURCES, ...] on the device; out_specs: (per-image shape, dtype,
  init or None) per output; launch(inputs, outputs) runs the kernel on [N, ...] tensors.  Runs
  the batch of case.batch images and each source alone, checks every image, the canaries and the
  integer outputs (SE sums) row by row; returns the batch-1 outputs [SOURCES, ...] per output."""
  n, b, extra = case.batch, boundary_image(case), extra_images(case)
  assert 0 < b < n - 1 and all(0 < e < n - 1 for e in extra)
  assert len(set([b] + extra)) == 1 + len(extra) <= 1 + SOURCES - 6
  src = sources(n, b, extra)
  singles = []
  for s in range(SOURCES):
    outs = [Canaried((1,) + tuple(shape), dtype, init) for shape, dtype, init in out_specs]
    launch([t[s:s + 1] for t in stacks], [o.t for o in outs])
    for o in outs:
      check_canary(o, '%s source %d alone' % (case.name, s))
    singles.append([o.t[0].clone() for o in outs])
    del outs, o
  singles = [torch.stack([one[j] for one in singles]) for j in range(len(out_specs))]
  big = [t[src] for t in stacks]
  outs = [Canaried((n,) + tuple(shape), dtype, init) for shape, dtype, init in out_specs]
  launch(big, [o.t for o in outs])
  torch.cuda.synchronize()
  del big
  for j, o in enumerate(outs):
    check_canary(o, '%s output %d' % (case.name, j))
    check_images(o.t, singles[j], src, '%s output %d' % (case.name, j))
  del outs, o
  free_all()
  return singles


def _randn(shape, seed, dtype=torch.float16, scale=1.0):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _span_bias(n, seed):
  g = torch.Generator().manual_seed(seed)
  return torch.linspace(-26.0, 10.0, n)[torch.randperm(n, generator=g)].to(DEV)


def _cpu(t):
  return t.cpu()


@pytest.fixture(autouse=True)
def _release():
  yield
  free_all()


# ---------------------------------------------------------------------------------------------
# the cases
@pytest.mark.parametrize('impl', [0, 1], ids=['tensor_core', 'cuda_core'])
def test_stem_conv(impl):
  ops = _ops()
  case = case_table()['stem']
  gate(case)
  size, cout = case.layer['image'], case.layer['cout']
  x = _randn((SOURCES, size, size, 3), 1, torch.float32, 2.0)
  k = _randn((3, 3, 3, cout), 2, scale=0.3)
  bias = _span_bias(cout, 3)
  wt = k.reshape(27, cout).contiguous()
  ho = _cdiv(size, 2)

  def launch(ins, outs):
    ops.stem_conv(ins[0], outs[0], wt, bias, SWISH)

  ops.set_option('stem_impl', impl)
  try:
    got, = run_case(case, [x], [((ho, ho, cout), torch.float16, None)], launch)
  finally:
    ops.set_option('stem_impl', 0)
  for s in (4, 5):
    ref = eo.conv2d_same(x[s:s + 1].double().permute(0, 3, 1, 2), k.double(), stride=2)
    ref = act_ref(ref + bias.double().view(1, -1, 1, 1), SWISH).permute(0, 2, 3, 1)
    check_close(got[s:s + 1], ref, 'stem source %d' % s)


def _dw_inputs(name):
  lay = case_table()[name].layer
  h, c, k = lay['h'], lay['c'], lay['k']
  x = _randn((SOURCES, h, h, c), 10 + k)
  taps = _randn((k * k, c), 11 + k, torch.float32, 1.0 / k)
  return x, taps, _span_bias(c, 12 + k)


@pytest.mark.parametrize('se', [True, False], ids=['se', 'no_se'])
@pytest.mark.parametrize('impl', [0, 1], ids=['tiled', 'register'])
@pytest.mark.parametrize('name', ['dw_k3s1', 'dw_k5s2'])
def test_depthwise_conv(name, impl, se):
  ops = _ops()
  case = case_table()[name]
  gate(case)
  lay = case.layer
  h, c, k, st = lay['h'], lay['c'], lay['k'], lay['s']
  assert lay['se'] and dw_tiled(h, h, c, k, st), 'a tiled-kernel map of an SE block'
  x, taps, bias = _dw_inputs(name)
  ho = _cdiv(h, st)
  specs = [((ho, ho, c), torch.float16, None)]
  if se:
    specs.append(((c,), torch.int64, 0))

  def launch(ins, outs):
    ops.depthwise_conv(ins[0], outs[0], taps, bias, SWISH, k, st, outs[1] if se else None)

  ops.set_option('dw_impl', impl)
  try:
    res = run_case(case, [x], specs, launch)
  finally:
    ops.set_option('dw_impl', 0)
  tiled = impl == 0
  for s in (4, 5):
    y, z, m = _dw_reference(_cpu(x[s:s + 1]), _cpu(taps), _cpu(bias), SWISH, k, st)
    check_close(res[0][s:s + 1], y, '%s source %d' % (name, s))
    if se:
      _check_se_sums(_cpu(res[1][s:s + 1]), y, z, m, SWISH, k, dw_partials(ho, ho, c, k, st, tiled),
                     '%s source %d' % (name, s))


def test_mbconv_expand_dw():
  from test_gpu_convt_mbconv_kernels import _mbf_reference, check_mbf, mbf_partials
  ops = _ops()
  case = case_table()['mbconv']
  gate(case)
  lay = case.layer
  h, cin, cmid, k, st = lay['h'], lay['cin'], lay['cmid'], lay['k'], lay['s']
  assert lay['se']
  x = _randn((SOURCES, h, h, cin), 20)
  we = _randn((cmid, cin), 21, scale=cin**-0.5)
  be = _randn((cmid,), 22, torch.float32, 0.5)
  taps = _randn((k * k, cmid), 23, torch.float32, 1.0 / k)
  bd = _span_bias(cmid, 24)
  ho = _cdiv(h, st)

  def launch(ins, outs):
    ops.mbconv_expand_dw(ins[0], we, be, taps, bd, outs[0], SWISH, k, st, outs[1])

  got, sums = run_case(case, [x], [((ho, ho, cmid), torch.float16, None), ((cmid,), torch.int64, 0)],
                       launch)
  for s in (4, 5):
    y, z, m, flip = _mbf_reference(_cpu(x[s:s + 1]), _cpu(we), _cpu(be), _cpu(taps), _cpu(bd), SWISH,
                                   k, st)
    check_mbf(_cpu(got[s:s + 1]), y, z, m, flip, SWISH, k, 'mbconv source %d' % s)
    _check_se_sums(_cpu(sums[s:s + 1]), y, z, m + flip / ((k * k + 1) * U), SWISH, k,
                   mbf_partials(h, h, k, st), 'mbconv source %d' % s)


@pytest.mark.parametrize('plan', ['pw_rows', 'pw_image_w', 'pw_simt'])
def test_pointwise_conv(plan):
  ops = _ops()
  case = case_table()[plan]
  gate(case)
  lay = case.layer
  rows, k, nout, ldo = lay['rows'], lay['k'], lay['nout'], lay['ldo']
  per_image_w = plan == 'pw_image_w'
  has_res = plan == 'pw_rows'
  assert lay['residual'] and lay['se']
  a = _randn((SOURCES, rows, k), 30)
  stacks = [a]
  if per_image_w:
    stacks.append(_randn((SOURCES, nout, k), 31, scale=k**-0.5))
  else:
    w = _randn((nout, k), 31, scale=k**-0.5)
  if has_res:
    stacks.append(_randn((SOURCES, rows, nout), 32))
  bias = _span_bias(nout, 33)
  impl = ops.PW_SIMT if plan == 'pw_simt' else ops.PW_TCGEN05

  def launch(ins, outs):
    n = ins[0].shape[0]
    if per_image_w:
      ops.pointwise_conv(ins[0], ins[1], bias, outs[0], SWISH, rows=rows, batch=n, nout=nout,
                         impl=impl)
    else:
      ops.pointwise_conv(ins[0], w, bias, outs[0], SWISH, residual=ins[1] if has_res else None,
                         rows=n * rows, batch=1, nout=nout, impl=impl)

  got, = run_case(case, stacks, [((rows, ldo), torch.float16, None)], launch)
  pad = got[..., nout:]
  assert bool(((pad == CANARY[torch.float16]) | (pad == 0)).all()), 'pad columns past nout written'
  for s in (4, 5):
    ws = stacks[1][s] if per_image_w else w
    ref = act_ref(a[s].double() @ ws.double().t() + bias.double(), SWISH)
    if has_res:
      ref = ref + stacks[1][s].double()
    check_close(got[s, :, :nout], ref, '%s source %d' % (plan, s))


@pytest.mark.parametrize('name', ['conv_s1', 'conv_s2'])
def test_conv2d(name):
  from test_gpu_persistent_kernels import _conv_reference
  ops = _ops()
  case = case_table()[name]
  gate(case)
  lay = case.layer
  h, cin, cout, k, st, has_res = (lay[f] for f in ('h', 'cin', 'cout', 'k', 's', 'residual'))
  assert has_res == (name == 'conv_s1')
  ho = _cdiv(h, st)
  x = _randn((SOURCES, h, h, cin), 40)
  wk = _randn((k, k, cin, cout), 41, scale=1.0 / (k * cin**0.5))
  wt = wk.permute(0, 1, 3, 2).reshape(k * k, cout, cin).contiguous()
  bias = _span_bias(cout, 42)
  stacks = [x] + ([_randn((SOURCES, ho, ho, cout), 43)] if has_res else [])

  def launch(ins, outs):
    ops.conv2d(ins[0], wt, bias, outs[0], SWISH, k, st, residual=ins[1] if has_res else None)

  got, = run_case(case, stacks, [((ho, ho, cout), torch.float16, None)], launch)
  for s in (4, 5):
    ref = _conv_reference(x[s:s + 1], wk, bias, stacks[1][s:s + 1] if has_res else None, SWISH, st)
    check_close(got[s:s + 1], ref, '%s source %d' % (name, s))


def test_conv2d_transpose():
  from test_gpu_conv_transpose import reference as convt_f64
  ops = _ops()
  case = case_table()['convt']
  gate(case)
  lay = case.layer
  h, c0, c1, cout = lay['h'], lay['c0'], lay['c1'], lay['cout']
  assert c1 == c0
  a0, a1 = _randn((SOURCES, h, h, c0), 50), _randn((SOURCES, h, h, c1), 51)
  kernel = _randn((3, 3, cout, c0 + c1), 52, scale=3.0 / (2.25 * (c0 + c1))**0.5)
  bias = _span_bias(cout, 53)
  wt = torch.from_numpy(ops.conv_transpose_weights(_cpu(kernel).double().numpy(), c0)).half().to(DEV)

  def launch(ins, outs):
    ops.conv2d_transpose(ins[0], wt, bias, outs[0], SWISH, cout, a1=ins[1])

  got, = run_case(case, [a0, a1], [((2 * h, 2 * h, cout), torch.float16, None)], launch)
  for s in (4, 5):
    x = torch.cat([a0[s:s + 1], a1[s:s + 1]], -1).double()
    check_close(got[s:s + 1], convt_f64(x, kernel.double(), bias.double(), SWISH),
                'convt source %d' % s)


@pytest.mark.parametrize('per_channel', [False, True], ids=['fuse_dw', 'fuse_dw_channel'])
@pytest.mark.parametrize('name', ['fuse_up', 'fuse_down'])
def test_fuse_dw(name, per_channel):
  from test_gpu_memory_bound_kernels import fuse_reference
  ops = _ops()
  case = case_table()[name]
  gate(case)
  lay = case.layer
  f, h, modes, ins = lay['f'], lay['h'], lay['modes'], lay['ins']
  code = {'same': ops.RS_SAME, 'up': ops.RS_UP, 'down': ops.RS_DOWN}
  stacks = [_randn((SOURCES, i, i, f), 60 + j) for j, i in enumerate(ins)]
  taps = _randn((9, f), 64, torch.float32, 1.0 / 3)
  rng = np.random.default_rng(65)
  scalar = [float(v) for v in rng.uniform(0.1, 0.6, size=len(modes)).astype(np.float32)]
  channel = torch.from_numpy(rng.uniform(0.1, 0.6, size=(len(modes), f)).astype(np.float32)).to(DEV)

  def launch(tens, outs):
    specs = [(t, code[m], pool, wt) for t, (m, pool), wt in zip(tens, modes, scalar)]
    ops.fuse_dw(specs, taps, outs[0], SWISH, channel_weights=channel if per_channel else None)

  got, = run_case(case, stacks, [((h, h, f), torch.float16, None)], launch)
  weights = _cpu(channel).numpy() if per_channel else scalar
  for s in (4, 5):
    ref = fuse_reference([_cpu(t[s:s + 1]) for t in stacks], modes, (h, h), _cpu(taps), weights,
                         per_channel, SWISH)
    check_close(got[s:s + 1], ref, '%s source %d' % (name, s))


@pytest.mark.parametrize('name', ['sepconv_tma', 'sepconv'])
def test_sepconv(name):
  """lite0's P3 (F = 64) runs the TMA-staged kernel, D2's (F = 112) the global-load one."""
  from test_gpu_persistent_kernels import check_sepconv
  ops = _ops()
  case = case_table()[name]
  gate(case)
  f, h = case.layer['f'], case.layer['h']
  assert f <= ops.SEPCONV_MAX_C
  x = _randn((SOURCES, h, h, f), 70)
  dw_w = _randn((9, f), 71, torch.float32, 1.0 / 3)
  pw = _randn((f, f), 72, scale=f**-0.5)
  bias = _span_bias(f, 73)

  def launch(ins, outs):
    ops.sepconv([(ins[0], ops.RS_SAME, None, 1.0)], NONE, dw_w, pw, bias, outs[0], SWISH)

  got, = run_case(case, [x], [((h, h, f), torch.float16, None)], launch)
  for s in (4, 5):
    check_sepconv(_cpu(got[s:s + 1]), x[s:s + 1], dw_w, pw, bias, SWISH, f, '%s source %d' % (name, s))


def test_max_pool():
  ops = _ops()
  case = case_table()['max_pool']
  gate(case)
  c, pool, h = case.layer['c'], case.layer['pool'], case.layer['h']
  ho = _cdiv(h, pool[2])
  x = _randn((SOURCES, h, h, c), 80)

  def launch(ins, outs):
    ops.max_pool(ins[0], outs[0], pool[:2], pool[2:])

  got, = run_case(case, [x], [((ho, ho, c), torch.float16, None)], launch)
  for s in (4, 5):
    ref = eo.max_pool_same(x[s:s + 1].float().permute(0, 3, 1, 2), pool[:2], pool[2:])
    assert torch.equal(got[s:s + 1].float(), ref.permute(0, 2, 3, 1)), 'max_pool source %d' % s


def test_global_avg_pool():
  from test_gpu_classifier_top import check_pool
  ops = _ops()
  case = case_table()['gap']
  gate(case)
  h, c = case.layer['h'], case.layer['c']
  x = _randn((SOURCES, h, h, c), 90, scale=2.0) + 0.5

  def launch(ins, outs):
    ops.global_avg_pool(ins[0], outs[0])

  got, = run_case(case, [x], [((c,), torch.float32, None)], launch)
  for s in (4, 5):
    check_pool(got[s:s + 1], x[s:s + 1])


def test_class_argmax():
  """The D7x level-3 class head fused with the class arg-max; each image alone equals the stored
  path of test_gpu_class_argmax (pointwise logits, then pre_nms) bit for bit."""
  from test_gpu_class_argmax import _pad, _stored_path
  ops = _ops()
  case = case_table()['class_argmax']
  gate(case)
  f, h, na, nc = (case.layer[k] for k in ('f', 'h', 'na', 'nc'))
  a = _randn((SOURCES, h, h, f), 130)
  w = _randn((na * nc, f), 131, scale=f**-0.5)
  b = _randn((na * nc,), 132, torch.float32) - 2.0
  wpad, bpad = (t.to(DEV) for t in _pad(_cpu(w), _cpu(b), na, nc))
  total = h * h * na

  def launch(ins, outs):
    ops.class_argmax(ins[0], wpad, bpad, outs[0], outs[1], 0, na)

  scores, classes = run_case(case, [a], [((total,), torch.float32, None), ((total,), torch.int32, None)],
                             launch)
  for s in (4, 5):
    _, want_s, want_c = _stored_path(ops, a[s:s + 1], w, b, na, nc)
    assert torch.equal(scores[s:s + 1], want_s) and torch.equal(classes[s:s + 1], want_c), s
    free_all()


PREP_MEAN, PREP_STD = [100.5, 120.25, 90.75], [50.0, 60.5, 70.125]


def _images(src, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randint(0, 256, (SOURCES,) + tuple(src) + (3,), generator=g, device=DEV,
                       dtype=torch.uint8)


def _check_preprocess(got, imgs, size, name):
  for s in (4, 5):
    ref, _ = po.image_preprocess(_cpu(imgs[s]).numpy(), size, PREP_MEAN, PREP_STD)
    np.testing.assert_array_equal(_cpu(got[s]).numpy(), ref, err_msg='%s source %d' % (name, s))


def test_preprocess():
  ops = _ops()
  case = case_table()['preprocess']
  gate(case)
  size, src = case.layer['size'], case.layer['src']
  imgs = _images(src, 100)

  def launch(ins, outs):
    ops.preprocess(ins[0], outs[0], PREP_MEAN, PREP_STD)

  got, = run_case(case, [imgs], [((size, size, 3), torch.float32, None)], launch)
  _check_preprocess(got, imgs, size, 'preprocess')


def test_preprocess_ragged():
  """The images are packed back to back in one uint8 buffer of more than 2^32 bytes, so the byte
  offsets of the last ones in the descriptor need both of their int32 words."""
  from automl_b200 import inference
  ops = _ops()
  case = case_table()['preprocess_ragged']
  gate(case)
  size, src = case.layer['size'], case.layer['src']
  assert case.batch * src[0] * src[1] * 3 > 1 << 32
  imgs = _images(src, 101)

  def launch(ins, outs):
    n = ins[0].shape[0]
    desc, total, _ = inference.preprocess_table([tuple(src)] * n, size)
    assert total == ins[0].numel()
    ops.preprocess_ragged(ins[0].view(-1), torch.from_numpy(desc).to(DEV), outs[0], PREP_MEAN,
                          PREP_STD)

  got, = run_case(case, [imgs], [((size, size, 3), torch.float32, None)], launch)
  _check_preprocess(got, imgs, size, 'preprocess_ragged')


def test_pre_nms():
  """D7x's level 3 with stored logits (ld 816 for 9 x 90 classes); +inf in the logits' pad
  columns and NaN in the box codes' (a read of either reaches a score, class or box).  Each image
  alone is checked as test_gpu_postprocess_kernels.test_pre_nms checks it: classes and scores
  against po.pre_nms, boxes within check_decode's bound."""
  from test_gpu_postprocess_kernels import Head, check_decode, model_head
  ops = _ops()
  case = case_table()['pre_nms']
  gate(case)
  lay = case.layer
  h, na, nc, ld_cls, ld_box = (lay[k] for k in ('h', 'na', 'nc', 'ld_cls', 'ld_box'))
  m = model_head('efficientdet-d7x')
  head = Head(lay['image'], m.C, m.num_scales, m.aspect_ratios, m.anchor_scale, 3, 3)
  assert head.A == na and head.C == nc and head.total_anchors == h * h * na
  cls = _randn((SOURCES, h, h, ld_cls), 140, scale=2.0) - 4.0
  cls[..., na * nc:] = float('inf')
  box = _randn((SOURCES, h, h, ld_box), 141, scale=0.5)
  box[..., na * 4:] = float('nan')
  anc = head.anchors()
  danc = torch.from_numpy(anc).to(DEV)
  k = h * h * na

  def launch(ins, outs):
    ops.pre_nms([ins[0]], [ins[1]], [(h, h)], na, nc, danc, outs[0], outs[1], outs[2])

  boxes, scores, classes = run_case(
      case, [cls, box], [((k, 4), torch.float32, None), ((k,), torch.float32, None),
                         ((k,), torch.int32, None)], launch)
  for s in (4, 5):
    c64, b64 = _cpu(cls[s:s + 1, ..., :na * nc]).numpy(), _cpu(box[s:s + 1, ..., :na * 4]).numpy()
    _, ref_scores, ref_classes = po.pre_nms(head.params(), [c64], [b64])
    np.testing.assert_array_equal(_cpu(classes[s:s + 1]).numpy(), ref_classes)
    np.testing.assert_allclose(_cpu(scores[s:s + 1]).numpy(), ref_scores, rtol=1e-6, atol=1e-7)
    check_decode(_cpu(boxes[s:s + 1]).numpy(), b64.reshape(1, -1, 4), anc, 'pre_nms source %d' % s)


def test_cls_preprocess():
  """L2's eval pre-process (the legacy bicubic recipe at 800) over packed images past 2^32 bytes:
  the descriptor's byte offsets need both of their int32 words.  Each image alone equals
  classify_oracle.preprocess_image bit for bit, as in test_gpu_classify."""
  import classify_oracle as co
  from automl_b200.efficientnetv2 import preprocessing
  ops = _ops()
  case = case_table()['cls_preprocess']
  gate(case)
  size, src = case.layer['size'], case.layer['src']
  legacy = preprocessing.is_legacy(effnetv2_model.EffNetV2Arch('efficientnet-l2').cfg.data.augname)
  assert legacy
  assert case.batch * src[0] * src[1] * 3 > 1 << 32
  imgs = _images(src, 150)
  table = preprocessing.device_table(DEV)

  def launch(ins, outs):
    n = ins[0].shape[0]
    desc, total = preprocessing.image_table([tuple(src)] * n, size, legacy)
    assert total == ins[0].numel()
    ops.cls_preprocess(ins[0].view(-1), torch.from_numpy(desc).to(DEV), outs[0], ops.CLS_BICUBIC,
                       table)

  got, = run_case(case, [imgs], [((size, size, 3), torch.float32, None)], launch)
  for s in (4, 5):
    ref = co.preprocess_image(_cpu(imgs[s]).numpy(), size, legacy)
    assert torch.equal(_cpu(got[s]), torch.from_numpy(ref)), 'cls_preprocess source %d' % s


def test_softmax_topk():
  from test_gpu_classify import _check_topk
  ops = _ops()
  case = case_table()['softmax_topk']
  gate(case)
  c, k = case.layer['c'], case.layer['k']
  logits = _randn((SOURCES, c), 110, torch.float32, 3.0)

  def launch(ins, outs):
    ops.softmax_topk(ins[0], outs[0], outs[1])

  probs, classes = run_case(case, [logits], [((k,), torch.float32, None), ((k,), torch.int32, None)],
                            launch)
  for s in (4, 5):
    _check_topk(logits[s:s + 1], _cpu(probs[s:s + 1]), _cpu(classes[s:s + 1]))


# ---------------------------------------------------------------------------------------------
def test_checks_catch_misplaced_images():
  """The checks the cases use report each kind of misplacement in doctored outputs: the boundary
  image replaced by another image's result, one bit flipped in the last image, a stray write into
  image 0, one changed canary word, an SE-sum row taken from another image."""
  n, b = 12, 7
  src = sources(n, b)
  singles = _randn((SOURCES, 5, 3, 8), 120)
  sums = torch.randint(-2**40, 2**40, (SOURCES, 8), device=DEV, dtype=torch.int64)

  def fresh():
    out = Canaried((n, 5, 3, 8), torch.float16)
    out.t.copy_(singles[src])
    se = Canaried((n, 8), torch.int64)
    se.t.copy_(sums[src])
    return out, se

  out, se = fresh()
  check_images(out.t, singles, src)
  check_images(se.t, sums, src)
  check_canary(out)
  check_canary(se)

  out, _ = fresh()
  out.t[b] = singles[1]
  assert mismatched_images(out.t, singles, src) == [b]
  out, _ = fresh()
  _bits(out.t)[n - 1, 4, 2, 7] ^= 1
  assert mismatched_images(out.t, singles, src) == [n - 1]
  out, _ = fresh()
  out.t[0, 2, 1, 3] = 0.125
  assert mismatched_images(out.t, singles, src) == [0]
  out, _ = fresh()
  out.buf[out.numel + GUARD - 1] = 0.0
  with pytest.raises(AssertionError, match='canary'):
    check_canary(out)
  _, se = fresh()
  se.t[b] = sums[5]
  with pytest.raises(AssertionError, match='differ'):
    check_images(se.t, sums, src)
  assert mismatched_images(se.t, sums, src) == [b]
