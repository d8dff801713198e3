"""The feature-network variants on the device: edet_fuse_dw_channel (per-channel fusion weights) and
the two QuFPN node signatures against float64, then whole networks (QuFPN, channel_attn /
channel_fastattn, conv_after_downsample, conv_bn_act_pattern) against the fp32 variant oracle
(tests/fpn_variant_oracle.py)."""
import numpy as np
import pytest
import torch

from automl_b200 import arch
from automl_b200 import hparams_config
from automl_b200 import utils
from automl_b200 import weights
from oracle import efficientdet_oracle as eo
from oracle import postprocess_oracle as po
import fpn_variant_oracle as fvo
import precision_model as pm

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
REL_TOL = 1e-3
SENTINEL = -1234.0


def _ops():
  from automl_b200 import ops  # deferred: loads the CUDA library
  return ops


def rel_l2(a, b):
  a, b = a.double().flatten(), b.double().flatten()
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


# ---------------------------------------------------------------------------------------------
# node shapes: (mode, finer / coarser / same) per input, in order; 'generic' has no compile-time
# signature (an upsampled input first)
SIGS = {
    'same_up': ['same', 'up'],
    'same_down': ['same', 'down'],
    'same_same_down': ['same', 'same', 'down'],
    'same_same': ['same', 'same'],
    'same_same_up': ['same', 'same', 'up'],
    'generic': ['up', 'same', 'down'],
}


def _node_inputs(ops, sig, n, h, w, c, g):
  uh, uw = (h - 1) // 2 + 1, (w - 1) // 2 + 1          # coarser level -> nearest upsample
  dh, dw = h * 2 - (h % 2), w * 2 - (w % 2)            # finer level  -> max-pool 3x3 s2
  nchw = lambda t: t.double().permute(0, 3, 1, 2)
  tens, specs, res = [], [], []
  for mode in SIGS[sig]:
    if mode == 'same':
      t = torch.randn(n, h, w, c, generator=g).half()
      specs.append((ops.RS_SAME, None))
      res.append(nchw(t))
    elif mode == 'up':
      t = torch.randn(n, uh, uw, c, generator=g).half()
      specs.append((ops.RS_UP, None))
      res.append(eo.resize_nearest_tf1(nchw(t), h, w))
    else:
      t = torch.randn(n, dh, dw, c, generator=g).half()
      specs.append((ops.RS_DOWN, (3, 3, 2, 2)))
      res.append(eo.max_pool_same(nchw(t), (3, 3), (2, 2)))
    tens.append(t)
  return tens, specs, res


def _reference(res, wts, dwk, act):
  """float64 fusion (weights [inputs, C] or scalars) -> act -> depthwise 3x3 'same', NHWC."""
  fused = sum(r * torch.as_tensor(np.asarray(wt, np.float64)).view(1, -1, 1, 1) if np.ndim(wt)
              else r * float(wt) for r, wt in zip(res, wts))
  if act == utils.ACT_SWISH:
    fused = fused * torch.sigmoid(fused)
  return eo.depthwise_conv2d_same(fused, dwk.double().unsqueeze(-1)).permute(0, 2, 3, 1)


def _out_with_sentinel(n, h, w, c):
  buf = torch.full((n * h * w * c + 4096,), SENTINEL, dtype=torch.float16, device=DEV)
  return buf, buf[:n * h * w * c].view(n, h, w, c)


@pytest.mark.parametrize('sig', sorted(SIGS))
@pytest.mark.parametrize('c', [40, 64, 88])
@pytest.mark.parametrize('hw', [(13, 9), (20, 20), (5, 37)])
def test_fuse_dw_channel_against_float64(sig, c, hw):
  """Per-channel weights that differ across channels (c = 40 / 88: the last 32-channel chunk is
  partial), ragged tiles; nothing outside `out` is written.  The scalar form of the same node is
  checked too (the two QuFPN signatures are new for it as well)."""
  ops = _ops()
  n = 2
  h, w = hw
  g = torch.Generator().manual_seed(h * 1000 + w * 10 + c + len(sig))
  tens, modes, res = _node_inputs(ops, sig, n, h, w, c, g)
  k = len(tens)
  raw = np.random.default_rng(c + k).uniform(0.05, 1.0, size=(k, c)).astype(np.float32)
  cw = raw / raw.sum(0, keepdims=True)
  dwk = (torch.randn(3, 3, c, generator=g) / 3).half()
  dw_w = dwk.reshape(9, c).float().to(DEV)
  specs = [(t.to(DEV), m, pool, 0.0) for t, (m, pool) in zip(tens, modes)]
  for act in (utils.ACT_SWISH, utils.ACT_NONE):
    buf, out = _out_with_sentinel(n, h, w, c)
    ops.fuse_dw(specs, dw_w, out, act, channel_weights=torch.from_numpy(cw).to(DEV))
    torch.cuda.synchronize()
    ref = _reference(res, list(cw), dwk, act)
    assert torch.allclose(out.cpu().double(), ref, rtol=2e-3, atol=2e-3), (sig, c, hw, act)
    assert bool((buf[n * h * w * c:] == SENTINEL).all())
  # the scalar entry point on the same node shape
  sw = [0.45, 0.35, 0.2][:k]
  buf, out = _out_with_sentinel(n, h, w, c)
  ops.fuse_dw([(t, m, pool, wt) for (t, m, pool, _), wt in zip(specs, sw)], dw_w, out, utils.ACT_SWISH)
  torch.cuda.synchronize()
  ref = _reference(res, [np.float32(x) for x in sw], dwk, utils.ACT_SWISH)
  assert torch.allclose(out.cpu().double(), ref, rtol=2e-3, atol=2e-3), (sig, c, hw)
  assert bool((buf[n * h * w * c:] == SENTINEL).all())


@pytest.mark.parametrize('sig', sorted(SIGS))
@pytest.mark.parametrize('c', [40, 88])
def test_fuse_dw_channel_with_equal_weights_is_the_scalar_kernel(sig, c):
  """Per-channel weights equal to w in every channel give the bits of edet_fuse_dw with weight w
  (same products, same accumulation order)."""
  ops = _ops()
  n, h, w = 2, 19, 11
  g = torch.Generator().manual_seed(7 * c + len(sig))
  tens, modes, _ = _node_inputs(ops, sig, n, h, w, c, g)
  wts = [0.61, 0.27, 0.12][:len(tens)]
  dw_w = (torch.randn(9, c, generator=g) / 3).float().to(DEV)
  specs = [(t.to(DEV), m, pool, wt) for t, (m, pool), wt in zip(tens, modes, wts)]
  cw = torch.tensor([[wt] * c for wt in wts], dtype=torch.float32, device=DEV)
  for act in (utils.ACT_SWISH, utils.ACT_RELU6, utils.ACT_NONE):
    a = torch.empty(n, h, w, c, dtype=torch.float16, device=DEV)
    b = torch.empty_like(a)
    ops.fuse_dw(specs, dw_w, a, act)
    ops.fuse_dw(specs, dw_w, b, act, channel_weights=cw)
    torch.cuda.synchronize()
    assert torch.equal(a, b), (sig, c, act)


def test_fuse_dw_channel_rejects_bad_weights():
  ops = _ops()
  x = torch.zeros(1, 4, 4, 8, dtype=torch.float16, device=DEV)
  out = torch.empty_like(x)
  dw_w = torch.zeros(9, 8, device=DEV)
  with pytest.raises(ValueError):
    ops.fuse_dw([(x, ops.RS_SAME, None, 1.0)], dw_w, out, utils.ACT_NONE,
                channel_weights=torch.zeros(2, 8, device=DEV))
  with pytest.raises(ValueError):
    ops.fuse_dw([(x, ops.RS_SAME, None, 1.0)], dw_w, out, utils.ACT_NONE,
                channel_weights=torch.zeros(1, 8, dtype=torch.float16, device=DEV))


# ---------------------------------------------------------------------------------------------
def _setup(name, image_size, n, seed=0, **over):
  c = hparams_config.get_efficientdet_config(name)
  c.override(dict(image_size=image_size, **over))
  a = arch.DetArch(c)
  w = weights.synthetic_weights(a, seed)
  h, wd = a.image_hw
  x = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, size=(n, h, wd, 3)).astype(np.float32)
  return c, a, w, x


def _engine(c, w, n, **kw):
  from automl_b200.engine import Engine
  return Engine(c, w, n, **kw)


@pytest.mark.parametrize('name,size,n,over', [
    ('efficientdet-d0', 256, 2, dict(fpn_name='qufpn')),
    ('efficientdet-d0', 128, 1, dict(fpn_weight_method='channel_fastattn')),
    ('efficientdet-d1', 128, 1, dict(fpn_weight_method='channel_attn')),
    ('efficientdet-d0', 128, 2, dict(fpn_name='qufpn', conv_after_downsample=True)),
    ('efficientdet-d0', 128, 1, dict(conv_bn_act_pattern=True)),
], ids=['d0_qufpn', 'd0_channel_fastattn', 'd1_channel_attn', 'd0_qufpn_conv_after_downsample',
        'd0_conv_bn_act_pattern'])
def test_network_parity(name, size, n, over):
  c, a, w, x = _setup(name, size, n, **over)
  orc = fvo.VariantOracle(c, w, torch.float32)
  cls_ref, box_ref = orc(x)
  eng = _engine(c, w, n, use_cuda_graph=False)
  cls_out, box_out = eng.forward(torch.from_numpy(x))
  torch.cuda.synchronize()
  if over.get('fpn_weight_method', '').startswith('channel_'):
    assert any(r['kind'] == 'bifpn_fuse_dw' for r in eng.op_info)
  for l in a.levels:
    got = eng.fpn_feats[l].float().cpu().permute(0, 3, 1, 2)
    assert rel_l2(got, orc.endpoints['fpn_%d' % l]) < REL_TOL, 'fpn %d' % l
    assert rel_l2(cls_out[l].float().cpu(), cls_ref[l]) < REL_TOL, 'cls %d' % l
    assert rel_l2(box_out[l].float().cpu(), box_ref[l]) < REL_TOL, 'box %d' % l


def test_network_parity_lite0_qufpn_vs_format_model():
  """lite0 + QuFPN: relu6 and un-normalised 'sum' fusion on every one of the 21 nodes per cell,
  quad-add nodes included.  On random weights this network is ill-conditioned like lite3
  (tests/test_gpu_network.py): every BiFPN / class / box tensor within 1.5x the fp16 format model
  (fvo.DeviceModel: the fp32 variant oracle with the engine's rounding sites) + 1e-4."""
  c, a, w, x = _setup('efficientdet-lite0', 256, 1, seed=5, fpn_name='qufpn')
  assert a.fpn_weight_method == 'sum' and len(a.cells[0]['nodes']) == 21
  eng = _engine(c, w, 1, use_cuda_graph=False)
  cls_out, box_out = eng.forward(torch.from_numpy(x))
  torch.cuda.synchronize()
  m = fvo.DeviceModel(c, a, w, x)
  for l in a.levels:
    got = eng.fpn_feats[l].float().cpu().permute(0, 3, 1, 2)
    ref = m.ref.endpoints['fpn_%d' % l]
    assert rel_l2(got, ref) < pm.bar(m.endpoint_error('fpn_%d' % l)), 'fpn %d' % l
    assert rel_l2(cls_out[l].float().cpu(), m.cls_ref[l]) < pm.bar(m.cls_error(l)), 'cls %d' % l
    assert rel_l2(box_out[l].float().cpu(), m.box_ref[l]) < pm.bar(m.box_error(l)), 'box %d' % l


def test_qufpn_detect_matches_oracle_postprocess():
  c, a, w, x = _setup('efficientdet-d0', 128, 2, seed=5, fpn_name='qufpn')
  eng = _engine(c, w, 2)
  det = eng.detect(torch.from_numpy(x)).cpu().numpy().copy()
  eng.forward(torch.from_numpy(x))
  torch.cuda.synchronize()
  params = c.as_dict()
  cls_l = [eng.cls_out[l][..., :810].float().cpu().numpy() for l in a.levels]
  box_l = [eng.box_out[l][..., :36].float().cpu().numpy() for l in a.levels]
  ref_boxes, ref_scores, ref_classes = po.pre_nms(params, cls_l, box_l)
  np.testing.assert_array_equal(eng.classes.cpu().numpy(), ref_classes)
  np.testing.assert_allclose(eng.scores.cpu().numpy(), ref_scores, rtol=1e-6, atol=1e-7)
  gb, gs, gc = eng.boxes.cpu().numpy(), eng.scores.cpu().numpy(), eng.classes.cpu().numpy()
  iou_t, score_t, tf_sigma = po.nms_v5_params(params['nms_configs'])
  for i in range(2):
    idx, sc, v = po.non_max_suppression_v5(gb[i], gs[i], 100, iou_t, score_t, tf_sigma, True)
    assert int(eng.valid[i]) == v
    np.testing.assert_array_equal(eng.sel_index[i].cpu().numpy(), idx)
    np.testing.assert_array_equal(det[i, :, 5], sc)
    np.testing.assert_array_equal(det[i, :, 1:5], po.clip_boxes(gb[i][idx], 128))
    np.testing.assert_array_equal(det[i, :, 6], (gc[i][idx] + 1).astype(np.float32))


@pytest.mark.parametrize('over', [dict(fpn_name='qufpn', conv_after_downsample=True),
                                  dict(fpn_name='qufpn', fpn_weight_method='channel_fastattn')])
def test_qufpn_pipelined_graph_and_eager_runs_agree(over):
  """QuFPN cell 0 reads P3 / P4 again late (nodes 8 and 15): the pipelined step, which lets the
  next backbone overwrite P3..P5 after cell 0, the single-graph step and eager launches give the
  same bits."""
  c, a, w, _ = _setup('efficientdet-d0', 128, 2, seed=11, **over)
  rng = np.random.default_rng(12)
  xs = [torch.from_numpy(rng.uniform(-2, 2, size=(2, 128, 128, 3)).astype(np.float32)).cuda()
        for _ in range(4)]
  eager = _engine(c, w, 2, use_cuda_graph=False, pipeline=False)
  want = [eager.detect(x).clone() for x in xs]
  graph = _engine(c, w, 2, use_cuda_graph=True, pipeline=False)
  pipe = _engine(c, w, 2, use_cuda_graph=True, pipeline=True)
  assert pipe.num_backbone_ops < pipe._cell0_end < pipe.num_network_ops  # pylint: disable=protected-access
  got = [torch.empty_like(want[0]) for _ in xs]
  for i, x in enumerate(xs):
    pipe.input.copy_(x, non_blocking=True)
    pipe.run(postprocess=True, after_nms=lambda det, i=i: got[i].copy_(det, non_blocking=True))
  pipe.wait_detections()
  torch.cuda.synchronize()
  assert not torch.equal(want[0], want[1])
  for i, x in enumerate(xs):
    assert torch.equal(graph.detect(x), want[i]), 'graph step %d' % i
    assert torch.equal(got[i], want[i]), 'pipelined step %d' % i
  _, box_e = eager.forward(xs[3])
  _, box_g = graph.forward(xs[3])
  torch.cuda.synchronize()
  for l in a.levels:
    assert torch.equal(box_e[l], box_g[l])


def test_efficientdet_call_surface_with_variants():
  from automl_b200 import efficientdet_arch
  x = torch.zeros(1, 64, 64, 3)
  cls_out, box_out = efficientdet_arch.efficientdet(
      x, model_name='efficientdet-d0', image_size=64, fpn_name='qufpn',
      fpn_weight_method='channel_fastattn', conv_bn_act_pattern=True, conv_after_downsample=True)
  assert sorted(cls_out) == [3, 4, 5, 6, 7]
  assert tuple(cls_out[3].shape) == (1, 8, 8, 810) and tuple(box_out[7].shape) == (1, 1, 1, 36)
  assert all(bool(torch.isfinite(t).all()) for t in list(cls_out.values()) + list(box_out.values()))
