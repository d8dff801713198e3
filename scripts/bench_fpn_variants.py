"""EfficientDet-D0 640 x 640 batch 32 with the feature-network variants (BiFPN as the yardstick,
QuFPN, channel_fastattn): images/s of the network alone (one CUDA graph, forward()) and of the
pipelined detect step, and the summed BiFPN-node fuse_dw time per node signature
(fuse_common.cuh) with its algorithmic bytes per us (Engine.op_info).  Each fuse_dw launch is timed
alone as a CUDA graph replayed REPS times with CUDA events.  The detect step includes NMS-V5, whose
time depends on the scores: on seeded synthetic weights a variant can send every image to the
full-queue NMS kernel, so the count of such images is reported with it.  Prints the GPU's name
and power limit with the numbers.
usage: python scripts/bench_fpn_variants.py [out.json]"""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automl_b200 import arch, hparams_config, weights  # noqa: E402
from automl_b200.engine import Engine  # noqa: E402

BATCH, SIZE, REPS, STEPS, WARMUP = 32, 640, 50, 60, 10
VARIANTS = [('bifpn', {}), ('qufpn', {'fpn_name': 'qufpn'}),
            ('channel_fastattn', {'fpn_weight_method': 'channel_fastattn'})]
# node input modes (after conv_after_downsample moved a pool in front of its conv) -> the
# compile-time signature edet_fuse_dw picks (fuse_common.cuh::fuse_signature)
SIGNATURES = {('same', 'up'): 'SameUp', ('same', 'down'): 'SameDown',
              ('same', 'same', 'down'): 'SameSameDown', ('same', 'same'): 'SameSame',
              ('same', 'same', 'up'): 'SameSameUp'}


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name()


def _time(fn):
  """ms per replay of a CUDA graph of fn, over REPS replays after a warm-up."""
  fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    fn()
  for _ in range(5):
    g.replay()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(REPS):
    g.replay()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / REPS


def _images_per_s(eng, postprocess):
  def step():
    eng.run(postprocess=postprocess)
    if postprocess:
      eng.wait_detections()
  for _ in range(WARMUP):
    step()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(STEPS):
    eng.run(postprocess=postprocess)
  if postprocess:
    eng.wait_detections()
  e1.record()
  torch.cuda.synchronize()
  return BATCH * STEPS / (e0.elapsed_time(e1) * 1e-3)


def _signature(a, node):
  modes = tuple('same' if a.conv_after_pool(r) else r.mode for r in node.inputs)
  return SIGNATURES.get(modes, 'generic')


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_fpn_variants.py needs an H100')
  x = torch.from_numpy(np.random.default_rng(0).uniform(-2, 2, size=(BATCH, SIZE, SIZE, 3))
                       .astype(np.float32))
  rows = []
  for label, over in VARIANTS:
    c = hparams_config.get_efficientdet_config('efficientdet-d0')
    c.override(dict(image_size=SIZE, **over))
    a = arch.DetArch(c)
    eng = Engine(c, weights.synthetic_weights(a, 0), BATCH)
    eng.set_input(x)
    net_ips = _images_per_s(eng, postprocess=False)
    ips = _images_per_s(eng, postprocess=True)
    fallback = eng.nms_fallback_count()
    eng.forward()
    torch.cuda.synchronize()
    sig_of = {n.scope + '/fuse_dw': _signature(a, n) for cell in a.cells for n in cell['nodes']}
    per_sig = collections.defaultdict(lambda: {'launches': 0, 'us': 0.0, 'bytes': 0})
    for (name, fn), info in zip(eng._ops, eng.op_info):  # pylint: disable=protected-access
      if info['kind'] != 'bifpn_fuse_dw':
        continue
      s = per_sig[sig_of[name]]
      s['launches'] += 1
      s['us'] += _time(fn) * 1e3
      s['bytes'] += info['bytes']
    row = {'variant': label, 'network_images_per_s': round(net_ips, 1),
           'detect_images_per_s': round(ips, 1), 'nms_full_queue_images': fallback, 'fuse_dw': {
        k: {'launches': v['launches'], 'us': round(v['us'], 2), 'MB': round(v['bytes'] / 1e6, 2),
            'bytes_per_us': round(v['bytes'] / v['us'], 1)} for k, v in sorted(per_sig.items())},
           'gpu': _gpu(), 'config': 'efficientdet-d0 %dx%d batch %d' % (SIZE, SIZE, BATCH)}
    rows.append(row)
    print(json.dumps(row))
    del eng
    torch.cuda.empty_cache()
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
