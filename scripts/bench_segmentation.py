"""Times the segmentation head's launches (edet_conv2d_transpose, one per stage) of EfficientDet-D0
at 640 x 640, batch 32, with CUDA events: each stage replayed R times as a CUDA graph, and the whole
head the same way.  Reports per stage the time, the algorithmic HBM bytes (Engine.op_info) and the
achieved rate, and prints the GPU's name and power limit with the numbers.
usage: python scripts/bench_segmentation.py [out.json]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automl_b200 import arch, hparams_config, weights  # noqa: E402
from automl_b200.engine import Engine  # noqa: E402

BATCH, SIZE, REPS = 32, 640, 50


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name()


def _time(fns):
  """ms per replay of a CUDA graph of fns, over REPS replays after a warm-up."""
  for fn in fns:
    fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for fn in fns:
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


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_segmentation.py needs an H100')
  c = hparams_config.get_efficientdet_config('efficientdet-d0')
  c.override(dict(image_size=SIZE, heads=['segmentation']))
  eng = Engine(c, weights.synthetic_weights(arch.DetArch(c), 0), BATCH)
  eng.set_input(torch.from_numpy(
      np.random.default_rng(0).uniform(-2, 2, size=(BATCH, SIZE, SIZE, 3)).astype(np.float32)))
  eng.forward()     # BiFPN outputs the head reads
  torch.cuda.synchronize()
  stages = [(name, fn, info) for (name, fn), info in zip(eng._ops, eng.op_info)  # pylint: disable=protected-access
            if info['kind'] == 'conv_transpose_tc']
  rows = []
  for name, fn, info in stages:
    ms = _time([fn])
    rows.append({'stage': name, 'us': round(ms * 1e3, 2), 'MB': round(info['bytes'] / 1e6, 2),
                 'TB/s': round(info['bytes'] / (ms * 1e-3) / 1e12, 3)})
    print(json.dumps(rows[-1]))
  ms = _time([fn for _, fn, _ in stages])
  total = sum(info['bytes'] for _, _, info in stages)
  rows.append({'stage': 'whole head', 'us': round(ms * 1e3, 2), 'MB': round(total / 1e6, 2),
               'TB/s': round(total / (ms * 1e-3) / 1e12, 3), 'gpu': _gpu(),
               'config': 'efficientdet-d0 %dx%d batch %d' % (SIZE, SIZE, BATCH)})
  print(json.dumps(rows[-1]))
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
