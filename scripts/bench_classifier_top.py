"""Measures what the classification top costs EfficientNetV2-S at 384 x 384 (batch 128 and batch 1):

  * the step (one CUDA-graph replay) of the include_top=False and include_top=True models, timed
    with CUDA events in alternating windows of STEPS replays in one process, ROUNDS times each;
  * the pool and the Dense launch alone over many launches.  The pool rotates over COPIES
    separate head maps so that no launch finds its input in the L2 cache; the Dense weights are
    L2-resident in this loop;
  * their algorithmic bytes (EffNetV2Model.op_info, from shapes) and bytes / time;
  * the bytes serve_stream() copies to the host per batch in both modes.

Prints the GPU's name and power limit with the numbers.  Needs the GPU: there is no CPU path.
usage: python scripts/bench_classifier_top.py [out.json]"""
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automl_b200 import ops  # noqa: E402
from automl_b200.efficientnetv2 import effnetv2_model  # noqa: E402

NAME, SIZE = 'efficientnetv2-s', 384
STEPS, ROUNDS, WARMUP = 10, 5, 5
COPIES, LAUNCH_REPLAYS = 4, 200


def _gpu():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        stdout=subprocess.PIPE, text=True, check=True).stdout.strip()


def _window(fn, reps):
  """ms per call of fn over reps calls between two CUDA events."""
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


def _launch_us(fns):
  """us per launch: the launches of fns captured as one CUDA graph, replayed LAUNCH_REPLAYS times."""
  for fn in fns:
    fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for fn in fns:
      fn()
  _window(g.replay, 10)
  return _window(g.replay, LAUNCH_REPLAYS) / len(fns) * 1e3


def measure(batch):
  arch = effnetv2_model.EffNetV2Arch(NAME)
  w = effnetv2_model.synthetic_weights(arch, 0, include_top=True)
  x = torch.from_numpy(np.random.default_rng(0).uniform(
      -1, 1, size=(batch, SIZE, SIZE, 3)).astype(np.float32))
  models = {top: effnetv2_model.get_model(NAME, include_top=top, weights=w, batch_size=batch,
                                          image_size=SIZE) for top in (False, True)}
  for m in models.values():
    m(x)
    _window(m.run, WARMUP)
  steps = {False: [], True: []}
  for _ in range(ROUNDS):
    for top in (False, True):
      steps[top].append(_window(models[top].run, STEPS))
  row = {'config': '%s %dx%d batch %d' % (NAME, SIZE, SIZE, batch),
         'windows': '%d x %d steps each, alternating' % (ROUNDS, STEPS)}
  for top in (False, True):
    key = 'step_ms_top' if top else 'step_ms_no_top'
    row[key] = round(statistics.median(steps[top]), 4)
    row[key + '_min_max'] = [round(min(steps[top]), 4), round(max(steps[top]), 4)]
    row['d2h_bytes_per_batch_' + ('top' if top else 'no_top')] = (
        models[top].output.numel() * models[top].output.element_size())
  m = models[True]
  info = {o['name']: o for o in m.op_info}
  head, pooled, logits = m.endpoints['head_1x1'], m.endpoints['pooled_features'], m.output
  heads = [head] + [head.clone() for _ in range(COPIES - 1)]
  us = _launch_us([lambda h=h: ops.global_avg_pool(h, pooled) for h in heads])
  row['avg_pool'] = {'us': round(us, 2), 'MB': round(info['avg_pool']['bytes'] / 1e6, 3),
                     'TB/s': round(info['avg_pool']['bytes'] / us / 1e6, 3)}
  dense = dict(m._ops)['dense']  # pylint: disable=protected-access
  us = _launch_us([dense] * COPIES)
  row['dense'] = {'us': round(us, 2), 'MB': round(info['dense']['bytes'] / 1e6, 3),
                  'GFLOP': round(info['dense']['flops'] / 1e9, 4),
                  'TB/s': round(info['dense']['bytes'] / us / 1e6, 3),
                  'TFLOP/s': round(info['dense']['flops'] / us / 1e6, 3)}
  assert tuple(logits.shape) == (batch, 1000)
  return row


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_classifier_top.py needs an H100')
  gpu = _gpu()
  rows = []
  for batch in (128, 1):
    rows.append(dict(measure(batch), gpu=gpu))
    print(json.dumps(rows[-1]))
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
