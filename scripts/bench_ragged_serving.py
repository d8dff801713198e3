"""Measures ServingDriver on ragged requests (images of different sizes), the traffic real serving
sees, against the uniform batch that bench.py's e2e row times.

EfficientDet-D0 at 640 x 640, batch 32, seeded synthetic weights.  Ragged requests draw each image's
size from a seeded COCO-like mix (MIX); the arrays are ordinary (pageable) numpy arrays, as a
decoder returns them.  Three arms, each REQS requests through submit() with three in flight,
alternating for ROUNDS windows:
  * uniform:     one pinned uint8 [32, 480, 640, 3] tensor (bench.py e2e);
  * ragged:      the ragged lists, staged behind a descriptor table, one H2D and one
                 edet_preprocess_ragged launch per request;
  * per_image:   the same lists through the per-image path this replaced (restated below: a pageable
                 H2D copy and one ops.preprocess launch per image, on the current stream).
Reported per arm: images/s (median, [min, max]) and the host time spent inside submit() per
request.  Also: the ragged launch alone (CUDA-event window over a graph of COPIES launches on
separate inputs) with its algorithmic bytes 3 * sum(h * w) + 12 * n * H * W, the 32 per-image
launches of the old path timed the same way, and whether the ragged and per-image arms return equal
detections on the timed inputs.  Prints the GPU's name and power limit with the numbers.  Needs the
GPU: there is no CPU path.
usage: python scripts/bench_ragged_serving.py [out.json]"""
import collections
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automl_b200 import inference  # noqa: E402
from automl_b200 import ops  # noqa: E402

MODEL, SIZE, BATCH = 'efficientdet-d0', 640, 32
MIX = [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375), (612, 612), (640, 640)]
NREQ = 4                      # distinct ragged requests, cycled
REQS, ROUNDS, WARMUP = 12, 5, 2
COPIES, LAUNCH_REPLAYS = 4, 50


class PerImageDriver(inference.ServingDriver):
  """The ragged path before the staged launch: every image of the request is its own pageable H2D
  copy and its own edet_preprocess launch on the current stream."""

  def _stage(self, eng, slot, request, table=None, mirrored=False):
    for i, im in enumerate(request.images):
      raw = torch.as_tensor(np.ascontiguousarray(im), dtype=torch.uint8).to(self.device)[None]
      slot.scales[i] = ops.preprocess(raw, eng.input[i:i + 1], self.mean_rgb, self.stddev_rgb)
    eng.image_scales.copy_(slot.scales, non_blocking=True)


def _gpu():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        stdout=subprocess.PIPE, text=True, check=True).stdout.strip()


def _window(fn, reps):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


def _graph_us(fns):
  """Device time of one call of `fns` (in order), from a CUDA graph of all of them."""
  for fn in fns:
    fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for fn in fns:
      fn()
  _window(g.replay, 5)
  return _window(g.replay, LAUNCH_REPLAYS) * 1e3


def _requests(rng):
  out = []
  for _ in range(NREQ):
    sizes = [MIX[i] for i in rng.integers(0, len(MIX), size=BATCH)]
    out.append([rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes])
  return out


def bench_launches(requests, mean, std):
  dev = 'cuda:0'
  images = requests[0]
  desc, total, _ = inference.preprocess_table([im.shape[:2] for im in images], SIZE)
  rng = np.random.default_rng(3)
  d = torch.from_numpy(desc).to(dev)
  packed = [torch.from_numpy(rng.integers(0, 256, size=total, dtype=np.uint8)).to(dev)
            for _ in range(COPIES)]
  out = torch.empty((BATCH, SIZE, SIZE, 3), dtype=torch.float32, device=dev)
  ragged_us = _graph_us([lambda p=p: ops.preprocess_ragged(p, d, out, mean, std) for p in packed]) / COPIES
  singles = [torch.from_numpy(im[None].copy()).to(dev) for im in images]
  loop_us = _graph_us([lambda i=i, r=r: ops.preprocess(r, out[i:i + 1], mean, std)
                       for i, r in enumerate(singles)])
  nbytes = 3 * sum(im.shape[0] * im.shape[1] for im in images) + 12 * BATCH * SIZE * SIZE
  return {'kernel': 'preprocess_ragged',
          'config': 'D0 %d^2 batch %d, sizes from the COCO-like mix' % (SIZE, BATCH),
          'us': round(ragged_us, 2), 'MB': round(nbytes / 1e6, 3),
          'TB/s': round(nbytes / ragged_us / 1e6, 3),
          'per_image_launches_us': round(loop_us, 2)}


def _run(driver, reqs):
  """REQS requests through submit(), three in flight: (seconds, host seconds inside submit, results)."""
  pending, results, in_submit = collections.deque(), [], 0.0
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for r in reqs:
    s = time.perf_counter()
    pending.append(driver.submit(r))
    in_submit += time.perf_counter() - s
    if len(pending) >= driver.MAX_IN_FLIGHT:
      results.append(pending.popleft().result())
  while pending:
    results.append(pending.popleft().result())
  torch.cuda.synchronize()
  return time.perf_counter() - t0, in_submit, results


def bench_serving(requests):
  rng = np.random.default_rng(1)
  uniform = torch.from_numpy(rng.integers(0, 256, size=(BATCH, 480, 640, 3), dtype=np.uint8)).pin_memory()
  new = inference.ServingDriver(MODEL, '_', batch_size=BATCH, model_params={'image_size': SIZE})
  old = PerImageDriver(MODEL, '_', batch_size=BATCH, model_params={'image_size': SIZE})
  ragged_reqs = [requests[i % NREQ] for i in range(REQS)]
  arms = {'uniform': (new, [uniform] * REQS), 'ragged': (new, ragged_reqs),
          'per_image': (old, ragged_reqs)}
  for driver, reqs in arms.values():
    for _ in range(WARMUP):
      _run(driver, reqs)
  rates = {k: [] for k in arms}
  submit_ms = {k: [] for k in arms}
  last = {}
  for _ in range(ROUNDS):
    for key, (driver, reqs) in arms.items():
      secs, in_submit, results = _run(driver, reqs)
      rates[key].append(REQS * BATCH / secs)
      submit_ms[key].append(in_submit / REQS * 1e3)
      last[key] = results
  row = {'config': '%s %d^2 batch %d' % (MODEL, SIZE, BATCH),
         'windows': '%d x %d requests per arm, alternating, three in flight' % (ROUNDS, REQS),
         'ragged_equals_per_image': all(np.array_equal(a, b)
                                        for a, b in zip(last['ragged'], last['per_image']))}
  for key in arms:
    row[key + '_images_per_s'] = round(statistics.median(rates[key]), 1)
    row[key + '_min_max'] = [round(min(rates[key]), 1), round(max(rates[key]), 1)]
    row[key + '_submit_ms_per_request'] = round(statistics.median(submit_ms[key]), 3)
  return row


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_ragged_serving.py needs an H100')
  gpu = _gpu()
  requests = _requests(np.random.default_rng(0))
  params = inference.ServingDriver(MODEL, '_').params
  mean, std = inference._rgb3(params['mean_rgb']), inference._rgb3(params['stddev_rgb'])
  rows = [bench_launches(requests, mean, std), bench_serving(requests)]
  for r in rows:
    r['gpu'] = gpu
    print(json.dumps(r))
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
