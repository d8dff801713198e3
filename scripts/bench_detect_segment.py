"""Measures detections and masks of the same images: ServingDriver.serve_stream_with_masks (one
pipelined pass per request) against serve_stream followed by segment_stream over the same requests
(two passes), next to serve_stream alone.

EfficientDet-D0 at 640 x 640, batch 32, heads=['object_detection', 'segmentation'], seeded
synthetic weights; each image's size is drawn from the COCO-like mix of
scripts/bench_ragged_serving.py.  All three run on one driver, so they share its engine, and
alternate within each round.  Reported, one line each: images/s (every image counted once, with its
boxes, and its mask where asked for; three requests in flight), median and [min, max] over ROUNDS
windows of REQS requests, after WARMUP windows.  The first request's combined result is checked
bit for bit against the two passes.  The GPU's name, power limit and SM clocks are printed with the
numbers.  Needs the GPU: there is no CPU path.
usage: python scripts/bench_detect_segment.py [out.json]"""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from automl_b200 import inference  # noqa: E402
from bench_ragged_serving import BATCH, MIX, MODEL, NREQ, SIZE  # noqa: E402

REQS, ROUNDS, WARMUP = 12, 5, 1


def _gpu():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                         '--format=csv,noheader'],
                        stdout=subprocess.PIPE, text=True, check=True).stdout.strip()


def _requests(rng):
  out = []
  for _ in range(NREQ):
    sizes = [MIX[i] for i in rng.integers(0, len(MIX), size=BATCH)]
    out.append([rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes])
  return out


def _two_passes(driver, reqs):
  """serve_stream, then segment_stream over the same requests: yields one result per request."""
  dets = list(driver.serve_stream(reqs))
  masks = driver.segment_stream(reqs)
  return zip(dets, masks)


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_detect_segment.py needs an H100')
  gpu = _gpu()
  requests = _requests(np.random.default_rng(0))
  driver = inference.ServingDriver(MODEL, '_', batch_size=BATCH,
                                   model_params={'image_size': SIZE,
                                                 'heads': ['object_detection', 'segmentation']})
  reqs = [requests[i % NREQ] for i in range(REQS)]
  runs = {
      'serve_stream_with_masks': lambda: (len(d) for d, _ in driver.serve_stream_with_masks(reqs)),
      'serve_stream+segment_stream': lambda: (len(d) for d, _ in _two_passes(driver, reqs)),
      'serve_stream': lambda: (len(d) for d in driver.serve_stream(reqs)),
  }
  for fn in runs.values():
    for _ in range(WARMUP):
      sum(fn())
  rates = {k: [] for k in runs}
  for _ in range(ROUNDS):
    for name, fn in runs.items():
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      n = sum(fn())
      rates[name].append(n / (time.perf_counter() - t0))
  det, masks = driver.serve_images_with_masks(requests[0])
  same = bool(np.array_equal(det, driver.serve_images(requests[0])) and
              all(np.array_equal(a, b) for a, b in zip(masks, driver.segment_images(requests[0]))))
  rows = []
  for name, r in rates.items():
    rows.append({'measure': name + ' images/s',
                 'config': '%s %d^2 batch %d heads=[object_detection, segmentation], sizes from the '
                           'COCO-like mix' % (MODEL, SIZE, BATCH),
                 'windows': '%d x %d requests, three in flight, the three runs alternating'
                            % (ROUNDS, REQS),
                 'images_per_s': round(statistics.median(r), 1),
                 'min_max': [round(min(r), 1), round(max(r), 1)],
                 'gpu': gpu})
  rows[0]['equals_two_passes'] = same
  for r in rows:
    print(json.dumps(r))
  rows.append({'gpu_after': _gpu()})
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
