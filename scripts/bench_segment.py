"""Measures segmentation serving from decoded images: ServingDriver.segment_stream and the
edet_seg_masks launch.

EfficientDet-D0 at 640 x 640, batch 32, heads=['segmentation'], seeded synthetic weights; each
image's size is drawn from the COCO-like mix of scripts/bench_ragged_serving.py.  Reported:
  * images/s through segment_stream (three requests in flight), median and [min, max] over ROUNDS
    windows of REQS requests, after WARMUP windows;
  * the mask kernel alone: CUDA events around LAUNCHES back-to-back launches on the engine's own
    logits, its algorithmic bytes (the logits cells it samples, once each, the table and the
    sum(h * w) mask bytes) and their rate as a share of the H100 SXM's 3.35 TB/s.
The GPU's name, power limit and SM clocks are printed with the numbers.  Needs the GPU: there is
no CPU path.
usage: python scripts/bench_segment.py [out.json]"""
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
from automl_b200 import ops  # noqa: E402
from bench_ragged_serving import BATCH, MIX, MODEL, NREQ, SIZE  # noqa: E402

REQS, ROUNDS, WARMUP = 12, 5, 2
LAUNCHES = 200
HBM_TBS = 3.35          # H100 SXM data sheet


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


def bench_stream(driver, requests):
  reqs = [requests[i % NREQ] for i in range(REQS)]
  for _ in range(WARMUP):
    list(driver.segment_stream(reqs))
  rates = []
  for _ in range(ROUNDS):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = sum(len(m) for m in driver.segment_stream(reqs))
    rates.append(n / (time.perf_counter() - t0))
  return {'config': '%s %d^2 batch %d heads=[segmentation], sizes from the COCO-like mix'
                    % (MODEL, SIZE, BATCH),
          'windows': '%d x %d requests, three in flight' % (ROUNDS, REQS),
          'segment_stream_images_per_s': round(statistics.median(rates), 1),
          'min_max': [round(min(rates), 1), round(max(rates), 1)]}


def bench_kernel(driver, images):
  shapes = [im.shape[:2] for im in images]
  masks = driver.segment_images(images)          # leaves this request's logits in the engine
  eng = driver._engines[len(images)]             # pylint: disable=protected-access
  c = driver.config.seg_num_classes
  f = 2 ** (driver.config.min_level - 1)
  table, total = inference.seg_mask_table(shapes, SIZE)
  tb = torch.from_numpy(table).cuda()
  out = torch.empty(total, dtype=torch.uint8, device='cuda')
  max_hw = tuple(int(v) for v in np.max(np.asarray(shapes), axis=0))
  launch = lambda: ops.seg_masks(eng.seg_out, c, f, tb, max_hw, out)
  for _ in range(10):
    launch()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(LAUNCHES):
    launch()
  e1.record()
  torch.cuda.synchronize()
  us = e0.elapsed_time(e1) / LAUNCHES * 1e3
  packed = np.concatenate([m.ravel() for m in masks])
  same = bool(np.array_equal(out.cpu().numpy(), packed))
  hs, ws, ld = eng.seg_out.shape[1:]
  cells = 0
  for h, w, sh, sw in table[:, 2:].astype(np.int64):
    cy = np.minimum((2 * np.arange(h) + 1) * sh // (2 * h * f), hs - 1)
    cx = np.minimum((2 * np.arange(w) + 1) * sw // (2 * w * f), ws - 1)
    cells += len(np.unique(cy)) * len(np.unique(cx))
  nbytes = cells * 2 * ld + table.nbytes + total
  return {'kernel': 'seg_masks', 'config': 'D0 %d^2 batch %d, C=%d, logits [%d, %d, %d, %d] fp16'
                                           % (SIZE, BATCH, c, BATCH, hs, ws, ld),
          'us': round(us, 2), 'mask_MB': round(total / 1e6, 3), 'MB': round(nbytes / 1e6, 3),
          'TB/s': round(nbytes / us / 1e6, 3),
          'share_of_3.35TB/s': round(nbytes / us / 1e6 / HBM_TBS, 3),
          'logits_MB_at_network_res': round(BATCH * hs * ws * ld * 2 / 1e6, 3),
          'launch_equals_served_masks': same}


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_segment.py needs an H100')
  gpu = _gpu()
  requests = _requests(np.random.default_rng(0))
  driver = inference.ServingDriver(MODEL, '_', batch_size=BATCH,
                                   model_params={'image_size': SIZE, 'heads': ['segmentation']})
  rows = [bench_stream(driver, requests), bench_kernel(driver, requests[0])]
  rows[0]['gpu'] = rows[1]['gpu'] = gpu
  for r in rows:
    print(json.dumps(r))
  rows.append({'gpu_after': _gpu()})
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
