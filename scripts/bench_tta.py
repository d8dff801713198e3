"""Measures horizontal-flip test-time augmentation from decoded images: ServingDriver.serve_stream_tta
next to serve_stream, and the three launches TTA adds.

EfficientDet-D0 at 640 x 640, batch 32, seeded synthetic weights; each image's size is drawn from the
COCO-like mix of scripts/bench_ragged_serving.py.  Reported:
  * images/s through serve_stream_tta and serve_stream (three requests in flight), median and
    [min, max] over ROUNDS windows of REQS requests, after WARMUP windows, alternating the two;
  * CUDA-event times of edet_preprocess_mirrored (32 images -> 64 inputs), of edet_per_class_nms
    over the 64 images with the config's nms_configs, and of edet_wbf (2 models x 100 rows per
    image), each over back-to-back launches on the request's own buffers.
The GPU's name, power limit and SM clocks are printed with the numbers.  Needs the GPU: there is
no CPU path.
usage: python scripts/bench_tta.py [out.json]"""
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
from automl_b200 import staging  # noqa: E402
from bench_ragged_serving import BATCH, MIX, MODEL, NREQ, SIZE  # noqa: E402

REQS, ROUNDS, WARMUP = 12, 5, 1
LAUNCHES = {'preprocess_mirrored': 100, 'per_class_nms': 10, 'wbf': 100}


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
  streams = {'serve_stream_tta': driver.serve_stream_tta, 'serve_stream': driver.serve_stream}
  for fn in streams.values():
    for _ in range(WARMUP):
      list(fn(reqs))
  rates = {k: [] for k in streams}
  for _ in range(ROUNDS):
    for name, fn in streams.items():
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      n = sum(len(r) for r in fn(reqs))
      rates[name].append(n / (time.perf_counter() - t0))
  row = {'config': '%s %d^2 batch %d, sizes from the COCO-like mix' % (MODEL, SIZE, BATCH),
         'windows': '%d x %d requests, three in flight, the two streams alternating' % (ROUNDS, REQS)}
  for name, r in rates.items():
    row[name + '_images_per_s'] = round(statistics.median(r), 1)
    row[name + '_min_max'] = [round(min(r), 1), round(max(r), 1)]
  return row


def _time(launch, count):
  for _ in range(3):
    launch()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(count):
    launch()
  e1.record()
  torch.cuda.synchronize()
  return round(e0.elapsed_time(e1) / count * 1e3, 2)


def bench_kernels(driver, images):
  n = len(images)
  driver.serve_images_tta(images)
  tta = next(s.tta for s in driver._slots[2 * n] if s.tta is not None)  # pylint: disable=protected-access
  eng = driver._engines[2 * n]                   # pylint: disable=protected-access
  desc, total, _ = inference.preprocess_table([im.shape[:2] for im in images], SIZE)
  packed = np.zeros(total, np.uint8)
  staging.pack(packed, [], images, desc[:, :2].copy().view(np.int64)[:, 0])
  pk, ds = torch.from_numpy(packed).cuda(), torch.from_numpy(desc).cuda()
  mir = torch.empty_like(eng.input)
  nms = driver.config.as_dict()['nms_configs']
  pre = eng.pre_nms_only()
  det = torch.empty_like(tta.rows)
  cap = 2 * eng.max_output_size
  clusters = torch.empty(n, cap, 7, device='cuda')
  counts = torch.empty(n, dtype=torch.int32, device='cuda')
  launches = {
      'preprocess_mirrored': lambda: ops.preprocess_mirrored(pk, ds, mir, driver.mean_rgb,
                                                             driver.stddev_rgb),
      'per_class_nms': lambda: ops.per_class_nms(
          pre['boxes'], pre['scores'], pre['classes'], tta.ids, tta.scales,
          driver.config.num_classes, eng.max_output_size, nms['method'], nms.get('iou_thresh'),
          det, tta.keep, tta.valid, sigma=nms.get('sigma'),
          score_thresh=nms.get('score_thresh'), work=tta.work),
      'wbf': lambda: ops.wbf(det, 2, driver.config.num_classes, clusters, counts, 0b10,
                             tta.scales[:n], SIZE),
  }
  row = {'config': 'D0 %d^2 batch %d -> %d inputs, nms %s, %d anchors, %d rows per model'
                   % (SIZE, n, 2 * n, nms['method'], pre['scores'].shape[1], eng.max_output_size)}
  for name, fn in launches.items():
    row[name + '_us'] = _time(fn, LAUNCHES[name])
  row['preprocess_equals_served_input'] = bool(torch.equal(mir, eng.input))
  row['nms_equals_served_rows'] = bool(torch.equal(det, tta.rows))
  return row


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_tta.py needs an H100')
  gpu = _gpu()
  requests = _requests(np.random.default_rng(0))
  driver = inference.ServingDriver(MODEL, '_', batch_size=BATCH, model_params={'image_size': SIZE})
  rows = [bench_stream(driver, requests), bench_kernels(driver, requests[0])]
  for r in rows:
    r['gpu'] = gpu
    print(json.dumps(r))
  rows.append({'gpu_after': _gpu()})
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
