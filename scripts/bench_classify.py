"""Measures the classification serving path from decoded images:

  * the eval pre-process launch (edet_cls_preprocess) for EfficientNetV2-S at 384 x 384, batch
    128, from 500 x 375 sources (bilinear, no crop), and for EfficientNetV2-B0 at 224 x 224,
    batch 128, from the same sources (bicubic, center crop); algorithmic bytes = the crop
    footprint read (3 bytes per pixel) + 12 S^2 written per image, over the launch time;
  * the softmax top-k launch (edet_softmax_topk, k = 5) at C = 1000 and 21 843, batch 1 and 128;
  * EfficientNetV2-S 384 batch 128 end to end: classify_stream (pinned uint8 500 x 375 batches in,
    top-5 out) against serve_stream (pinned float32 384 x 384 batches in, logits out), in
    alternating windows of REQS requests, ROUNDS windows each: images/s median and [min, max].

Launch times are CUDA-event windows over LAUNCH_REPLAYS replays of a CUDA graph holding COPIES
launches on separate inputs.  Prints the GPU's name and power limit with the numbers.  Needs the
GPU: there is no CPU path.
usage: python scripts/bench_classify.py [out.json]"""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automl_b200 import ops  # noqa: E402
from automl_b200.efficientnetv2 import effnetv2_model  # noqa: E402
from automl_b200.efficientnetv2 import preprocessing  # noqa: E402

SRC_H, SRC_W, BATCH = 375, 500, 128
COPIES, LAUNCH_REPLAYS = 4, 100
REQS, ROUNDS, WARMUP = 8, 7, 3


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


def _launch_us(fns):
  for fn in fns:
    fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for fn in fns:
      fn()
  _window(g.replay, 10)
  return _window(g.replay, LAUNCH_REPLAYS) / len(fns) * 1e3


def bench_preprocess(name, size, legacy):
  rng = np.random.default_rng(0)
  dev = 'cuda:0'
  desc, total = preprocessing.image_table([(SRC_H, SRC_W)] * BATCH, size, legacy)
  d = torch.from_numpy(desc).to(dev)
  raws = [torch.from_numpy(rng.integers(0, 256, size=total, dtype=np.uint8)).to(dev)
          for _ in range(COPIES)]
  out = torch.empty((BATCH, size, size, 3), dtype=torch.float32, device=dev)
  table = preprocessing.device_table(dev) if legacy else None
  mode = ops.CLS_BICUBIC if legacy else ops.CLS_BILINEAR
  us = _launch_us([lambda r=r: ops.cls_preprocess(r, d, out, mode, table) for r in raws])
  _, _, ch, cw = preprocessing.crop_window(SRC_H, SRC_W, size, legacy)
  nbytes = BATCH * (3 * ch * cw + 12 * size * size)
  return {'kernel': 'cls_preprocess', 'config': '%s %d^2 batch %d from %dx%d, %s' % (
      name, size, BATCH, SRC_W, SRC_H, 'bicubic, crop %d' % ch if legacy else
      ('bilinear, crop %d' % ch if ch != SRC_H else 'bilinear, no crop')),
          'us': round(us, 2), 'MB': round(nbytes / 1e6, 3), 'TB/s': round(nbytes / us / 1e6, 3)}


def bench_topk(c, n, k=5):
  g = torch.Generator(device='cuda:0').manual_seed(c + n)
  logits = [torch.randn((n, c), generator=g, device='cuda:0') for _ in range(COPIES)]
  probs = torch.empty((n, k), device='cuda:0')
  classes = torch.empty((n, k), dtype=torch.int32, device='cuda:0')
  us = _launch_us([lambda x=x: ops.softmax_topk(x, probs, classes) for x in logits])
  return {'kernel': 'softmax_topk', 'config': 'C %d batch %d k %d' % (c, n, k), 'us': round(us, 2),
          'MB': round(4 * n * c / 1e6, 3)}


def bench_end_to_end():
  name, size = 'efficientnetv2-s', 384
  arch = effnetv2_model.EffNetV2Arch(name)
  w = effnetv2_model.synthetic_weights(arch, 0, include_top=True)
  model = effnetv2_model.get_model(name, include_top=True, weights=w, batch_size=BATCH,
                                   image_size=size)
  rng = np.random.default_rng(1)
  raw = [torch.from_numpy(rng.integers(0, 256, size=(BATCH, SRC_H, SRC_W, 3), dtype=np.uint8)).pin_memory()
         for _ in range(2)]
  flt = [torch.from_numpy(rng.uniform(-1, 1, size=(BATCH, size, size, 3)).astype(np.float32)).pin_memory()
         for _ in range(2)]

  def classify():
    for _ in model.classify_stream([raw[i % 2] for i in range(REQS)], top_k=5):
      pass

  def serve():
    for _ in model.serve_stream([flt[i % 2] for i in range(REQS)]):
      pass

  arms = {'classify_stream': classify, 'serve_stream': serve}
  for fn in arms.values():
    for _ in range(WARMUP):
      fn()
  rates = {k: [] for k in arms}
  for _ in range(ROUNDS):
    for key, fn in arms.items():
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      fn()
      torch.cuda.synchronize()
      rates[key].append(REQS * BATCH / (time.perf_counter() - t0))
  row = {'config': '%s %d^2 batch %d' % (name, size, BATCH),
         'windows': '%d x %d requests each, alternating' % (ROUNDS, REQS),
         'h2d_bytes_per_request': {'classify_stream': BATCH * SRC_H * SRC_W * 3 + 32 * BATCH,
                                   'serve_stream': BATCH * size * size * 12},
         'd2h_bytes_per_request': {'classify_stream': BATCH * 5 * 8, 'serve_stream': BATCH * 1000 * 4}}
  for key, v in rates.items():
    row[key + '_images_per_s'] = round(statistics.median(v), 1)
    row[key + '_min_max'] = [round(min(v), 1), round(max(v), 1)]
  return row


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_classify.py needs an H100')
  gpu = _gpu()
  rows = [bench_preprocess('efficientnetv2-s', 384, False), bench_preprocess('efficientnetv2-b0', 224, True)]
  rows += [bench_topk(c, n) for c in (1000, 21843) for n in (1, 128)]
  rows.append(bench_end_to_end())
  for r in rows:
    r['gpu'] = gpu
    print(json.dumps(r))
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
