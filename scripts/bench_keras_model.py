"""Measures EfficientDetModel (the TF2 Keras model: pre-process, network and global NMS in one call)
from uint8 and from float32 images, next to ServingDriver.serve_images, and the float32 pre-process.

EfficientDet-D0 at 640 x 640, batch 32 of 480 x 640 images held in host memory (numpy), seeded
synthetic weights.  Reported:
  * images/s of EfficientDetModel.__call__ on uint8 and on float32 images, and of
    ServingDriver.serve_images on the uint8 images: each call is synchronous (the model's results
    are on the device when the window's final synchronise returns, the driver's in host memory);
    median and [min, max] over ROUNDS windows of CALLS calls after WARMUP windows, the three
    alternating;
  * CUDA-event time per launch of edet_preprocess_float and, for comparison, edet_preprocess on the
    same images already on the device, over back-to-back launches, with the bytes each launch must
    move (12 h w in for float32 or 3 h w for uint8, 12 H W out, per image) and the rate that gives.
The GPU's name, power limit and SM clocks are printed with the numbers.  Needs the GPU: there is no
CPU path.
usage: python scripts/bench_keras_model.py [out.json]"""
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
from automl_b200 import hparams_config  # noqa: E402
from automl_b200 import inference  # noqa: E402
from automl_b200 import ops  # noqa: E402
from automl_b200.efficientdet_keras import EfficientDetModel  # noqa: E402

MODEL, SIZE, BATCH, RAW = 'efficientdet-d0', 640, 32, (480, 640)
CALLS, ROUNDS, WARMUP = 10, 5, 1
LAUNCHES = 200


def _gpu():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                         '--format=csv,noheader'],
                        stdout=subprocess.PIPE, text=True, check=True).stdout.strip()


def bench_calls(model, driver, u8, f32):
  calls = {
      'model_uint8': lambda: model(u8),
      'model_float32': lambda: model(f32),
      'serve_images_uint8': lambda: driver.serve_images(u8),
  }
  for fn in calls.values():
    for _ in range(WARMUP * CALLS):
      fn()
  torch.cuda.synchronize()
  rates = {k: [] for k in calls}
  for _ in range(ROUNDS):
    for name, fn in calls.items():
      t0 = time.perf_counter()
      for _ in range(CALLS):
        fn()
      torch.cuda.synchronize()
      rates[name].append(CALLS * BATCH / (time.perf_counter() - t0))
  row = {'config': 'D0 %d^2 batch %d from %dx%d host images, one synchronous call at a time'
                   % (SIZE, BATCH, RAW[0], RAW[1]),
         'windows': '%d x %d calls, the three alternating' % (ROUNDS, CALLS)}
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
  return e0.elapsed_time(e1) / count * 1e3


def bench_kernels(config, u8, f32):
  mean, std = inference._rgb3(config.mean_rgb), inference._rgb3(config.stddev_rgb)  # pylint: disable=protected-access
  du8, df32 = torch.from_numpy(u8).cuda(), torch.from_numpy(f32).cuda()
  out = torch.empty(BATCH, SIZE, SIZE, 3, device='cuda')
  ref = torch.empty_like(out)
  ops.preprocess(du8, ref, mean, std)
  ops.preprocess_float(df32, out, mean, std)
  row = {'config': 'batch %d, %dx%d -> %d^2' % (BATCH, RAW[0], RAW[1], SIZE),
         'float_equals_uint8_bits': bool(torch.equal(out.view(torch.int32), ref.view(torch.int32)))}
  pix_in, pix_out = BATCH * RAW[0] * RAW[1], BATCH * SIZE * SIZE
  for name, fn, nbytes in (
      ('preprocess_float', lambda: ops.preprocess_float(df32, out, mean, std), 12 * (pix_in + pix_out)),
      ('preprocess_uint8', lambda: ops.preprocess(du8, out, mean, std), 3 * pix_in + 12 * pix_out)):
    us = _time(fn, LAUNCHES)
    row[name + '_us'] = round(us, 2)
    row[name + '_bytes'] = nbytes
    row[name + '_GB_per_s'] = round(nbytes / us / 1e3, 1)
  return row


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_keras_model.py needs an H100')
  gpu = _gpu()
  config = hparams_config.get_efficientdet_config(MODEL)
  config.override(dict(image_size=SIZE))
  u8 = np.random.default_rng(0).integers(0, 256, size=(BATCH,) + RAW + (3,), dtype=np.uint8)
  f32 = u8.astype(np.float32)       # integral values: the model's float path gives the uint8 bits
  model = EfficientDetModel(config=config)
  driver = inference.ServingDriver(MODEL, '_', batch_size=BATCH, model_params={'image_size': SIZE})
  rows = [bench_calls(model, driver, u8, f32), bench_kernels(config, u8, f32)]
  for r in rows:
    r['gpu'] = gpu
    print(json.dumps(r))
  rows.append({'gpu_after': _gpu()})
  if len(sys.argv) > 1:
    with open(sys.argv[1], 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
