"""BASELINE config 3: EfficientNetV2-S 384x384 backbone-only, batch 128, one H100 (not the bench.py
headline; a reported parity-case number).  CUDA graph replay, CUDA events, 20 steps after 5."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automl_b200.efficientnetv2 import effnetv2_model  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else 'efficientnetv2-s'
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 128
size = int(sys.argv[3]) if len(sys.argv) > 3 else 384
model = effnetv2_model.get_model(name, weights=None, batch_size=batch, image_size=size)
x = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, size=(batch, size, size, 3)).astype(np.float32)).cuda()
model(x)
for _ in range(5):
  model.run()
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
steps = 20
a.record()
for _ in range(steps):
  model.run()
b.record()
torch.cuda.synchronize()
ms = a.elapsed_time(b) / steps
# per-op (eager, one at a time)
evs = []
for nm, fn in model._ops:
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record(); fn(); e1.record(); evs.append((nm, e0, e1))
torch.cuda.synchronize()
kinds = {}
for (nm, e0, e1), info in zip(evs, model.op_info):
  k = kinds.setdefault(info['kind'], {'ms': 0.0, 'bytes': 0, 'flops': 0, 'launches': 0})
  k['ms'] += e0.elapsed_time(e1); k['bytes'] += info['bytes']; k['flops'] += info['flops']; k['launches'] += 1
flops = sum(i['flops'] for i in model.op_info)
print(json.dumps({
    'config': '%s %dx%d batch %d backbone + head conv, fp16 storage / fp32 accumulate, synthetic weights' % (name, size, size, batch),
    'images_per_s': batch / (ms / 1e3), 'ms_per_step': ms, 'TFLOPs': flops / (ms / 1e3) / 1e12,
    'GFLOP_per_image': flops / batch / 1e9,
    'per_kind': {k: {'ms': round(v['ms'], 3), 'GBps': round(v['bytes'] / max(v['ms'], 1e-9) / 1e6, 1),
                     'TFLOPs': round(v['flops'] / max(v['ms'], 1e-9) / 1e9, 1), 'launches': v['launches']}
                 for k, v in kinds.items()}}))
