"""`efficientdet(features, model_name=None, config=None, **kwargs)` on the H100 path.

Same call surface as /root/reference/efficientdet/efficientdet_arch.py:547-577:
  * raises ValueError when neither model_name nor config is given;
  * a dict config is wrapped in hparams_config.Config; kwargs go through Config.override
    (unknown keys -> KeyError);
  * returns (class_outputs, box_outputs): dicts level -> [N, H_l, W_l, A*C] / [N, H_l, W_l, 4A]
    float32 tensors (channels_first configs get the NCHW transposes the reference applies).

Differences forced by the runtime: `features` is a float32 CUDA tensor (or anything
torch.as_tensor accepts; it is copied to the device), and variables are not created inside a
TF graph: pass them with `weights=` (dict keyed by reference variable names, Keras layouts).
Without `weights`, seeded synthetic weights are used, like `ckpt_path='_'` in the reference.
Engines are cached per (config, batch, weights object, device) in a small LRU that keeps the
weights object alive (clear_engines() empties it).
"""
import collections
import json

import torch

from automl_b200 import hparams_config
from automl_b200 import weights as weights_lib
from automl_b200.arch import DetArch
from automl_b200.engine import Engine

# key -> (engine, weights object).  The entry keeps the weights dict alive, so `id(weights)` in
# the key cannot be recycled by CPython for a different checkpoint while the entry exists; the
# cache is a small LRU so engines (device buffers + CUDA graphs) of configurations that are no
# longer used are released.
_ENGINE_CACHE = collections.OrderedDict()
ENGINE_CACHE_SIZE = 4


def clear_engines():
  """Drops every cached engine (their device buffers and graphs are freed with them)."""
  _ENGINE_CACHE.clear()


def resolve_config(model_name=None, config=None, **kwargs):
  if not config and not model_name:
    raise ValueError('please specify either model name or config')
  if not config:
    config = hparams_config.get_efficientdet_config(model_name)
  elif isinstance(config, dict):
    config = hparams_config.Config(config)
  if kwargs:
    config.override(kwargs)
  return config


def get_engine(config, batch_size, weights=None, device='cuda:0', **engine_kwargs):
  """Engine for (config, batch, weights OBJECT, device).  The weights dict is treated as
  immutable once passed: edit a copy (a new dict is a new cache key), or call clear_engines()."""
  key = (json.dumps(config.as_dict(), sort_keys=True, default=str), int(batch_size),
         id(weights) if weights is not None else None, str(device),
         tuple(sorted(engine_kwargs.items())))
  hit = _ENGINE_CACHE.get(key)
  if hit is not None and hit[1] is weights:
    _ENGINE_CACHE.move_to_end(key)
    return hit[0]
  w = weights if weights is not None else weights_lib.synthetic_weights(DetArch(config), seed=0)
  eng = Engine(config, w, batch_size, device=device, **engine_kwargs)
  _ENGINE_CACHE[key] = (eng, weights)
  _ENGINE_CACHE.move_to_end(key)
  while len(_ENGINE_CACHE) > ENGINE_CACHE_SIZE:
    _ENGINE_CACHE.popitem(last=False)
  return eng


def _detection_only(config):
  """The legacy graph (efficientdet_arch.py:547-577) builds the class / box nets whatever
  config.heads says and has no segmentation head (that one is EfficientDetNet's,
  automl_b200/efficientdet_keras.py)."""
  if list(config.get('heads', None) or ['object_detection']) == ['object_detection']:
    return config
  config = hparams_config.Config(config.as_dict())
  config.heads = ['object_detection']
  return config


def efficientdet(features, model_name=None, config=None, weights=None, device='cuda:0',
                 **kwargs):
  """Build + run the EfficientDet network; see module docstring."""
  config = _detection_only(resolve_config(model_name, config, **kwargs))
  x = torch.as_tensor(features)
  if config.data_format == 'channels_first':
    x = x.permute(0, 2, 3, 1)
  eng = get_engine(config, x.shape[0], weights=weights, device=device)
  cls_out, box_out = eng.forward(x.contiguous())
  cls_out = {l: t.float() for l, t in cls_out.items()}
  box_out = {l: t.float() for l, t in box_out.items()}
  if config.data_format == 'channels_first':
    cls_out = {l: t.permute(0, 3, 1, 2) for l, t in cls_out.items()}
    box_out = {l: t.permute(0, 3, 1, 2) for l, t in box_out.items()}
  return cls_out, box_out
