"""Generates tests/golden/seg_structure.json: the segmentation head's layers as the REAL reference
constructors build them, run under the recording TensorFlow stand-in (tests/golden/tf_stub.py).

For each model it instantiates /root/reference/efficientdet/tf2/efficientdet_keras.py::
EfficientDetNet(config=...) with heads = ['object_detection', 'segmentation'] (as
efficientdet_keras_test.py:41 does) and records every Keras layer SegmentationHead.__init__
(efficientdet_keras.py:647-692) creates, in creation order:

  ['conv_transpose', filters, kernel, stride, padding, use_bias]   (Conv2DTranspose)
  ['bn', name]                                                     (BatchNormalization)

together with the config values it depends on.  tests/test_segmentation_pins.py holds the
product's and the oracle's layer lists to exactly this.  Run from the repo root:
  python tests/golden/make_seg_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/efficientdet'

MODELS = ['efficientdet-d0', 'efficientdet-d1', 'efficientdet-lite0', 'efficientdet-d7x']


def _one(v):
  if isinstance(v, (list, tuple)):
    assert len(set(v)) == 1, v
    return v[0]
  return v


def seg_layers(log):
  start = [i for i, (cls, _, _) in enumerate(log) if cls == 'SegmentationHead']
  assert len(start) == 1, start
  out = []
  for cls, args, kw in log[start[0] + 1:]:
    kind = cls.split('.')[-1]
    if kind == 'Conv2DTranspose':
      filters = kw.get('filters', args[0] if args else None)
      kernel = kw.get('kernel_size', args[1] if len(args) > 1 else None)
      out.append(['conv_transpose', filters, _one(kernel), _one(kw.get('strides', 1)),
                  kw.get('padding', 'valid'), bool(kw.get('use_bias', True))])
    elif kind == 'BatchNormalization':
      out.append(['bn', kw.get('name')])
  return out


def main():
  sys.path.insert(0, HERE)
  import tf_stub
  tf_stub.install()
  sys.path.insert(0, REF)
  import hparams_config  # pylint: disable=g-import-not-at-top
  from tf2 import efficientdet_keras as ek  # pylint: disable=g-import-not-at-top

  out = {}
  for name in MODELS:
    config = hparams_config.get_efficientdet_config(name)
    config.heads = ['object_detection', 'segmentation']
    del tf_stub.LOG[:]
    ek.EfficientDetNet(config=config)
    out[name] = {'min_level': config.min_level, 'max_level': config.max_level,
                 'fpn_num_filters': config.fpn_num_filters, 'act_type': config.act_type,
                 'seg_num_classes': config.seg_num_classes, 'layers': seg_layers(tf_stub.LOG)}
    print(name, len(out[name]['layers']), 'layers')
  path = os.path.join(os.environ.get('SEG_GOLDEN_OUT', HERE), 'seg_structure.json')
  with open(path, 'w') as f:
    json.dump(out, f, sort_keys=True, indent=1)
    f.write('\n')
  print('wrote', path)


if __name__ == '__main__':
  main()
