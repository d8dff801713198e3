"""Generates tests/golden/classify_configs.json: the eval pre-process settings the REAL reference
config gives every registered EfficientNet V1 / V2 classifier, read from the unmodified
/root/reference/efficientnetv2/effnetv2_configs.py::get_model_config under the recording
TensorFlow stand-in (tests/golden/tf_stub.py; the config module only needs `tf` importable):
  augname   cfg.data.augname ('effnetv1_*' selects the legacy bicubic recipe,
            preprocessing.py:133)
  isize     cfg.eval.isize (infer.py:64: the default image size of the eval pre-process)
Run from the repo root:
  python tests/golden/make_classify_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/efficientnetv2'

MODELS = ['efficientnet-b%d' % i for i in range(9)] + ['efficientnet-l2'] + [
    'efficientnetv2-%s' % s for s in ('s', 'm', 'l', 'xl', 'b0', 'b1', 'b2', 'b3')]


def main():
  sys.path.insert(0, HERE)
  import tf_stub  # pylint: disable=g-import-not-at-top
  tf_stub.install()
  sys.path.insert(0, REF)
  import effnetv2_configs  # pylint: disable=g-import-not-at-top
  out = {}
  for model in MODELS:
    cfg = effnetv2_configs.get_model_config(model)
    out[model] = {'augname': cfg.data.augname, 'isize': cfg.eval.isize}
  path = os.path.join(os.environ.get('CLASSIFY_GOLDEN_OUT', HERE), 'classify_configs.json')
  with open(path, 'w') as f:
    json.dump(out, f, sort_keys=True, indent=1)
    f.write('\n')
  print('wrote', path, len(out), 'entries')


if __name__ == '__main__':
  main()
