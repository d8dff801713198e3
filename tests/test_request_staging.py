"""Host side of request staging (no GPU): staging.pack against a plain restatement for every offset
layout the driver and the classifier stage, and what decoded_images reports of a request."""
import numpy as np
import pytest
import torch

from automl_b200 import inference
from automl_b200 import staging
from automl_b200.efficientnetv2 import preprocessing

RAGGED = [(120, 161), (37, 300), (5, 7), (300, 300), (64, 48)]
UNIFORM = [(96, 127)] * 4
PAD = 0xA5
ODD = np.arange(15, dtype=np.int32).reshape(5, 3)    # 60 bytes: the next table needs padding


def _images(shapes, seed):
  rng = np.random.default_rng(seed)
  return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def _offsets(table):
  return table[:, :2].copy().view(np.int64)[:, 0]


def _layout(name):
  """(images, the layout's own table, image offsets) as the driver or the classifier builds them."""
  if name == 'classifier':
    images = _images(RAGGED, 1)
    desc, _ = preprocessing.image_table(RAGGED, 224, True)
    return images, desc, _offsets(desc)
  if name == 'ragged':
    images = _images(RAGGED, 2)
    desc, _, _ = inference.preprocess_table(RAGGED, 512)
    return images, desc, _offsets(desc)
  images = _images(UNIFORM, 3)       # uniform and mirrored: image i at byte i * h * w * 3
  h, w = UNIFORM[0]
  desc, _, _ = inference.preprocess_table(UNIFORM, 512)
  desc[:, :2] = (np.arange(len(UNIFORM), dtype=np.int64) * (h * w * 3)).view(np.int32).reshape(-1, 2)
  return images, desc, _offsets(desc)


def _restated(tables, images, offsets):
  """The staged bytes written out plainly: (head, table ranges, bytes; PAD where nothing is)."""
  out, ranges = bytearray(), []
  for t in tables:
    out += bytes([PAD]) * (-len(out) % 8)
    ranges.append((len(out), len(out) + t.nbytes))
    out += t.tobytes()
  out += bytes([PAD]) * (-len(out) % 16)
  head = len(out)
  body = bytearray([PAD]) * max(int(o) + im.size for o, im in zip(offsets, images))
  for im, o in zip(images, offsets):
    body[int(o):int(o) + im.size] = im.tobytes()
  return head, ranges, np.frombuffer(bytes(out + body), np.uint8)


@pytest.mark.parametrize('ntables', [0, 1, 2])
@pytest.mark.parametrize('layout', ['ragged', 'uniform', 'mirrored', 'classifier'])
def test_pack_equals_restatement(layout, ntables):
  images, desc, offsets = _layout(layout)
  if layout == 'uniform':            # a uniform detection request stages no table of its own
    own = [] if ntables < 2 else [inference.seg_mask_table(UNIFORM, 512)[0]]
    tables = [ODD] * (ntables - len(own)) + own
  else:
    tables = [[], [desc], [ODD, desc]][ntables]
  head, ranges, want = _restated(tables, images, offsets)
  host = np.full(len(want) + 64, PAD, np.uint8)
  got_head, got_ranges = staging.pack(host, tables, images, offsets)
  assert got_head == head and got_ranges == ranges
  np.testing.assert_array_equal(host[:len(want)], want)
  assert (host[len(want):] == PAD).all()                 # nothing past the last image
  assert head % 16 == 0 and all(a % 8 == 0 for a, _ in ranges)
  for t, (a, b) in zip(tables, ranges):
    np.testing.assert_array_equal(host[a:b].view(np.int32).reshape(t.shape), t)
  for im, o in zip(images, offsets):
    np.testing.assert_array_equal(host[head + o:head + o + im.size].reshape(im.shape), im)


def test_decoded_request_forms():
  images = _images(UNIFORM, 4)
  for request in (images, np.stack(images), torch.from_numpy(np.stack(images))):
    d = staging.decoded_images(request, n=len(images))
    assert d.shapes == UNIFORM and d.uniform and not d.pinned and not d.cuda
    assert all(np.array_equal(a, b) for a, b in zip(d.images, images))
  d = staging.decoded_images(images[:2] + _images([(5, 7)], 5))
  assert d.shapes == UNIFORM[:2] + [(5, 7)] and not d.uniform
  with pytest.raises(ValueError, match='expected 3 images'):
    staging.decoded_images(images, n=3)
