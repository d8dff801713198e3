"""One serving request on its way to the device, for ServingDriver and EffNetV2Model.classify.

A request is decoded uint8 images.  `decoded_images` checks it.  `StagingSlot.stage` writes its int32
tables and its images into one pinned buffer, in the layout `pack` defines, and uploads that buffer
in one H2D copy on a copy stream.  A request already in pinned memory is copied without packing, and
one on the device is read in place.  Each slot's events order the reuse of its two buffers, so
requests on different slots overlap.  `pipelined` keeps a number of submitted requests in flight.
"""
import collections

import numpy as np
import torch


class Decoded(collections.namedtuple('Decoded', ['images', 'shapes', 'uniform', 'pinned', 'cuda'])):
  """A checked request.  `shapes` [(h, w), ...] of its images and `uniform` whether they are all equal.
  `images` is the request itself, a contiguous uint8 [N, h, w, 3] tensor, when it is in pinned
  memory (`pinned`) or on the device (`cuda`); otherwise it is the list of uint8 [h, w, 3] numpy
  arrays to pack."""


def decoded_images(image_arrays, n=None, device=None):
  """Checks one request of decoded images: a list of uint8 [h, w, 3] arrays (sizes may differ), a
  uint8 [N, h, w, 3] numpy array or CPU tensor (pinned or not), or such a tensor on `device` (None:
  the current device).  Raises ValueError for an empty request, a count other than `n` (when not
  None), an image that is not uint8 [h, w, 3], and a CUDA tensor on another device."""
  pinned = cuda = False
  if isinstance(image_arrays, torch.Tensor):
    t = image_arrays
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[3] != 3:
      raise ValueError('expected a uint8 [N, h, w, 3] tensor, got %s %s' % (t.dtype, tuple(t.shape)))
    if t.is_cuda:
      want = torch.device('cuda' if device is None else device)
      if want.index is None:
        want = torch.device('cuda', torch.cuda.current_device())
      if t.device != want:
        raise ValueError('images are on %s, the request is served on %s' % (t.device, want))
      images, cuda = t, True
    elif t.is_pinned() and t.is_contiguous():
      images, pinned = t, True
    else:
      images = list(t.numpy())
    shapes = [tuple(int(v) for v in t.shape[1:3])] * t.shape[0]
  else:
    images = [np.asarray(im) for im in image_arrays]
    for im in images:
      if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
        raise ValueError('expected uint8 [h, w, 3] images, got %s %s' % (im.dtype, im.shape))
    shapes = [im.shape[:2] for im in images]
  if not shapes:
    raise ValueError('empty request')
  if n is not None and len(shapes) != n:
    raise ValueError('expected %d images, got %d' % (n, len(shapes)))
  if cuda:
    images = images.contiguous()
  return Decoded(images, shapes, len(set(shapes)) == 1, pinned, cuda)


def _layout(tables):
  """(head, [(start, end) of each table]): the tables back to back at 8-byte aligned offsets, the
  head padded to 16 bytes."""
  ranges, pos = [], 0
  for t in tables:
    pos = (pos + 7) // 8 * 8
    ranges.append((pos, pos + t.nbytes))
    pos += t.nbytes
  return (pos + 15) // 16 * 16, ranges


def pack(host_u8, tables, images, offsets):
  """Writes a request into the uint8 buffer `host_u8`: the int32 `tables`, each at an 8-byte aligned
  offset, then image i at byte head + offsets[i], the head being the tables' bytes padded to 16.
  Bytes between them are left as they are.  Returns (head, [(start, end) of each table])."""
  head, ranges = _layout(tables)
  for t, (a, b) in zip(tables, ranges):
    host_u8[a:b] = t.view(np.uint8).ravel()
  for im, off in zip(images, offsets):
    host_u8[head + off:head + off + im.size] = im.reshape(-1)
  return head, ranges


def grow(buf, nbytes, **kw):
  """`buf` if it holds `nbytes`, else a new uint8 buffer of at least twice its size."""
  if buf is not None and buf.numel() >= nbytes:
    return buf
  return torch.empty(max(nbytes, 2 * buf.numel() if buf is not None else 0), dtype=torch.uint8, **kw)


class StagingSlot(object):
  """The staging of one in-flight request: a pinned buffer and its device twin, each holding the
  request's tables then its images as `pack` lays them out.  ev_h2d marks the H2D copy that read
  the pinned buffer, ev_raw_free the last kernel that read the device buffer (`release`)."""

  def __init__(self, device):
    self.device = device
    self.host = self.dev = None
    self.ev_h2d, self.ev_raw_free = torch.cuda.Event(), torch.cuda.Event()

  def stage(self, copy_stream, tables, request, offsets):
    """Uploads the int32 `tables` and the images of the Decoded `request`, image i at byte
    offsets[i] of the image region, in one H2D on `copy_stream`, and makes the current stream wait
    for it.  Returns (device views of the tables, the uint8 image region), valid until the slot's
    next request: a CUDA tensor request is that region itself, never copied."""
    main = torch.cuda.current_stream()
    head, ranges = _layout(tables)
    images = request.images
    packing = not (request.pinned or request.cuda)
    if packing:
      total = max((int(off) + im.size for off, im in zip(offsets, images)), default=0)
    else:
      total = images.numel()
    staged = head + (total if packing else 0)
    need = head + (0 if request.cuda else total)
    self.ev_h2d.synchronize()             # the slot's previous H2D has read the pinned buffer
    self.host = grow(self.host, staged, pin_memory=True)
    if self.dev is None or self.dev.numel() < need:
      main.synchronize()                  # no queued kernel still reads the old buffer
      self.dev = grow(self.dev, need, device=self.device)
    pack(self.host.numpy(), tables, images if packing else [], offsets)
    with torch.cuda.stream(copy_stream):
      copy_stream.wait_event(self.ev_raw_free)   # the slot's previous request has been read
      if staged:
        self.dev[:staged].copy_(self.host[:staged], non_blocking=True)
      if request.pinned:
        self.dev[head:need].copy_(images.view(-1), non_blocking=True)
      self.ev_h2d.record(copy_stream)
    main.wait_event(self.ev_h2d)
    views = [self.dev[a:b].view(torch.int32).view(t.shape) for t, (a, b) in zip(tables, ranges)]
    return views, (images.view(-1) if request.cuda else self.dev[head:need])

  def release(self):
    """Call after the last kernel that reads the staged buffer: the slot's next H2D waits for it."""
    self.ev_raw_free.record(torch.cuda.current_stream())


def pipelined(submit, batches, depth):
  """Yields submit(batch).result() for each of `batches`, in order, keeping `depth` submitted
  requests in flight."""
  pending = collections.deque()
  for batch in batches:
    pending.append(submit(batch))
    if len(pending) >= depth:
      yield pending.popleft().result()
  while pending:
    yield pending.popleft().result()
