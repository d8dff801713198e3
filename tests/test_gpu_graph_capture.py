"""CUDA graph capture (lowering.capture_graph, used by Engine and EffNetV2Model) pauses Python's cyclic
garbage collector, so a dropped engine or model that the collector frees never destroys its CUDA
graphs or pinned buffers while another capture is underway, and restores the collector's state."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('enabled', [True, False])
def test_capture_pauses_the_collector(enabled):
  from automl_b200.lowering import capture_graph
  x = torch.zeros(4, device='cuda:0')
  seen = []

  def fn():
    seen.append(gc.isenabled())
    x.add_(1.0)

  was = gc.isenabled()
  (gc.enable if enabled else gc.disable)()
  try:
    torch.cuda.synchronize()
    g = capture_graph(fn)
    assert gc.isenabled() == enabled
  finally:
    (gc.enable if was else gc.disable)()
  g.replay()
  torch.cuda.synchronize()
  assert seen == [False]
  assert x.tolist() == [1.0] * 4          # the capture ran nothing; one replay added 1 once
