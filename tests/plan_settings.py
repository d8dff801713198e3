"""The option settings under which the pointwise GEMM (edet_pointwise_conv / edet_class_argmax) must
give the bits of the default plan: three consumer warpgroups, smaller shared-memory budgets, and a
pinned grid.  The grid is pinned with max_ctas = G, so the plan a setting selects depends only on
the shapes, not on which H100 runs the test; G = 1 makes one CTA wrap its work-unit ring and every
stage ring many times."""
import torch

from automl_b200._lib import EdetError

GRIDS = (1, 3, 8, 33)
SMEM_KB = (96, 128, 160, 192)
# (option, value); ('grid', G) sets max_ctas = G
SETTINGS = [('pw_teams', 3)] + [('pw_smem_kb', kb) for kb in SMEM_KB] + [('grid', g) for g in GRIDS]
# Every shape runs from this budget up with two consumers (include/automl_b200.h): 1 KiB alignment
# + two 24 KiB stages (64 x 64 A + streamed 128 x 64 W) per consumer + one 16 KiB slab set per
# consumer + 32.5 KiB of bias (nout 8256: 65 N tiles of 128) + 960 bytes of barriers and tile ring
# = 162.4 KiB.  With three consumers: three stages more and one slab set more, 226.4 KiB.
SMEM_FLOOR_KB = 163
SMEM_FLOOR_KB_3 = 227
# The budgets the hand-picked test shapes must all run at (they are narrower than nout 8192).
MUST_RUN_KB = 160


def setting_id(s):
  return '%s=%d' % s


def must_run(setting):
  name, value = setting
  return name != 'pw_smem_kb' or value >= MUST_RUN_KB


def reset(ops):
  for opt in ('pw_teams', 'pw_smem_kb', 'pw_share_w', 'persist_slack', 'max_ctas'):
    ops.set_option(opt, 0)


def apply(ops, setting):
  name, value = setting
  ops.set_option('max_ctas' if name == 'grid' else name, value)


def run_under(ops, setting, launch):
  """Runs launch() with `setting` applied; returns False if the plan was refused (EdetError)."""
  try:
    if setting is not None:
      apply(ops, setting)
    try:
      launch()
    except EdetError:
      return False
    torch.cuda.synchronize()
    return True
  finally:
    reset(ops)
