"""The inventory of cross-stream hand-offs: every wait_event, wait_stream and synchronize() call in
the engine, the serving driver, request staging and the EfficientNet V1/V2 classifier must be listed
in tests/test_gpu_stream_handoffs.py's HANDOFFS, with the stall case that exercises it and either
the control that drops it or the reason it has none.  A hand-off added without a test fails here,
on any machine."""
import ast
import collections
import os

import test_gpu_stream_handoffs as handoffs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODULES = ('engine.py', 'inference.py', 'staging.py', 'efficientnetv2/effnetv2_model.py')
WAITS = ('wait_event', 'wait_stream', 'synchronize')
# the timing loop behind Engine.profile_ops synchronises the device between its event pairs;
# it orders no hand-off between streams
OUT_OF_SCOPE = {('engine.py', 'Engine._profile_ops')}


def inventory():
  """[(module, qualified function, call source)] of every wait in MODULES, in source order."""
  found = []
  for module in MODULES:
    with open(os.path.join(ROOT, 'automl_b200', module)) as f:
      tree = ast.parse(f.read())

    def walk(node, scope):
      for child in ast.iter_child_nodes(node):
        if isinstance(child, (ast.FunctionDef, ast.ClassDef)):
          walk(child, scope + [child.name])
          continue
        if (isinstance(child, ast.Call) and isinstance(child.func, ast.Attribute)
            and child.func.attr in WAITS):
          name = '.'.join(scope)
          if (module, name) not in OUT_OF_SCOPE:
            found.append((module, name, ast.unparse(child)))
        walk(child, scope)
    walk(tree, [])
  return found


def test_every_handoff_is_listed():
  listed = collections.Counter((m, f, c) for m, f, c, _, _ in handoffs.HANDOFFS)
  found = collections.Counter(inventory())
  assert sorted((found - listed).elements()) == [], 'waits without an entry in HANDOFFS'
  assert sorted((listed - found).elements()) == [], 'HANDOFFS entries no source has'


def test_every_entry_names_its_case_and_its_control_or_reason():
  tests = {n for n in dir(handoffs) if n.startswith('test_')}
  for module, function, call, case, control in handoffs.HANDOFFS:
    assert case in tests, (call, case)
    assert control in tests or (control.startswith('no control: ') and len(control) > 40), (call, control)
  controls = {c for *_, c in handoffs.HANDOFFS if c in tests}
  assert controls == {n for n in tests if n.startswith('test_control_')}


def test_profile_ops_is_left_out_by_name():
  """Engine._profile_ops really is where profile_ops' device synchronisations are."""
  everything = []
  saved = set(OUT_OF_SCOPE)
  OUT_OF_SCOPE.clear()
  try:
    everything = inventory()
  finally:
    OUT_OF_SCOPE.update(saved)
  left_out = [c for m, f, c in everything if (m, f) in saved]
  assert left_out == ['torch.cuda.synchronize()'] * 3
