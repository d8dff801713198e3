"""The programmatic-dependent-launch rule (common.cuh, DESIGN.md section 4) as far as the compiled
code can show it, without a GPU.

On sm_90a `griddepcontrol.launch_dependents` compiles to PREEXIT and `griddepcontrol.wait` to
ACQBULK.  In every kernel of libautoml_b200.so:
  - PREEXIT and ACQBULK come together: a kernel that lets the next one start must itself wait, and
    one that waits has no reason not to let the next one start;
  - the kernels with neither are exactly NON_PDL, so a new kernel is classified on purpose;
  - no global store, reduction or atomic, and no TMA store, comes before the first ACQBULK in
    instruction order: a kernel writes nothing the previous one may still read.
A generic ST before the wait may be a shared-memory store made through a generic pointer; SASS
cannot tell, so tests/test_gpu_pdl_chains.py settles those (and every read) on the GPU."""
import collections
import os
import re
import shutil
import subprocess

import pytest

# kernel families launched with <<<>>> (no PDL): the pre-processes and the post-NMS stages, which
# follow torch copies or host work, and the SIMT pointwise reference
NON_PDL = {
    'preprocess_kernel', 'cls_preprocess_kernel', 'softmax_topk_kernel', 'nms_v5_kernel',
    'nms_v5_fast_kernel', 'pre_nms_topk_kernel', 'per_class_nms_kernel',
    'per_class_soft_nms_kernel', 'pointwise_simt_kernel',
}
# global stores, reductions and atomics, and TMA stores / reductions
GLOBAL_WRITES = {'STG', 'RED', 'REDG', 'ATOMG', 'UTMASTG', 'UTMAREDG'}


def _cuobjdump():
  found = shutil.which('cuobjdump')
  if found:
    return found
  cand = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
  return cand if os.path.exists(cand) else None


def _family(mangled):
  """The unqualified function name of an Itanium-mangled kernel name (the last identifier of its
  nested name, before any template arguments): edet::dw_tile_kernel<3, 1, ...> -> dw_tile_kernel."""
  m = re.match(r'_ZN?(.*)', mangled)
  rest, last = m.group(1), None
  while True:
    d = re.match(r'(\d+)', rest)
    if not d:
      return last
    n = int(d.group(1))
    start = len(d.group(1))
    last = rest[start:start + n]
    rest = rest[start + n:]


def _is_global_write(ins):
  op = ins.split('.')[0]
  if op in GLOBAL_WRITES:
    return True
  # bulk copy, destination space first: UBLKCP.G.S stores shared memory to global memory
  return ins.startswith('UBLKCP.G.')


@pytest.fixture(scope='module')
def kernels():
  """mangled kernel name -> its SASS instructions (opcode with modifiers), in address order."""
  tool = _cuobjdump()
  if tool is None:
    pytest.skip('cuobjdump not found')
  import __graft_entry__
  lib = __graft_entry__.build()
  sass = subprocess.run([tool, '-sass', lib], stdout=subprocess.PIPE, text=True, check=True).stdout
  out = collections.OrderedDict()
  cur = None
  for line in sass.splitlines():
    m = re.match(r'\s*Function : (\S+)', line)
    if m:
      cur = out.setdefault(m.group(1), [])
      continue
    m = re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)', line)
    if cur is not None and m:
      cur.append(m.group(1))
  assert out, 'no kernels in %s' % lib
  return out


def _has(instrs, op):
  return any(i.split('.')[0] == op for i in instrs)


def test_family_names_parse(kernels):
  for mangled in kernels:
    fam = _family(mangled)
    assert fam and fam.endswith('_kernel'), (mangled, fam)


def test_every_kernel_that_triggers_also_waits(kernels):
  bad = sorted(_family(k) + ' ' + k for k, ins in kernels.items()
               if _has(ins, 'PREEXIT') != _has(ins, 'ACQBULK'))
  assert not bad, 'PREEXIT without ACQBULK or the reverse:\n' + '\n'.join(bad)


def test_kernels_without_pdl_are_the_listed_families(kernels):
  without = {_family(k) for k, ins in kernels.items()
             if not _has(ins, 'PREEXIT') and not _has(ins, 'ACQBULK')}
  with_pdl = {_family(k) for k, ins in kernels.items() if _has(ins, 'ACQBULK')}
  assert without == NON_PDL, ('kernels without PDL: %s, expected %s'
                              % (sorted(without), sorted(NON_PDL)))
  assert not without & with_pdl, 'a family launched both ways: %s' % sorted(without & with_pdl)


def test_no_global_write_before_the_first_wait(kernels):
  bad = []
  for k, ins in kernels.items():
    if not _has(ins, 'ACQBULK'):
      continue
    first = next(i for i, op in enumerate(ins) if op.split('.')[0] == 'ACQBULK')
    early = [op for op in ins[:first] if _is_global_write(op)]
    if early:
      bad.append('%s (%s): %s' % (_family(k), k, ', '.join(early)))
  assert not bad, 'global writes before griddepcontrol.wait:\n' + '\n'.join(bad)


def test_global_write_classifier():
  assert _is_global_write('STG.E.128')
  assert _is_global_write('REDG.E.ADD.64.STRONG.GPU')
  assert _is_global_write('ATOMG.E.ADD.STRONG.GPU')
  assert _is_global_write('UTMASTG.3D')
  assert _is_global_write('UBLKCP.G.S')
  assert not _is_global_write('UBLKCP.S.G')
  assert not _is_global_write('ATOMS.ADD')
  assert not _is_global_write('REDUX.SUM')
  assert not _is_global_write('STS.128')
