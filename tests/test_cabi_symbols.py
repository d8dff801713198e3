"""The C-ABI library builds for sm_90a, loads without a GPU, and exports every symbol that
include/automl_b200.h declares (and ctypes signatures exist for all of them)."""
import ctypes
import os
import re

from automl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
  with open(os.path.join(ROOT, 'include', 'automl_b200.h')) as f:
    text = f.read()
  text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
  return sorted(set(re.findall(r'\b(edet_[a-z0-9_]+)\s*\(', text)))


def test_library_exports_every_declared_symbol():
  import __graft_entry__
  __graft_entry__.build()
  names = _declared_symbols()
  assert len(names) >= 12
  lib = ctypes.CDLL(_lib.LIB_PATH)
  for name in names:
    assert hasattr(lib, name), 'missing export %s' % name
    assert name in _lib.SIGNATURES, 'no ctypes signature for %s' % name
  assert sorted(_lib.SIGNATURES) == names
  assert _lib.load().edet_version() >= 100


def test_no_product_import_of_oracle():
  """The oracle is test infrastructure: nothing under automl_b200/ may import it."""
  pkg = os.path.join(ROOT, 'automl_b200')
  for dirpath, _, files in os.walk(pkg):
    for fn in files:
      if fn.endswith('.py'):
        with open(os.path.join(dirpath, fn)) as f:
          src = f.read()
        assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), fn


def _declared_prototypes():
  """name -> list of parameter declarations, parsed from the header (comments stripped)."""
  with open(os.path.join(ROOT, 'include', 'automl_b200.h')) as f:
    text = f.read()
  text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
  protos = {}
  for m in re.finditer(r'\b(edet_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;', text, flags=re.S):
    params = [p.strip() for p in m.group(2).replace('\n', ' ').split(',')]
    if params in ([''], ['void']):
      params = []
    protos[m.group(1)] = params
  return protos


def test_ctypes_signatures_match_header_prototypes():
  """The ctypes binding (what a reference maintainer would vendor, INTEGRATION.md) has, for every
  entry point, as many arguments as the header prototype, pointers where the header has pointers
  or the stream handle, and c_int / c_float where it has scalars."""
  protos = _declared_prototypes()
  assert sorted(protos) == sorted(_lib.SIGNATURES)
  for name, params in protos.items():
    _, argtypes = _lib.SIGNATURES[name]
    assert len(argtypes) == len(params), (name, len(argtypes), params)
    for decl, ct in zip(params, argtypes):
      is_ptr = '*' in decl or decl.startswith('edet_stream_t')
      if is_ptr:
        assert ct is ctypes.c_void_p or hasattr(ct, 'contents') or ct is ctypes.c_char_p, (name, decl, ct)
      elif decl.startswith('float'):
        assert ct is ctypes.c_float, (name, decl, ct)
      elif decl.startswith('int'):
        assert ct is ctypes.c_int, (name, decl, ct)
