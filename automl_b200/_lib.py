"""ctypes binding of the C-ABI in include/automl_b200.h.

The CUDA library is the product: if it cannot be loaded this module raises — there is no CPU or
PyTorch fallback for any op of the path.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'csrc', 'libautoml_b200.so')

c_void_p, c_int, c_float, c_size_t = (ctypes.c_void_p, ctypes.c_int, ctypes.c_float,
                                      ctypes.c_size_t)

RS_SAME, RS_UP, RS_DOWN = 0, 1, 2
PW_TCGEN05, PW_SIMT = 0, 1
NMS_HARD, NMS_DIOU, NMS_GAUSSIAN, NMS_LINEAR = 0, 1, 2, 3
CLS_BILINEAR, CLS_BICUBIC = 0, 1


class FuseInput(ctypes.Structure):
  """edet_fuse_input."""
  _fields_ = [('ptr', c_void_p), ('h', c_int), ('w', c_int), ('mode', c_int),
              ('pool_h', c_int), ('pool_w', c_int), ('stride_h', c_int), ('stride_w', c_int),
              ('weight', c_float)]


# name -> (restype, argtypes); every symbol include/automl_b200.h declares.
SIGNATURES = {
    'edet_version': (c_int, []),
    'edet_last_error': (ctypes.c_char_p, []),
    'edet_set_option': (c_int, [ctypes.c_char_p, c_int]),
    'edet_get_option': (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int)]),
    'edet_device_info': (c_int, [ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    'edet_sched_bind': (c_int, [c_void_p, c_int]),
    'edet_last_sched_slot': (c_int, [ctypes.POINTER(c_void_p)]),
    'edet_preprocess': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                ctypes.POINTER(c_float), ctypes.POINTER(c_float),
                                ctypes.POINTER(c_float), c_void_p]),
    'edet_preprocess_ragged': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                       ctypes.POINTER(c_float), ctypes.POINTER(c_float), c_void_p]),
    'edet_preprocess_mirrored': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                         ctypes.POINTER(c_float), ctypes.POINTER(c_float), c_void_p]),
    'edet_preprocess_float': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                      ctypes.POINTER(c_float), ctypes.POINTER(c_float),
                                      ctypes.POINTER(c_float), c_void_p]),
    'edet_stem_conv': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                               c_int, c_int, c_void_p]),
    'edet_pointwise_conv': (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int,
                                    c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p]),
    'edet_class_argmax': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'edet_depthwise_conv': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                    c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'edet_conv2d': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                            c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'edet_conv2d_transpose': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p,
                                      c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                      c_void_p]),
    'edet_mbconv_expand_dw':(c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                      c_int, c_void_p]),
    'edet_se_fc': (c_int, [c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                           c_int, c_int, c_void_p]),
    'edet_fuse_dw': (c_int, [ctypes.POINTER(FuseInput), c_int, c_void_p, c_void_p, c_int, c_int,
                             c_int, c_int, c_int, c_void_p]),
    'edet_fuse_dw_channel': (c_int, [ctypes.POINTER(FuseInput), c_int, c_void_p, c_void_p, c_void_p,
                                     c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'edet_sepconv': (c_int, [ctypes.POINTER(FuseInput), c_int, c_int, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'edet_max_pool': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                              c_int, c_int, c_void_p]),
    'edet_global_avg_pool': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'edet_dense': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'edet_cls_preprocess': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p]),
    'edet_softmax_topk': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'edet_seg_masks': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                               c_int, c_void_p, c_void_p]),
    'edet_pre_nms': (c_int, [ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p),
                             ctypes.POINTER(c_int), c_int, c_int, c_int, c_int, c_int, c_void_p,
                             c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    'edet_pre_nms_topk': (c_int, [ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p),
                                  ctypes.POINTER(c_int), c_int, c_int, c_int, c_int, c_int, c_void_p,
                                  c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    'edet_nms_work_bytes': (c_size_t, [c_int, c_int]),
    'edet_nms_v5': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                            c_float, c_float, c_float, c_float, c_float, c_void_p, c_void_p,
                            c_void_p, c_void_p, c_void_p]),
    'edet_per_class_nms': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                   c_int, c_int, c_int, c_float, c_float, c_float, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_void_p]),
    'edet_wbf': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p,
                         c_void_p, c_void_p]),
}

_lib = None


class EdetError(RuntimeError):
  pass


def load():
  """Loads libautoml_b200.so (raises RuntimeError when it is missing: build it first with
  `python -m automl_b200.build` / __graft_entry__.build())."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise RuntimeError(
        'automl_b200 CUDA library not found at %s; run `python -m automl_b200.build`. '
        'There is no CPU fallback for this path.' % LIB_PATH)
  lib = ctypes.CDLL(LIB_PATH)
  for name, (restype, argtypes) in SIGNATURES.items():
    fn = getattr(lib, name)  # AttributeError if the symbol is missing
    fn.restype = restype
    fn.argtypes = argtypes
  _lib = lib
  # A/B switches from the environment (scripts/, bench.py runs): EDET_DW_IMPL, EDET_PW_TEAMS
  for env, opt in (('EDET_DW_IMPL', b'dw_impl'), ('EDET_PW_TEAMS', b'pw_teams'),
                   ('EDET_STEM_IMPL', b'stem_impl'), ('EDET_SEPCONV_IMPL', b'sepconv_impl'),
                   ('EDET_PW_SMEM_KB', b'pw_smem_kb'), ('EDET_PERSIST_SLACK', b'persist_slack'),
                   ('EDET_PW_SHARE_W', b'pw_share_w')):
    if os.environ.get(env):
      if lib.edet_set_option(opt, int(os.environ[env])) != 0:
        raise EdetError('bad %s=%s' % (env, os.environ[env]))
  return lib


def check(rc):
  if rc != 0:
    msg = load().edet_last_error()
    raise EdetError('automl_b200 call failed (%d): %s' % (rc, (msg or b'').decode()))


def call(name, *args):
  """Calls an int-returning entry point and raises EdetError on a non-zero status."""
  check(getattr(load(), name)(*args))
