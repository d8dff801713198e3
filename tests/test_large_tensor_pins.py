"""The large-tensor cases of test_gpu_large_tensors, checked without a GPU: the batches at which each
registered model's largest activation passes 2^31 elements, and each case's layer, batch and
memory."""
import test_gpu_large_tensors as lt
from automl_b200.efficientnetv2 import effnetv2_model
from test_gpu_memory_bound_kernels import _det_arch, _pools, dw_shapes, fpn_shapes, pool_shapes

# model: (native size, elements of the largest per-image tensor, batch at which it reaches 2^31)
TABLE = {
    'efficientdet-d7x': (1536, 113246208, 19),    # blocks_4 expand
    'efficientdet-d7': (1536, 113246208, 19),     # blocks_3 expand
    'efficientdet-d6': (1280, 78643200, 28),
    'efficientdet-d5': (1280, 58982400, 37),
    'efficientnet-l2': (800, 69120000, 32),
    'efficientdet-d4': (1024, 37748736, 57),
    'efficientnet-b7': (600, 17280000, 125),
    'efficientnetv2-xl': (512, 4194304, 512),     # blocks_4 expand
    'efficientnetv2-l': (480, 3686400, 583),
    'efficientnetv2-s': (384, 1769472, 1214),
}


def test_crossing_batches_of_the_registered_models():
  assert lt.crossing_batches() == TABLE
  # at batch 32, D6-D7x and L2 need 64-bit element offsets and D5 64-bit fp16 byte offsets; at
  # batch 1024, V2-S needs 64-bit fp16 byte offsets (its elements pass 2^31 at 1214)
  assert all(TABLE[m][2] <= 32 for m in ('efficientdet-d6', 'efficientdet-d7', 'efficientdet-d7x',
                                         'efficientnet-l2'))
  assert TABLE['efficientdet-d5'][2] > 32 and 32 * TABLE['efficientdet-d5'][1] * 2 > lt.B31
  assert TABLE['efficientnetv2-s'][2] > 1024 and 1024 * TABLE['efficientnetv2-s'][1] * 2 > lt.B31


def test_fused_expand_is_counted_at_the_output_size():
  """A Fused-MBConv block's strided k x k expand conv writes its output at the block's output
  size: V2-S's blocks_2 (24 -> 96, stride 2 at 192 x 192) is 96 x 96 x 96, not 192 x 192 x 96."""
  v = effnetv2_model.EffNetV2Arch('efficientnetv2-s')
  b, h = [(b, h) for b, h in lt.backbone_maps(v.blocks, 384, lambda b: b.strides) if b.name == 'blocks_2'][0]
  assert (b.conv_type, b.strides, b.mid_filters, h) == (1, 2, 96, 192)
  assert lt.largest_tensor([b], 2 * h, 1, lambda b: b.strides) == (96 * 96 * 96, 'blocks_2 expand')


def test_cases_are_real_layers_that_cross():
  cases = lt.case_table()
  assert set(cases) == {'stem', 'dw_k3s1', 'dw_k5s2', 'mbconv', 'pw_rows', 'pw_image_w', 'pw_simt',
                        'conv_s1', 'conv_s2', 'convt', 'fuse_up', 'fuse_down', 'sepconv', 'max_pool',
                        'gap', 'preprocess', 'preprocess_ragged', 'softmax_topk',
                        'class_argmax', 'sepconv_tma', 'pre_nms', 'cls_preprocess'}
  for c in cases.values():
    b = lt.boundary_image(c)
    # element 2^31 of the crossing tensor lies inside image b, which is neither the first nor the last
    assert b * c.per_image < lt.B31 < (b + 1) * c.per_image, c.name
    assert 0 < b < c.batch - 1 and c.batch * c.per_image > lt.B31, c.name
    # each further crossing also lies inside an image of its own, neither the first nor the last
    extra = lt.extra_images(c)
    for (_, per_image, limit), e in zip(c.extra, extra):
      assert e * per_image < limit < (e + 1) * per_image and 0 < e < c.batch - 1, c.name
    assert len(set([b] + extra)) == 1 + len(extra) <= lt.SOURCES - 5, c.name
    assert c.need <= lt.BUDGET, c.name
  # the layers, as the registry tests name them
  lay = {n: c.layer for n, c in cases.items()}
  assert (3, 1, 64, True, lt.SWISH) in dw_shapes() and (5, 2, 288, True, lt.SWISH) in dw_shapes()
  assert (lay['dw_k3s1']['k'], lay['dw_k3s1']['s'], lay['dw_k3s1']['c']) == (3, 1, 64)
  assert (lay['dw_k5s2']['k'], lay['dw_k5s2']['s'], lay['dw_k5s2']['c']) == (5, 2, 288)
  a = _det_arch('efficientdet-d7x')
  assert a.image_hw == (1536, 1536) and lay['stem'] == dict(image=1536, cout=a.stem_filters)
  assert any(b.input_filters == 48 and b.mid_filters == 288 and b.kernel_size == 3 and b.stride == 1
             for b in a.blocks) and lay['mbconv']['cmid'] == 288
  assert any(b.mid_filters == b.output_filters == 32 and b.has_skip and b.se_filters for b in a.blocks)
  v = effnetv2_model.EffNetV2Arch('efficientnetv2-l')
  fused = {(b.input_filters, b.mid_filters if b.expand_ratio != 1 else b.output_filters,
            b.kernel_size, b.strides, b.has_skip) for b in v.blocks if b.conv_type == 1}
  assert (32, 32, 3, 1, True) in fused and (32, 128, 3, 2, False) in fused
  assert (384, (lt.SAME, lt.UP)) in fpn_shapes() and (384, (lt.SAME, lt.SAME, lt.DOWN)) in fpn_shapes()
  assert (384, (3, 3, 2, 2)) in pool_shapes() and (384, (3, 3, 2, 2), (48, 48)) in _pools(a)
  assert _det_arch('efficientdet-d2').fpn_filters == lay['sepconv']['f'] == 112
  assert _det_arch('efficientdet-lite0').fpn_filters == lay['sepconv_tma']['f'] == 64
  assert lay['pre_nms']['ld_cls'] == 816 and lay['pre_nms']['h'] == 192
  assert effnetv2_model.EffNetV2Arch('efficientnet-l2').head_filters == lay['gap']['c'] == 5504
  # the ragged pre-process packs more than 2^32 bytes
  for name in ('preprocess_ragged', 'cls_preprocess'):
    src = lay[name]['src']
    assert cases[name].batch * src[0] * src[1] * 3 > 1 << 32
