"""CPU oracle of the EfficientNet V1 / V2 classification top (TEST INFRASTRUCTURE ONLY): the
pooling and the Dense classifier restated in torch on top of oracle/effnetv2_oracle.py's
backbone and head conv.

Restated from /root/reference/efficientnetv2/effnetv2_model.py:
  :472-496   Head.call: 'head_1x1' -> GlobalAveragePooling2D, or under local_pooling
             tf.nn.avg_pool with a window of the whole map, 'VALID' (the same mean, shape
             [N, 1, 1, C]) -> endpoint 'pooled_features' -> Dropout (the identity at inference)
             -> endpoint 'head'
  :571-578   _build: Dense(num_classes) when include_top and num_classes, else no `_fc`
  :487, :644-646   the Dense is applied to the squeezed [N, C] tensor
"""
from oracle import effnetv2_oracle


class EffNetV2TopOracle(effnetv2_oracle.EffNetV2Oracle):
  """call(images) -> the endpoints of EffNetV2Oracle plus 'pooled_features' and 'head' ([N, C], or
  [N, 1, 1, C] with local_pooling) and, when num_classes is non-zero, 'logits' [N, num_classes].
  They stay in the oracle's dtype: the device keeps them float32, so `store` does not apply."""

  def __call__(self, images):
    ep = super().__call__(images)
    s, mn = self.s, self.model_name
    pooled = ep['head_1x1'].mean((2, 3))
    ep['pooled_features'] = ep['head'] = (
        pooled.view(pooled.shape[0], 1, 1, -1) if s.local_pooling else pooled)
    if s.num_classes:
      ep['logits'] = pooled @ self.w[mn + '/dense/kernel'] + self.w[mn + '/dense/bias']
    return ep
