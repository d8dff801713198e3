"""EfficientNet V1/V2 classifier backbones on the H100 path (reference: efficientnetv2/)."""
