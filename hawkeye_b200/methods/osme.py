"""OSMENet with the reference's surface (model/methods/OSME.py:8-64).

``OSME_block`` = squeeze (spatial mean) -> Linear -> ReLU -> Linear -> sigmoid -> channel-wise re-scaling of the feature map;
``OSME`` = P such blocks, each followed by a Linear over the flattened gated map; ``OSMENet`` = ResNet-101 trunk + OSME +
classifier, returning ``(logits, per-attention features)`` for the MAMC loss (model/loss/MAMC_loss.py, not part of this package).
All arithmetic runs on the library's kernels (hk_row_mean, hk_linear, hk_relu, hk_se_gate); the reference hard-codes a 7x7 feature
map (OSME.py:57) — here ``config.feature_shape`` may override it (14 for 448x448 inputs).
"""
import torch
import torch.nn as nn

from .. import ops, ops_cin
from ..backbone.resnet import resnet101
from ..registry import MODEL


class OSME_block(nn.Module):
    def __init__(self, channels, ratio):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)          # parameter-free; kept for attribute parity
        self.block = nn.Sequential(nn.Linear(channels, channels // ratio), nn.ReLU(inplace=True),
                                   nn.Linear(channels // ratio, channels), nn.Sigmoid())

    def forward(self, x):
        N, C, H, W = x.size()
        z = ops.RowMeanFn.apply(x.reshape(N, C, H * W))                                  # OSME.py:21
        h = ops.ReluFn.apply(ops.linear(z, self.block[0].weight, self.block[0].bias))
        m = ops.linear(h, self.block[2].weight, self.block[2].bias)                      # pre-sigmoid excitation
        return ops_cin.SEGateFn.apply(x, m)                                              # sigmoid(m) * x, OSME.py:22-23


class OSME(nn.Module):
    def __init__(self, in_channels, out_channels=1024, feature_shape=(7, 7), num_attention=2):
        super().__init__()
        reduce_ratio = 16
        fc_in = in_channels * feature_shape[0] * feature_shape[1] if isinstance(feature_shape, tuple) \
            else in_channels * feature_shape * feature_shape
        self.blocks = nn.ModuleList([OSME_block(in_channels, reduce_ratio) for _ in range(num_attention)])
        self.fcs = nn.ModuleList([nn.Linear(fc_in, out_channels) for _ in range(num_attention)])

    def forward(self, x):
        N = x.size(0)
        s = [block(x) for block in self.blocks]
        features = [ops.linear(s[i].reshape(N, -1), fc.weight, fc.bias) for i, fc in enumerate(self.fcs)]
        return sum(features), torch.stack(features, dim=1)                               # OSME.py:44


@MODEL.register
class OSMENet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.num_attention = config.num_attention
        self.num_classes = config.num_classes
        ops.check_num_classes(self.num_classes)
        shape = config.feature_shape if 'feature_shape' in config else 7
        self.backbone = resnet101(pretrained=True)
        self.osme = OSME(2048, 1024, feature_shape=shape, num_attention=self.num_attention)
        self.classifier = nn.Linear(1024, self.num_classes)

    def forward(self, x):
        x = self.backbone(x)
        x1, x_part = self.osme(x)
        return ops.linear(x1, self.classifier.weight, self.classifier.bias), x_part
