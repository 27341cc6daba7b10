"""Interp-Parts (interpretable and accurate fine-grained recognition via region grouping, Huang & Li, CVPR 2020) with the
reference's surface (model/methods/Interp_Parts.py).

Same module names as the reference's ``ResNet(Bottleneck, layers, num_classes, num_parts)`` — ``conv1, bn1, layer1..layer3,
grouping.{weight, smooth_factor}, post_block.*, attconv.{0,1,2,3}.*, groupingbn.*, mylinear.*`` — so reference checkpoints
load strictly, and the reference's initialisers (:300-313, :36-54).  ``forward(x)`` returns ``(logits, att [N, 1, K, 1],
assign [N, K, H, W])`` as the reference does (:333-371).

The trunk (ResNet v1.5 cut after layer3) runs on ops_resnet and hands its NHWC map to the grouping unit directly; the
grouping unit, the attention head with the part sum and the shaping loss's occupancy run on hk_ip_*; the Bottleneck1x1
stacks run on ops_resnet's block helpers over P = N*K rows; groupingbn on hk_bn_*; mylinear on hk_linear_*.
"""
import torch
import torch.nn as nn

from .. import ops, ops_interp_parts, ops_resnet
from ..backbone.resnet import BODY_KEYS, Bottleneck, ResNetBody
from ..registry import MODEL
from ..utils import load_pretrained


class Bottleneck1x1(nn.Module):
    """Interp_Parts.py:212-248: a bottleneck whose three convolutions are all 1x1 (parameter container)."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=1, stride=stride, padding=0, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * self.expansion, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride


class GroupingUnit(nn.Module):
    """Interp_Parts.py:25-128: centres ``weight`` [K, C, 1, 1] and ``smooth_factor`` [K]."""

    def __init__(self, in_channels, num_parts):
        super().__init__()
        self.num_parts, self.in_channels = num_parts, in_channels
        self.weight = nn.Parameter(torch.FloatTensor(num_parts, in_channels, 1, 1))
        self.smooth_factor = nn.Parameter(torch.FloatTensor(num_parts))

    def reset_parameters(self):
        """:36-54 without the clustering initialisation the reference never calls: kaiming normal clamped at 1e-5, and
        smooth_factor 0."""
        nn.init.kaiming_normal_(self.weight)
        self.weight.data.clamp_(min=1e-5)
        nn.init.constant_(self.smooth_factor, 0)

    def forward(self, x_nhwc):
        """NHWC map [N, H, W, C] -> (region features [N, K, C], assign [N, K, H, W])."""
        return ops_interp_parts.grouping(x_nhwc, self.weight, self.smooth_factor)

    def __repr__(self):
        return f'{self.__class__.__name__} ({self.in_channels} -> {self.num_parts})'


class ResNet(ResNetBody):
    """Interp_Parts.py:251-371 with ``block`` = Bottleneck, cut after layer3 (``layers[3]`` is not used)."""

    def __init__(self, layers, num_classes=1000, num_parts=32):
        ops_interp_parts.check_parts(num_parts)
        ops.check_num_classes(num_classes)
        super().__init__(layers[:3])
        self.n_parts, self.num_classes = num_parts, num_classes
        self.grouping = GroupingUnit(256 * Bottleneck.expansion, num_parts)
        self.grouping.reset_parameters()
        self.post_block = nn.Sequential(
            Bottleneck1x1(1024, 512, stride=1, downsample=nn.Sequential(nn.Conv2d(1024, 2048, kernel_size=1, stride=1, bias=False),
                                                                        nn.BatchNorm2d(2048))),
            Bottleneck1x1(2048, 512, stride=1),
            Bottleneck1x1(2048, 512, stride=1),
            Bottleneck1x1(2048, 512, stride=1),
        )
        self.attconv = nn.Sequential(
            Bottleneck1x1(1024, 256, stride=1),
            Bottleneck1x1(1024, 256, stride=1),
            nn.Conv2d(1024, 1, kernel_size=1, stride=1, padding=0, bias=True),
            nn.BatchNorm2d(1),
            nn.ReLU(),
        )
        self.groupingbn = nn.BatchNorm2d(2048)
        self.mylinear = nn.Linear(2048, num_classes)
        for m in self.modules():                                   # :300-313
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        for m in self.modules():
            if isinstance(m, (Bottleneck, Bottleneck1x1)):
                nn.init.constant_(m.bn3.weight, 0)
        self.__dict__['_trunk_plan'] = ops_resnet.TrunkPlan(self.trunk_modules())
        self.__dict__['_post_blocks'] = [ops_resnet.block_units(b) for b in self.post_block]
        self.__dict__['_att_blocks'] = [ops_resnet.block_units(b) for b in list(self.attconv)[:2]]

    def forward(self, x):
        N = x.shape[0]
        K = self.n_parts
        feat = ops_resnet.resnet_trunk(x, self._trunk_plan, self.training)          # NHWC [N, H, W, 1024]
        region, assign = self.grouping(feat)                                              # [N, K, C]: NHWC [N, K, 1, C]
        region = region.view(N, K, 1, region.shape[-1])
        a = ops_resnet.block_stack(region, self._att_blocks, self.training)
        p = ops_resnet.block_stack(region, self._post_blocks, self.training)
        conv, bn = self.attconv[2], self.attconv[3]
        pooled, att = ops_interp_parts.AttentionPoolFn.apply(a.view(N * K, -1), p.view(N * K, -1), conv.weight, conv.bias,
                                                             bn.weight, bn.bias, bn, self.training, N, K)
        out = ops_resnet.RowBatchNormFn.apply(pooled, self.groupingbn.weight, self.groupingbn.bias, self.groupingbn,
                                                    self.training)
        logits = ops.linear(out, self.mylinear.weight, self.mylinear.bias)
        return logits, att.view(N, 1, K, 1), assign

    def prediction(self, outputs):
        return outputs[0]


@MODEL.register
def IP_ResNet50(config):
    return load_pretrained(ResNet([3, 4, 6, 3], config.num_classes, config.num_parts), 'HAWKEYE_RESNET50_PTH', 'resnet50',
                           BODY_KEYS)


@MODEL.register
def IP_ResNet101(config):
    return load_pretrained(ResNet([3, 4, 23, 3], config.num_classes, config.num_parts), 'HAWKEYE_RESNET101_PTH', 'resnet101',
                           BODY_KEYS)
