"""AP-CNN (attention pyramid convolutional neural network, Ding et al., TIP 2021) with the reference's surface
(model/methods/APCNN.py).

Same module names as the reference's ``ResNet(num_classes, Bottleneck, [3, 4, 6, 3])`` — ``conv1, bn1, layer1..4`` at the top
level, ``fpn.P5_1.{conv_master,conv_gpb}.{conv,bn}``, ``fpn.P{5,4,3}_2``, ``fpn.P{4,3}_1``, ``apn.A{3,4,5}_1.conv`` (a
ConvTranspose2d), ``apn.A{3,4,5}_2.conv{1,2}``, ``cls5, cls4, cls3, cls_concate`` with the reference's Sequential indices —
so reference checkpoints load strictly, and the reference's initialisation loop (:418-424, nn.Conv2d and nn.BatchNorm2d only).
``forward(inputs, targets=None)`` returns ``(out_mean, out_list, mask_cat, roi_list)``.

The trunk runs on ops_resnet in NHWC: stem, layer1 and layer2 once; layer3, layer4, the pyramid, the attention and the heads
twice with the same weights, on the layer2 map and on its ROI-guided refinement, so every BatchNorm from layer3 on updates its
running statistics twice per training step, as in the reference.  The heads read the attended maps only through their
spatial mean, and mean_hw((s + ch) F) = mean_hw(s F) + ch mean_hw(F), so hk_apcnn_att_* produce the two pooled vectors and
A3..A5 are never written.  The ROI selection and the refinement run on hk_apcnn_roi / hk_apcnn_refine_* with the per-image
counts kept on the device: no host round trip in a step.

``roi_list`` departs from the reference's three variable-length tensors of (image, x1, y1, x2, y2, score) rows, which cannot
be built without reading the counts back: it is ``[(boxes [N, topk, 4], count [N])] * 3`` with (x1, y1, x2, y2) rows and
zeros past ``count``; ``ops_apcnn.roi_to_reference`` converts (on the host).  Equal gate values go to the highest flat index (what a stable
ascending sort gives; torch's argsort leaves it undefined).  The drop block of the refinement is drawn on the device
(torch.rand under the CUDA generator, so a replayed CUDA graph draws afresh) where the reference uses Python's ``random``;
``forward(..., draws=)`` takes the draws explicitly: [N, 2] in [0, 1), column 0 the branch (< 0.3 a level-3 ROI, < 0.6 a
level-4 ROI), column 1 the index as a fraction of the image's count.
"""
import math

import torch
import torch.nn as nn

from .. import ops, ops_apcnn, ops_resnet
from ..backbone.resnet import BODY_KEYS, ResNetBody
from ..ops_resnet import RowBatchNormFn
from ..registry import MODEL
from ..utils import load_pretrained


class BasicConv(nn.Module):
    """APCNN.py:73-90 as used by SimpleFPA: 1x1 conv without bias, BatchNorm2d(momentum 0.01), ReLU (parameter container)."""

    def __init__(self, in_planes, out_planes):
        super().__init__()
        self.out_channels = out_planes
        self.conv = nn.Conv2d(in_planes, out_planes, kernel_size=1, stride=1, padding=0, bias=False)
        self.bn = nn.BatchNorm2d(out_planes, eps=1e-5, momentum=0.01, affine=True)
        self.relu = nn.ReLU(inplace=True)
        self.__dict__['_unit'] = ops_resnet.Unit('1x1', self.conv, self.bn, True)

    def forward(self, x_nhwc):
        return ops_resnet.unit(x_nhwc, self._unit, self.training)


class SimpleFPA(nn.Module):
    """:170-199: master 1x1 branch plus a global-pooling branch broadcast over the map."""

    def __init__(self, in_planes, out_planes):
        super().__init__()
        self.channels_cond = in_planes
        self.conv_master = BasicConv(in_planes, out_planes)
        self.conv_gpb = BasicConv(in_planes, out_planes)

    def forward(self, x):
        N, _, _, C = x.shape
        gpb = self.conv_gpb(ops.NHWCMeanFn.apply(x).view(N, 1, 1, C))
        return ops_apcnn.BcastAddFn.apply(self.conv_master(x), gpb.view(N, -1))


class PyramidFeatures(nn.Module):
    """:202-233, NHWC in and out."""

    def __init__(self, B3_size, B4_size, B5_size, feature_size=256):
        super().__init__()
        self.P5_1 = SimpleFPA(B5_size, feature_size)
        self.P5_2 = nn.Conv2d(feature_size, feature_size, kernel_size=3, stride=1, padding=1)
        self.P4_1 = nn.Conv2d(B4_size, feature_size, kernel_size=1, stride=1, padding=0)
        self.P4_2 = nn.Conv2d(feature_size, feature_size, kernel_size=3, stride=1, padding=1)
        self.P3_1 = nn.Conv2d(B3_size, feature_size, kernel_size=1, stride=1, padding=0)
        self.P3_2 = nn.Conv2d(feature_size, feature_size, kernel_size=3, stride=1, padding=1)

    def forward(self, inputs):
        B3, B4, B5 = inputs
        c1, c3 = ops.Conv1x1Fn.apply, ops.Conv3x3Fn.apply
        P5 = self.P5_1(B5)
        P4 = ops_apcnn.LateralFn.apply(P5, c1(B4, self.P4_1.weight, self.P4_1.bias))
        P3 = ops_apcnn.LateralFn.apply(P4, c1(B3, self.P3_1.weight, self.P3_1.bias))
        return [c3(P3, self.P3_2.weight, self.P3_2.bias), c3(P4, self.P4_2.weight, self.P4_2.bias),
                c3(P5, self.P5_2.weight, self.P5_2.bias)]


class SpatialGate(nn.Module):
    def __init__(self, out_channels):
        super().__init__()
        self.conv = nn.ConvTranspose2d(out_channels, 1, kernel_size=3, stride=1, padding=1)


class ChannelGate(nn.Module):
    def __init__(self, out_channels):
        super().__init__()
        self.conv1 = nn.Conv2d(out_channels, out_channels // 16, kernel_size=1, stride=1, padding=0)
        self.conv2 = nn.Conv2d(out_channels // 16, out_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, pooled):
        """mean_hw F [N, C] -> conv2's output before the sigmoid (:291-294)."""
        w1, w2 = self.conv1.weight, self.conv2.weight
        h = ops.ActFn.apply(ops.linear(pooled, w1.view(w1.shape[0], -1), self.conv1.bias), False)
        return ops.linear(h, w2.view(w2.shape[0], -1), self.conv2.bias)


class PyramidAttentions(nn.Module):
    """:236-268 -> (the three gates [N, H_l, W_l], mean_hw F_l as [3, N, C], mean_hw A_l as [3, N, C])."""

    def __init__(self, channel_size=256):
        super().__init__()
        self.A3_1, self.A3_2 = SpatialGate(channel_size), ChannelGate(channel_size)
        self.A4_1, self.A4_2 = SpatialGate(channel_size), ChannelGate(channel_size)
        self.A5_1, self.A5_2 = SpatialGate(channel_size), ChannelGate(channel_size)

    def forward(self, inputs):
        gates, pm, psf, z = [], [], [], []
        for F, sg, cg in zip(inputs, (self.A3_1, self.A4_1, self.A5_1), (self.A3_2, self.A4_2, self.A5_2)):
            g, m, sf = ops_apcnn.AttentionFn.apply(F, sg.conv.weight, sg.conv.bias)
            gates.append(g)
            pm.append(m)
            psf.append(sf)
            z.append(cg(m))
        pm = torch.stack(pm)
        return gates, pm, ops_apcnn.MixFn.apply(torch.stack(z), pm, torch.stack(psf))


class Flatten(nn.Module):
    def forward(self, x):
        return x.view(x.size(0), -1)


def _head(in_features, hidden, num_classes, pool):
    mods = ([nn.AdaptiveAvgPool2d(1)] if pool else []) + [Flatten(), nn.BatchNorm1d(in_features), nn.Linear(in_features, hidden),
                                                          nn.BatchNorm1d(hidden), nn.ELU(inplace=True),
                                                          nn.Linear(hidden, num_classes)]
    return nn.Sequential(*mods)


def _run_head(seq, v, training):
    """BatchNorm1d -> Linear -> BatchNorm1d -> ELU -> Linear on pooled rows [N, F] (:377-414); the pooling and Flatten entries
    of the Sequential hold no state and have already happened."""
    bn1, fc1, bn2, _, fc2 = list(seq)[-5:]
    v = RowBatchNormFn.apply(v, bn1.weight, bn1.bias, bn1, training)
    v = RowBatchNormFn.apply(ops.linear(v, fc1.weight, fc1.bias), bn2.weight, bn2.bias, bn2, training)
    return ops.linear(ops.ActFn.apply(v, True), fc2.weight, fc2.bias)


class ResNet(ResNetBody):
    """APCNN.py:344-599 with ``block`` = Bottleneck."""

    def __init__(self, num_classes, layers=(3, 4, 6, 3)):
        ops.check_num_classes(num_classes)
        super().__init__(layers)
        self.num_classes = num_classes
        hidden = 512 if num_classes == 200 else 256
        self.fpn = PyramidFeatures(512, 1024, 2048)
        self.apn = PyramidAttentions(channel_size=256)
        self.cls5 = _head(256, hidden, num_classes, True)
        self.cls4 = _head(256, hidden, num_classes, True)
        self.cls3 = _head(256, hidden, num_classes, True)
        self.cls_concate = _head(256 * 3, hidden, num_classes, False)
        for m in self.modules():                                   # :418-424
            if isinstance(m, nn.Conv2d):
                m.weight.data.normal_(0, math.sqrt(2. / (m.kernel_size[0] * m.kernel_size[1] * m.out_channels)))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        self.__dict__['_plan'] = ops_resnet.TrunkPlan(self.trunk_modules(2))
        self.__dict__['_blocks3'] = [ops_resnet.block_units(b) for b in self.layer3]
        self.__dict__['_blocks4'] = [ops_resnet.block_units(b) for b in self.layer4]
        self.register_buffer('nms_keep', torch.from_numpy(ops_apcnn.suppression_table()), persistent=False)

    def check_input(self, h, w):
        if h % 32 or w % 32 or h <= 0 or w <= 0:
            raise ValueError(f'APCNN: input {h}x{w}: both sides must be positive multiples of 32')
        win = ops_apcnn.central_windows(h // 8, w // 8, self.num_classes)
        if (win[:, 0] >= win[:, 1]).any() or (win[:, 2] >= win[:, 3]).any():
            raise ValueError(f'APCNN: input {h}x{w} is too small: the central window of a pyramid level is empty')
        return win

    def stage(self, x2):
        """layer3, layer4, pyramid, attention and the four heads on an NHWC layer2 map -> (logits [out3, out4, out5,
        out_concate], gates)."""
        x3 = ops_resnet.block_stack(x2, self._blocks3, self.training)
        x4 = ops_resnet.block_stack(x3, self._blocks4, self.training)
        gates, pm, v = self.apn(self.fpn([x2, x3, x4]))
        N = x2.shape[0]
        out_concate = _run_head(self.cls_concate, pm.permute(1, 0, 2).reshape(N, -1), self.training)
        outs = [_run_head(h, v[i], self.training) for i, h in enumerate((self.cls3, self.cls4, self.cls5))]
        return outs + [out_concate], gates

    def forward(self, inputs, targets=None, draws=None):
        n, _, img_h, img_w = inputs.shape
        win = self.check_input(img_h, img_w)
        if self.training and n < 2:
            raise ValueError('APCNN: the heads\' BatchNorm1d needs more than one image in train mode')
        x2 = ops_resnet.resnet_trunk(inputs, self._plan, self.training)
        outs1, gates = self.stage(x2)
        boxes, counts = ops_apcnn.roi_select(gates, torch.from_numpy(win), self.nms_keep, img_h, img_w)
        if self.training and draws is None:
            draws = torch.rand(n, 2, device=inputs.device, dtype=torch.float32)
        x2_crop = ops_apcnn.RefineFn.apply(x2, boxes, counts, draws if self.training else None)
        outs2, _ = self.stage(x2_crop)
        out_list = outs1 + outs2
        out_mean = torch.stack(out_list).mean(0)
        roi_list = [(boxes[:, o:o + k], counts[:, l]) for l, (o, k) in enumerate(zip(ops_apcnn.ROI_OFFSETS, ops_apcnn.TOPK))]
        return out_mean, out_list, ops_apcnn.mask_cat(gates), roi_list

    def prediction(self, outputs):
        return outputs[0]


def resnet50(num_classes):
    return ResNet(num_classes, (3, 4, 6, 3))


@MODEL.register
def APCNN(config):
    """torchvision's ResNet-50 at $HAWKEYE_RESNET50_PTH goes into conv1..layer4; the reference's load skips its fc, which the
    model does not have."""
    return load_pretrained(resnet50(int(config.num_classes)), 'HAWKEYE_RESNET50_PTH', 'resnet50', BODY_KEYS)
