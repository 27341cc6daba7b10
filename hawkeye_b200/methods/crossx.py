"""CrossX (reference model/methods/CrossX.py, ``MODEL`` entry ``CrossX``): a ResNet-50 whose last blocks of layer3 and
layer4 carry a multi-excitation layer (``me``, P gates of one BatchNorm output), with the layer4 parts fused into the
layer3 parts (``conv2_p`` 1x1 2048 -> 1024, nearest 2x upsample, ``conv3_p`` 3x3 and ``bn3_p``), and three classifiers
over the pooled parts: ``fc_ulti`` (mean of the layer4 parts), ``fc_plty`` (max of the layer3 parts) and ``fc_cmbn``
(mean of the fused maps).

The modules and their registration order are the reference's, so its state_dict loads strictly in both directions and the
initialisers draw in its RNG order; the ``me`` Linears are created as soon as their layer is built.  ``forward`` runs the
trunk on the ResNet units, the excitation blocks and the fusion on the hk_crossx_* kernels (ops_crossx), and the
classifiers on the linear GEMMs; the pooled features are [N, P, C], so each classifier reads them without a copy.
"""
import math

import torch
import torch.nn as nn

from .. import ops, ops_crossx, ops_resnet
from .._lib import HawkeyeLibError
from ..backbone.resnet import BODY_KEYS, ResNetBody
from ..registry import MODEL
from ..utils import load_pretrained


class MELayer(nn.Module):
    """P gates ``Linear(C, C / reduction) -> ReLU -> Linear(C / reduction, C) -> Sigmoid`` of one squeeze
    (CrossX.py:48-72); ``avg_pool`` is parameter-free and kept for attribute parity."""

    def __init__(self, channel, reduction=16, nparts=1):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.nparts = nparts
        self.parts = nn.Sequential(*[nn.Sequential(nn.Linear(channel, channel // reduction), nn.ReLU(inplace=True),
                                                   nn.Linear(channel // reduction, channel), nn.Sigmoid())
                                     for _ in range(nparts)])


class CrossXNet(ResNetBody):
    """ResNet(Bottleneck, [3, 4, 6, 3], nparts, meflag=nparts > 1, num_classes) of CrossX.py:126-263."""

    def __init__(self, num_classes=200, nparts=2):
        if nparts not in (1, 2, 3):
            raise HawkeyeLibError(f'CrossX: num_parts={nparts}; the reference builds 1, 2 or 3 parts')
        ops.check_num_classes(num_classes)
        self.__dict__['_me'] = nparts > 1

        def add_me(i, layer):
            if self._me and i in (2, 3):
                layer[-1].me = MELayer(layer[-1].conv3.out_channels, reduction=256, nparts=nparts)

        super().__init__((3, 4, 6, 3), on_layer=add_me)
        self.nparts, self.num_classes = nparts, num_classes
        self.adpavgpool = nn.AdaptiveAvgPool2d(1)
        self.fc_ulti = nn.Linear(2048 * nparts, num_classes)
        if nparts > 1:
            self.adpmaxpool = nn.AdaptiveMaxPool2d(1)
            self.fc_plty = nn.Linear(1024 * nparts, num_classes)
            self.fc_cmbn = nn.Linear(1024 * nparts, num_classes)
            names = [f'conv2_{i}' for i in (1, 2)] + [f'conv3_{i}' for i in (1, 2)] + [f'bn3_{i}' for i in (1, 2)]
            names += ['conv2_3', 'conv3_3', 'bn3_3'] if nparts == 3 else []
            for n in names:
                kind = n[:5]
                self.add_module(n, nn.Conv2d(2048, 1024, 1, bias=False) if kind == 'conv2' else
                                nn.Conv2d(1024, 1024, 3, padding=1, bias=False) if kind == 'conv3' else nn.BatchNorm2d(1024))
        for m in self.modules():                                    # CrossX.py:164-170
            if isinstance(m, nn.Conv2d):
                m.weight.data.normal_(0, math.sqrt(2. / (m.kernel_size[0] * m.kernel_size[1] * m.out_channels)))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        if not self._me:
            self.__dict__['_plan'] = ops_resnet.TrunkPlan(self.trunk_modules())
            return
        # layer1, layer2 and layer3 up to its excitation block; layer4 up to its own; the two excitation blocks
        self.__dict__['_plan'] = ops_resnet.TrunkPlan([self.conv1, self.bn1, self.relu, self.maxpool, self.layer1,
                                                       self.layer2, self.layer3[:-1]])
        self.__dict__['_l4'] = [ops_resnet.block_units(b) for b in self.layer4[:-1]]
        self.__dict__['_me_units'] = [self._excite_units(self.layer3[-1]), self._excite_units(self.layer4[-1])]
        self.__dict__['_fuse_units'] = [ops_resnet.Unit('3x3', getattr(self, f'conv3_{i + 1}'),
                                                        getattr(self, f'bn3_{i + 1}'), False) for i in range(nparts)]

    @staticmethod
    def _excite_units(blk):
        u1, u2, _, _ = ops_resnet.block_units(blk)
        return u1, u2, ops_resnet.Unit('1x1', blk.conv3, blk.bn3, False)

    def forward(self, x):
        if not self._me:
            feat = ops_resnet.resnet_trunk(x, self._plan, self.training)
            return ops.linear(ops.NHWCMeanFn.apply(feat), self.fc_ulti.weight, self.fc_ulti.bias)
        N, H, W = x.shape[0], x.shape[2], x.shape[3]
        h3, w3 = (H + 15) // 16, (W + 15) // 16
        if (h3, w3) != (28, 28):
            raise HawkeyeLibError(f'CrossX: a {H}x{W} input gives a {h3}x{w3} layer3 map; the fusion upsamples layer4 to '
                                  '28x28 (CrossX.py:212), which needs 433..448 pixels a side')
        return self.head(ops_resnet.resnet_trunk(x, self._plan, self.training))

    def head(self, x3):
        """Everything after the trunk blocks: layer3's last block, layer4, the fusion and the classifiers, on the NHWC
        output of layer3.4 [N, 28, 28, 1024] -> the 6-tuple of ``forward``."""
        if tuple(x3.shape[1:]) != (28, 28, 1024):
            raise HawkeyeLibError(f'CrossX.head: layer3 map {tuple(x3.shape)}, expected [N, 28, 28, 1024]')
        N, P, t = x3.shape[0], self.nparts, self.training
        out3, parts3 = ops_crossx.excite(x3, self._me_units[0], list(self.layer3[-1].me.parts), True, t)
        x4 = ops_resnet.block_stack(out3, self._l4, t)
        parts4 = ops_crossx.excite(x4, self._me_units[1], list(self.layer4[-1].me.parts), False, t)
        conv2 = [getattr(self, f'conv2_{i + 1}').weight for i in range(P)]
        ulti, *Rs = ops_crossx.UltiFn.apply(parts4, *conv2)                                # [N, P, 2048]
        plty, *Ss = ops_crossx.FuseFn.apply(parts3, *Rs)                                   # [N, P, 1024]
        cmbn = torch.stack([ops.NHWCMeanFn.apply(ops_resnet.unit(S, u, t)) for S, u in zip(Ss, self._fuse_units)],
                           1)                                                              # [N, P, 1024]
        xf = ops.linear(ulti.view(N, -1), self.fc_ulti.weight, self.fc_ulti.bias)
        xp = ops.linear(plty.view(N, -1), self.fc_plty.weight, self.fc_plty.bias)
        xc = ops.linear(cmbn.view(N, -1), self.fc_cmbn.weight, self.fc_cmbn.bias)
        views = [[f[:, i, :, None, None] for i in range(P)] for f in (ulti, plty, cmbn)]
        return (xf, xp, xc) + tuple(views)

    def prediction(self, outputs):
        """The logits that accuracy and validation score: xf + xp + xc (Examples/CrossX.py:52-56, 67-69)."""
        return outputs[0] + outputs[1] + outputs[2] if isinstance(outputs, tuple) else outputs


@MODEL.register
def CrossX(config):
    """CrossX.py:266-272: num_parts from the config (1 = a plain ResNet-50 with ``fc_ulti``), 200 classes by default,
    pretrained unless ``pretrained: false``.  torchvision's trunk comes from $HAWKEYE_RESNET50_PTH; its ``fc`` never loads
    (the reference's ``strict=False`` load skips it), and the ``me`` gates keep their initial values."""
    net = CrossXNet(config.num_classes if 'num_classes' in config else 200, config.num_parts)
    if not (config.pretrained if 'pretrained' in config else True):
        return net
    return load_pretrained(net, 'HAWKEYE_RESNET50_PTH', 'resnet50', BODY_KEYS, own=('.me.',))
