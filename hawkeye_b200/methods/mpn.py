"""Fast MPN-COV (iSQRT-COV) with the reference's surface (model/methods/MPNCOV.py:23-102)."""
import torch
import torch.nn as nn

from .. import ops, ops_resnet
from ..backbone.resnet import resnet50
from ..registry import MODEL


class MPNCOV(nn.Module):
    def __init__(self, iter_num=3, is_sqrt=True, is_vec=True, input_dim=2048, dimension_reduction=None):
        super().__init__()
        self.iterNum, self.is_sqrt, self.is_vec, self.dr = iter_num, is_sqrt, is_vec, dimension_reduction
        if self.dr is not None:
            self.conv_dr_block = nn.Sequential(nn.Conv2d(input_dim, self.dr, kernel_size=1, stride=1, bias=False),
                                               nn.BatchNorm2d(self.dr), nn.ReLU(inplace=True))
            self.__dict__['_dr_unit'] = ops_resnet.Unit('1x1', self.conv_dr_block[0], self.conv_dr_block[1], True)
        out = self.dr if self.dr else input_dim
        self.output_dim = int(out * (out + 1) / 2) if is_vec else int(out * out)
        for m in self.modules():                                          # MPNCOV.py:76-82
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def forward(self, x):
        if self.dr is not None:
            x = ops.ToNCHWFn.apply(ops_resnet.unit(ops.ToNHWCFn.apply(x), self._dr_unit, self.training))
        x = ops.CovpoolLayer(x)
        if self.is_sqrt:
            x = ops.SqrtmLayer(x, self.iterNum)
        if self.is_vec:
            x = ops.TriuvecLayer(x)
        return x


@MODEL.register
class MPN(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.backbone = resnet50(pretrained=True)                          # MPNCOV.py:28-29
        self.pool = MPNCOV(config.iter_num, config.is_sqrt, config.is_vec, config.input_dim, config.dimension_reduction)
        ops.check_num_classes(config.num_classes)
        self.classifier = nn.Linear(self.pool.output_dim, config.num_classes)

    def forward(self, x):
        x = self.backbone(x)
        x = self.pool(x)
        x = x.view(x.size(0), -1)
        return ops.linear(x, self.classifier.weight, self.classifier.bias)
