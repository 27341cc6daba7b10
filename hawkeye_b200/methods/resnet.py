"""The plain ResNet classifiers of the reference's registry (model/backbone/resnet.py, ``MODEL`` entries ``ResNet50`` and
``ResNet101``), trained by Examples/Baseline.py and Examples/PairConfusion.py.

Same modules as torchvision's ``resnet50`` / ``resnet101`` — ``conv1, bn1, layer1..layer4, avgpool, fc`` — so the state_dict
has torchvision's keys (320 / 626 entries) and the reference's checkpoints load strictly, in both directions; the
reference's initialisers, in its RNG order.  ``forward`` runs the trunk on ops_resnet, takes the spatial mean of its NHWC
map (ops.NHWCMeanFn) and applies ``fc`` on the linear GEMMs: no layout change on the way.
"""
import torch.nn as nn

from .. import ops, ops_resnet
from ..backbone.resnet import BODY_KEYS, ResNetBody
from ..registry import MODEL
from ..utils import load_pretrained


class ResNet(ResNetBody):
    """ResNet(Bottleneck, layers, num_classes) of model/backbone/resnet.py with zero_init_residual off."""

    def __init__(self, layers, num_classes=1000):
        ops.check_num_classes(num_classes)
        super().__init__(layers)
        self.num_classes = num_classes
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(2048, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        self.__dict__['_plan'] = ops_resnet.TrunkPlan(self.trunk_modules())

    def forward(self, x):
        feat = ops_resnet.resnet_trunk(x, self._plan, self.training)            # NHWC [N, H/32, W/32, 2048]
        return ops.linear(ops.NHWCMeanFn.apply(feat), self.fc.weight, self.fc.bias)


def _build(config, layers, env, arch):
    """The reference loads torchvision's checkpoint through its shape-filtered load_state_dict, so ``fc`` loads at 1000
    classes and keeps its initial values otherwise.  Here the trunk goes through load_pretrained's strict check (a missing
    or mis-shaped trunk tensor raises) and ``fc`` is mapped only when its shape is torchvision's."""
    net = ResNet(layers, config.num_classes)
    if not (config.pretrained if 'pretrained' in config else True):
        return net
    names = dict(BODY_KEYS, fc='fc') if net.num_classes == 1000 else BODY_KEYS
    return load_pretrained(net, env, arch, names)


@MODEL.register
def ResNet50(config):
    return _build(config, (3, 4, 6, 3), 'HAWKEYE_RESNET50_PTH', 'resnet50')


@MODEL.register
def ResNet101(config):
    return _build(config, (3, 4, 23, 3), 'HAWKEYE_RESNET101_PTH', 'resnet101')
