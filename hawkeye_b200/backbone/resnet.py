"""ResNet-50 v1.5 trunk with the reference's module / state_dict surface (model/backbone/resnet.py:89-252,296-306).

The modules below are parameter containers (same attribute names => same state_dict keys as the reference's
``nn.Sequential(*list(resnet50().children())[:-2])``, MPNCOV.py:28-29); ``forward`` runs the fused CUDA pipeline.
"""
import torch.nn as nn

from .. import ops_resnet
from ..registry import BACKBONE
from ..utils import load_pretrained

RESNET_NAMES = ('conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4')


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)   # v1.5: stride on 3x3
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride


def _make_layer(inplanes, planes, blocks, stride):
    downsample = None
    if stride != 1 or inplanes != planes * 4:
        downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, kernel_size=1, stride=stride, bias=False),
                                   nn.BatchNorm2d(planes * 4))
    layers = [Bottleneck(inplanes, planes, stride, downsample)]
    layers += [Bottleneck(planes * 4, planes) for _ in range(1, blocks)]
    return nn.Sequential(*layers)


def _resnet_modules(layers):
    """conv1, bn1, relu, maxpool and one stage of ``layers[i]`` blocks per entry, created in torchvision's order."""
    mods = [nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True),
            nn.MaxPool2d(kernel_size=3, stride=2, padding=1)]
    inplanes = 64
    for planes, n, stride in zip((64, 128, 256, 512), layers, (1, 2, 2, 2)):
        mods.append(_make_layer(inplanes, planes, n, stride))
        inplanes = planes * 4
    return mods


class ResNetBody(nn.Module):
    """conv1, bn1, relu, maxpool, layer1..layer{len(layers)} under torchvision's attribute names: the base of the methods'
    ResNets, which register their own modules after these."""

    def __init__(self, layers):
        super().__init__()
        for name, m in zip(RESNET_NAMES, _resnet_modules(layers)):
            self.add_module(name, m)
        self.num_layers = len(layers)

    def trunk_modules(self, cut=None):
        """[conv1, bn1, relu, maxpool, layer1..layer{cut}] (every layer without ``cut``), as ops_resnet.TrunkPlan takes it."""
        return [getattr(self, n) for n in RESNET_NAMES[:4 + (cut or self.num_layers)]]


class ResNetTrunk(nn.Sequential):
    """children()[:-2] of the reference ResNet: conv1, bn1, relu, maxpool, layer1..layer4 (indices 0..7)."""

    def __init__(self, layers=(3, 4, 6, 3)):
        mods = _resnet_modules(layers)
        super().__init__(*mods)
        self.out_channels = mods[-1][-1].conv3.out_channels
        for m in self.modules():                                   # resnet.py:191-196
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        self.__dict__['_plan'] = ops_resnet.TrunkPlan(self)

    def forward(self, x):
        return ops_resnet.resnet_trunk(x, self)


TRUNK_KEYS = {n: str(i) for i, n in enumerate(RESNET_NAMES)}      # torchvision's top-level name -> ResNetTrunk index
BODY_KEYS = {n: n for n in RESNET_NAMES}                           # -> ResNetBody attribute (layers past the body: skipped)


@BACKBONE.register
def resnet101(pretrained=False, progress=True, **kwargs):
    """Reference signature (resnet.py:309-319); the trunk of OSMENet (OSME.py:55-56).  Offline => reference initialisers
    unless $HAWKEYE_RESNET101_PTH points at torchvision's checkpoint."""
    trunk = ResNetTrunk((3, 4, 23, 3))
    return load_pretrained(trunk, 'HAWKEYE_RESNET101_PTH', 'resnet101', TRUNK_KEYS) if pretrained else trunk


@BACKBONE.register
def resnet50(pretrained=False, progress=True, **kwargs):
    """Reference signature (resnet.py:296-306); offline => reference initialisers unless $HAWKEYE_RESNET50_PTH is set."""
    trunk = ResNetTrunk((3, 4, 6, 3))
    return load_pretrained(trunk, 'HAWKEYE_RESNET50_PTH', 'resnet50', TRUNK_KEYS) if pretrained else trunk
