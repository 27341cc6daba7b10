"""VGG-16 'D' feature extractor with the reference's parameter surface (model/backbone/vgg.py:56-70,76,141-151).

``features`` is an ``nn.Sequential`` of real ``nn.Conv2d / nn.ReLU / nn.MaxPool2d`` modules, so
``state_dict()`` keys (``{0,2,5,...,28}.{weight,bias}``) and shapes are identical to the reference and
reference checkpoints load unchanged — but ``forward`` never calls those modules: the whole stack runs as
one fused CUDA pipeline (NHWC, wgmma implicit-GEMM convs) through ``ops.vgg_features``.
"""
import torch
import torch.nn as nn

from .. import ops
from ..registry import BACKBONE
from ..utils import initialize_weights

cfgs = {
    'D': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M'],
}


class VGGFeatures(nn.Sequential):
    """The 31-layer ``features`` stack BCNN/CBCNN slice out of vgg16 (BCNN.py:38-39)."""

    def __init__(self, cfg=None):
        cfg = list(cfg if cfg is not None else cfgs['D'])
        layers, cin = [], 3
        for v in cfg:
            if v == 'M':
                layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
            else:
                layers += [nn.Conv2d(cin, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
                cin = v
        super().__init__(*layers)
        self.cfg = tuple(cfg)
        self.out_channels = cin
        self.train_backbone = True
        self.apply(initialize_weights)   # vgg.py:45-46

    def conv_params(self):
        ps = []
        for m in self:
            if isinstance(m, nn.Conv2d):
                ps += [m.weight, m.bias]
        return ps

    def forward(self, x):
        return ops.vgg_features(x, self.cfg, self.conv_params(), self.train_backbone)


@BACKBONE.register
def vgg16(pretrained=False, progress=True, **kwargs):
    """Reference signature (vgg.py:141-151).  ``pretrained=True`` needs the torchvision checkpoint on disk
    (``$HAWKEYE_VGG16_PTH``); there is no network here, so otherwise the reference initialisers are used."""
    import os
    feats = VGGFeatures(cfgs['D'])
    path = os.environ.get('HAWKEYE_VGG16_PTH')
    if pretrained and path and os.path.exists(path):
        sd = torch.load(path, map_location='cpu')
        feats.load_state_dict({k[len('features.'):]: v for k, v in sd.items() if k.startswith('features.')})
    elif pretrained and os.environ.get('HAWKEYE_ALLOW_RANDOM_INIT', '0') != '1':
        # the reference downloads ImageNet weights here (vgg.py:83-85); silently training on a random VGG would be wrong
        import logging
        logging.getLogger('hawkeye_b200').warning(
            'vgg16(pretrained=True): no checkpoint at $HAWKEYE_VGG16_PTH (%r) — the backbone keeps the reference\'s RANDOM '
            'initialisation.  Point HAWKEYE_VGG16_PTH at torchvision\'s vgg16 .pth, or set HAWKEYE_ALLOW_RANDOM_INIT=1 '
            '(benchmarks / parity tests) to silence this.', path)
    return feats
