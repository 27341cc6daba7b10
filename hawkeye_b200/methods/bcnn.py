"""BCNN with the reference's constructor / attribute / state_dict surface (model/methods/BCNN.py:30-55)."""
import torch.nn as nn

from .. import ops
from ..backbone.vgg import vgg16
from ..registry import MODEL
from ..utils import initialize_weights


class BilinearPooling(nn.Module):
    """Fused Gram + sqrt(.+1e-5) + L2-normalise (BCNN.py:8-27) on the wgmma kernel."""

    def forward(self, x):
        return ops.bilinear_pool(x)


@MODEL.register
class BCNN(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.stage = config.stage if 'stage' in config else 2          # BCNN.py:36
        self.backbone = vgg16(pretrained=True)                           # BCNN.py:38-39 (all 31 feature layers)
        self.bilinear_pooling = BilinearPooling()
        ops.check_num_classes(config.num_classes)
        self.classifier = nn.Linear(self.backbone.out_channels ** 2, config.num_classes)
        self.classifier.apply(initialize_weights)
        if self.stage == 1:                                              # BCNN.py:45-47
            for p in self.backbone.parameters():
                p.requires_grad = False

    def features(self, x):
        x = self.backbone(x)
        return x.detach() if self.stage == 1 else x                      # BCNN.py:51-52

    def head(self, feat):
        return ops.linear(self.bilinear_pooling(feat), self.classifier.weight, self.classifier.bias)

    def forward(self, x):
        return self.head(self.features(x))
