"""Channel Interaction Network head with the reference's surface (model/methods/CIN.py:9-108).

``ChannelInteractionModule`` keeps the reference's constructor, parameters (``conv``, ``fc``) and outputs — ``Z`` in eval
mode, ``(Z, Z_CCI)`` in training — but runs on the library's kernels: the channel Gram ``X X^T / WH`` (:31) and both
``W . X`` products (:34, :55) on the wgmma GEMM, ``softmax(-G)`` (:32) and ``|W_SCI - w W_SCI_BA|`` (:53) as fused row /
elementwise kernels, the 3x3 convolution (:36, :57) on the implicit-GEMM conv, ``fc`` (:47-48) on the skinny GEMM.
Any spatial size works: TMA needs a 16-byte row pitch, so the [B, C, WH] view is zero-padded to a multiple of 4 columns
(7x7 = 49 -> 52), which changes neither the Gram (divided by the true WH) nor the products.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops, ops_cin
from ..backbone.resnet import resnet50
from ..registry import MODEL
from ..utils import initialize_weights


class ChannelInteractionModule(nn.Module):
    def __init__(self, in_channel=2048, spatial_size=(7, 7)):
        super().__init__()
        self.in_channel = in_channel
        self.spatial_size = spatial_size
        WH = spatial_size[0] * spatial_size[1]
        self.conv = nn.Conv2d(in_channel, in_channel, 3, 1, 1)
        self.fc = nn.Linear(2 * in_channel * WH, 1)

    def _conv(self, yp, B, C, W, H, WH):
        y = yp[:, :, :WH] if yp.shape[-1] != WH else yp
        return ops_cin.Conv3x3NCHWFn.apply(y.reshape(B, C, W, H), self.conv.weight, self.conv.bias).view(B, C, WH)

    def _fc(self, v):
        # nn.Linear(., 1): the GEMM kernels want a 16-byte pitch on the [rows, out] side, so the single output row is padded
        # to four (three zero rows) and column 0 is kept
        w4 = F.pad(self.fc.weight, (0, 0, 0, 3))
        b4 = F.pad(self.fc.bias, (0, 3))
        return ops.linear(v, w4, b4)[:, :1]

    def forward(self, x):
        B, C, W, H = x.size()
        assert B % 2 == 0, 'batch size should not be odd!'                         # CIN.py:27
        WH = W * H
        xf = x.reshape(B, C, WH)
        pad = (-WH) % 4
        xp = F.pad(xf, (0, pad)) if pad else xf
        # SCI module (CIN.py:30-38)
        g = ops_cin.GramFn.apply(xp, 1.0 / WH)
        w_sci = ops_cin.SoftmaxNegFn.apply(g)
        y = self._conv(ops_cin.WXFn.apply(w_sci, xp), B, C, W, H, WH)
        z = ops_cin.AddFn.apply(y, xf)
        if not self.training:
            return z
        # CCI module (CIN.py:43-59)
        yv = y.reshape(B, -1)
        y_a = torch.cat((yv[:B // 2], yv[B // 2:]), dim=1)
        y_b = torch.cat((yv[B // 2:], yv[:B // 2]), dim=1)
        weight = torch.cat((self._fc(y_a), self._fc(y_b)), dim=0).reshape(-1)
        w_cci = ops_cin.CCIWeightFn.apply(w_sci, weight)
        y_cci = self._conv(ops_cin.WXFn.apply(w_cci, xp), B, C, W, H, WH)
        return z, ops_cin.AddFn.apply(y_cci, xf)


class CINClassifier(nn.Module):
    """CIN.py:64-82: spatial mean + Linear; in training passes Z_CCI through untouched."""

    def __init__(self, in_channel=2048, num_classes=200):
        super().__init__()
        ops.check_num_classes(num_classes)
        self.classifier = nn.Linear(in_channel, num_classes)

    def _logits(self, z):
        return ops.linear(ops.RowMeanFn.apply(z), self.classifier.weight, self.classifier.bias)

    def forward(self, x):
        if isinstance(x, tuple):
            z, z_cci = x
            return self._logits(z), z_cci
        return self._logits(x)


@MODEL.register
class CIN(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.num_classes = config.num_classes if 'num_classes' in config else 200
        # the reference hard-codes (7, 7) (224x224 inputs, CIN.py:98); other resolutions via config.spatial_size
        size = tuple(config.spatial_size) if 'spatial_size' in config else (7, 7)
        self.backbone = resnet50(pretrained=True)
        self.ChannelInteraction = ChannelInteractionModule(in_channel=2048, spatial_size=size)
        self.classifier = CINClassifier(in_channel=2048, num_classes=self.num_classes)
        self.ChannelInteraction.apply(initialize_weights)
        self.classifier.apply(initialize_weights)

    def forward(self, x):
        return self.classifier(self.ChannelInteraction(self.backbone(x)))
