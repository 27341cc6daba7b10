"""APINet (attentive pairwise interaction, Zhuang et al., AAAI 2020) with the reference's surface (model/methods/APINet.py).

Same constructor, attributes (``backbone`` = ResNet-101 trunk, ``avg``, ``map1``, ``map2``, ``fc``, ``drop``, ``sigmoid``) and
``state_dict``, so reference checkpoints load unchanged.  ``forward(images, targets, flag='train')`` returns
``(self_logits, other_logits, labels1, labels2)`` like the reference; ``flag='val'`` or ``targets=None`` returns
``fc(pool)``, so ``model(images)`` evaluates it.  The pair mining runs on the device (the reference copies the distance
matrix to the host every step), so a training step never synchronises and can be captured in a CUDA graph.

Under torchrun each rank mines pairs within its own balanced batch — what the reference's ``nn.DataParallel`` does too, since
each replica runs ``get_pairs`` on its own shard.  Like the reference, the head expects 224x224 inputs (a 7x7 trunk map).
"""
import torch
import torch.nn as nn

from .. import _lib, ops, ops_apinet, ops_cin
from ..backbone.resnet import resnet101
from ..registry import MODEL


@MODEL.register
class APINet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.num_classes = config.num_classes
        ops.check_num_classes(self.num_classes)
        self.backbone = resnet101(pretrained=True)
        self.avg = nn.AvgPool2d(kernel_size=7, stride=1)         # parameter-free; the mean runs on hk_row_mean
        self.map1 = nn.Linear(2048 * 2, 512)
        self.map2 = nn.Linear(512, 2048)
        self.fc = nn.Linear(2048, self.num_classes)              # the reference hard-codes 200 in its logit buffers (:63-64)
        self.drop = nn.Dropout(p=0.5)
        self.sigmoid = nn.Sigmoid()                              # fused into the gate kernel
        self.device = None

    def pool(self, images):
        conv_out = self.backbone(images)
        n, C, H, W = conv_out.shape
        if (H, W) != (7, 7):
            raise _lib.HawkeyeLibError(f'APINet: the trunk map is {H}x{W}, expected 7x7 (224x224 inputs; the reference '
                                       'pools with AvgPool2d(7, stride=1))')
        return ops_cin.RowMeanFn.apply(conv_out.reshape(n, C, H * W))

    def forward(self, images, targets=None, flag='train'):
        self.device = images.device
        pool_out = self.pool(images)
        if flag != 'train' or targets is None:
            return ops.linear(pool_out, self.fc.weight, self.fc.bias)
        n = pool_out.shape[0]
        if n < 2:
            raise _lib.HawkeyeLibError(f'APINet: a training batch of {n} image(s) has no pairs (need at least 2)')
        idx2, labels1, labels2 = ops_apinet.mine_pairs(pool_out.detach(), targets)
        p = float(self.drop.p) if self.training else 0.0
        seed = torch.randint(0, 2 ** 62, (1,), device=pool_out.device, dtype=torch.int64) if p > 0 else None
        feats = ops_apinet.pair_head(pool_out, idx2, self.map1, self.map2, p, seed)
        logits = ops.linear(feats, self.fc.weight, self.fc.bias)             # [8n, K] = cat(self_logits, other_logits)
        return logits[:4 * n], logits[4 * n:], labels1, labels2
