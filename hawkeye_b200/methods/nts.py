"""NTS-Net (navigator-teacher-scrutinizer, Yang et al., ECCV 2018) with the reference's surface
(model/methods/NTS_Net/NTSNet.py, resnet.py, anchors.py).

Same attributes as the reference — ``pretrained_model`` (a full ResNet-50: conv1, bn1, layer1..4, avgpool, ``fc`` =
Linear(2048, 200)), ``proposal_net`` (down1..3, tidy1..3), ``concat_net`` = Linear(2048 (K + 1), 200), ``partcls_net`` =
Linear(2048, 200) — so the reference's 336-entry ``state_dict`` loads strictly.  The 200 classes are hard-coded, as in the
reference.  ``forward(x)`` returns ``[raw_logits, concat_logits, part_logits [B, T, 200], top_n_index int64 [B, T],
top_n_prob [B, T]]``.

The trunk runs on ops_resnet twice per call, on the B images and on the B*T part crops (detached input), so BatchNorm uses
the statistics of each pass and updates its running statistics twice per training step.  The proposal net runs on
hk_conv3x3_* and hk_nts_score_*, the NMS, the gather and the crops on hk_nts_nms / hk_nts_crop: no host round trip.

Reference quirk kept on purpose: resnet.py:148 applies ``nn.Dropout(p=0.5)(x)`` to the pooled feature through a module
built on every call, which is always in train mode, so dropout applies in eval mode too, and fc, concat_net and
partcls_net all see the dropped-out features.  ``pretrained_model.drop`` (an ``nn.Dropout``, no state) holds the
probability; set ``pretrained_model.drop.p = 0`` for deterministic evaluation.  The masks are a hash of a device seed drawn
per forward, so a captured CUDA graph draws new masks on every replay.

The anchors (``edge_anchors``, a non-persistent int32 buffer) are computed on the host once.  Any ``image_size`` that is a
multiple of 32 works; part crops are always 224 x 224.  ``proposal_num`` may not exceed the number of boxes every greedy NMS
pass is sure to keep (8 at 224, 26 at 448), computed from the anchors at construction, so the NMS always fills its T rows.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from .. import ops, ops_nts, ops_resnet
from ..backbone.resnet import BODY_KEYS, ResNetBody
from ..ops import nchw_to_nhwc
from ..registry import MODEL
from ..utils import load_pretrained

NUM_CLASSES = 200
# (stride, size, scales, aspect ratios) of the three anchor levels (anchors.py:3-7)
ANCHOR_LEVELS = ((32, 48, (2 ** (1 / 3), 2 ** (2 / 3)), (0.667, 1, 1.5)),
                 (64, 96, (2 ** (1 / 3), 2 ** (2 / 3)), (0.667, 1, 1.5)),
                 (128, 192, (1, 2 ** (1 / 3), 2 ** (2 / 3)), (0.667, 1, 1.5)))


def edge_anchors(image_size):
    """int32 [A, 4] (y0, x0, y1, x1) in the image zero-padded by 224: the reference's default anchor maps (level, then
    scale, then aspect ratio, then row-major position), with its float32 arithmetic, shifted by 224 and truncated."""
    f32 = np.float32
    out = []
    for stride, size, scales, ratios in ANCHOR_LEVELS:
        n = int(np.ceil(f32(image_size) / f32(stride)))
        centre = f32(stride / 2.0) + f32(stride) * np.arange(n, dtype=np.float64)   # float64 positions, stored in float32
        cy, cx = np.meshgrid(centre.astype(f32), centre.astype(f32), indexing='ij')
        for s in scales:
            for r in ratios:
                h, w = f32(size * s / float(r) ** 0.5), f32(size * s * float(r) ** 0.5)
                box = np.stack([cy - h / f32(2), cx - w / f32(2), cy + h / f32(2), cx + w / f32(2)], -1).astype(f32)
                out.append(box.reshape(-1, 4))
    return (np.concatenate(out) + f32(ops_nts.PAD)).astype(np.int64).astype(np.int32)


def survivor_bound(anchors):
    """The fewest boxes any greedy pass of hard_nms keeps: a pick removes at most its closed IoU >= 0.25 neighbourhood, so at
    least ceil(A / largest neighbourhood) boxes survive, whatever the scores."""
    a = anchors.astype(np.int64)
    dy = np.minimum(a[:, None, 2], a[None, :, 2]) - np.maximum(a[:, None, 0], a[None, :, 0])
    dx = np.minimum(a[:, None, 3], a[None, :, 3]) - np.maximum(a[:, None, 1], a[None, :, 1])
    inter = np.where((dy < 0) | (dx < 0), 0, dy * dx)
    area = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    covered = 4 * inter >= area[:, None] + area[None, :] - inter
    return math.ceil(len(a) / int(covered.sum(1).max()))


class ResNet(ResNetBody):
    """NTS_Net/resnet.py:94-152 with Bottleneck: forward(x, seed, call) -> (logits, layer4 map NCHW, dropped pooled feature)."""

    def __init__(self, num_classes=NUM_CLASSES):
        super().__init__((3, 4, 6, 3))
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(2048, num_classes)
        self.drop = nn.Dropout(p=0.5)
        for m in self.modules():                                  # resnet.py:110-116
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, 0, math.sqrt(2.0 / (m.kernel_size[0] * m.kernel_size[1] * m.out_channels)))
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        self.__dict__['_plan'] = ops_resnet.TrunkPlan(self.trunk_modules())

    def forward(self, x, seed, call):
        params = self._plan.params()
        fmap = ops_resnet.ResNetTrunkFn.apply(x, self._plan, ops.wants_grad(x, params), self.training, False, *params)
        n, C, H, W = fmap.shape
        feature = ops_nts.dropout(ops.RowMeanFn.apply(fmap.reshape(n, C, H * W)), float(self.drop.p), seed, call)
        return ops.linear(feature, self.fc.weight, self.fc.bias), fmap, feature


class ProposalNet(nn.Module):
    """NTSNet.py:63-82 (parameter container): forward(x NHWC, anchors, T) -> (rpn_score, top_n_prob, top_n_index, boxes)."""

    def __init__(self):
        super().__init__()
        self.down1 = nn.Conv2d(2048, 128, 3, 1, 1)
        self.down2 = nn.Conv2d(128, 128, 3, 2, 1)
        self.down3 = nn.Conv2d(128, 128, 3, 2, 1)
        self.ReLU = nn.ReLU()
        self.tidy1 = nn.Conv2d(128, 6, 1, 1, 0)
        self.tidy2 = nn.Conv2d(128, 6, 1, 1, 0)
        self.tidy3 = nn.Conv2d(128, 9, 1, 1, 0)

    def forward(self, x_nhwc, anchors, topn):
        return ops_nts.proposal(x_nhwc, self, anchors, topn)


@MODEL.register
class NTSNet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.topN = int(config.proposal_num)
        self.proposal_num = self.topN
        self.CAT_NUM = int(config.cat_num)
        self.image_size = int(config.image_size)
        if self.image_size <= 0 or self.image_size % 32:
            raise ValueError(f'NTSNet: image_size={self.image_size} must be a positive multiple of 32')
        if not 0 <= self.CAT_NUM <= self.topN:
            raise ValueError(f'NTSNet: cat_num={self.CAT_NUM} must lie in [0, proposal_num={self.topN}]')
        anchors = edge_anchors(self.image_size)
        if len(anchors) > 2048:
            raise ValueError(f'NTSNet: image_size={self.image_size} gives {len(anchors)} anchors, the NMS takes at most 2048')
        bound = survivor_bound(anchors)
        if not 1 <= self.topN <= bound:
            raise ValueError(f'NTSNet: proposal_num={self.topN} must lie in [1, {bound}]: at image_size {self.image_size} '
                             f'a greedy NMS pass may keep as few as {bound} boxes')
        self.pretrained_model = ResNet(NUM_CLASSES)
        self.proposal_net = ProposalNet()
        self.concat_net = nn.Linear(2048 * (self.CAT_NUM + 1), NUM_CLASSES)
        self.partcls_net = nn.Linear(2048, NUM_CLASSES)
        self.pad_side = ops_nts.PAD
        self.register_buffer('edge_anchors', torch.from_numpy(anchors), persistent=False)
        # torchvision's ResNet-50 without its 1000-way fc: the reference replaces fc after loading (NTSNet.py:19-21)
        load_pretrained(self.pretrained_model, 'HAWKEYE_RESNET50_PTH', 'resnet50', BODY_KEYS)

    def forward(self, x):
        B, T, K = x.shape[0], self.topN, self.CAT_NUM
        seed = torch.randint(0, 2 ** 62, (1,), device=x.device, dtype=torch.int64) if self.pretrained_model.drop.p > 0 else None
        raw_logits, rpn_feature, feature = self.pretrained_model(x, seed, ops_nts.DROP_IMAGES)
        _, prob, idx, boxes = self.proposal_net(nchw_to_nhwc(rpn_feature.detach()), self.edge_anchors, T)
        part_imgs = ops_nts.crop(x, boxes)
        _, _, part_features = self.pretrained_model(part_imgs, seed, ops_nts.DROP_PARTS)
        part_feature = part_features.view(B, T, -1)[:, :K].reshape(B, -1)
        concat_logits = ops.linear(torch.cat([part_feature, feature], dim=1), self.concat_net.weight, self.concat_net.bias)
        part_logits = ops.linear(part_features, self.partcls_net.weight, self.partcls_net.bias).view(B, T, -1)
        return [raw_logits, concat_logits, part_logits, idx, prob]
