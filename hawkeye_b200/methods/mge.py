"""MGE-CNN (granularity-specific experts, Zhang et al., ICCV 2019) with the reference's surface
(model/methods/MGE_CNN/MGE.py, grad_cam.py).

Same module names as the reference's LocalCamNet — ``conv4`` / ``conv5`` (a ResNet-50 cut after layer3: conv1, bn1, relu,
maxpool, layer1..3 at indices 0-6, and layer4's blocks), their copies ``_box``, ``_box_2`` and ``_gate``, ``classifier*``
(``Classifier`` wrapping ``.fc``), ``conv6*``, ``cls_part*``, ``cls_cat*``, the unused ``cls_cat_a`` and ``cls_gate`` — so
the reference's 1302-entry ``state_dict`` loads strictly.  ``forward(x, y=None, is_vis=False, vis_idx=None, gt_top=None)``
returns ``{'logits': [logits, logits_max, logits_cat, logits_box, logits_max_1, logits_cat_1, logits_box_2, logits_max_2,
logits_cat_2, logits_gate], 'pr_gate': [N, 3], 'boxes': int32 [2, N, 4]}``; ``boxes`` holds the two stages' crop boxes as
(y0, x0, y1, x1), end exclusive, which the reference computes and discards.

Each trunk runs on ops_resnet in NHWC and updates its BatchNorm statistics once per training step.  The two Grad-CAMs are
computed in closed form (ops_mge.cam_box): the hooked tensor is layer4's output, which the reference pools and feeds to the
main classifier for both CAMs (grad_cam.py:46), so the layer weights are relu(W_main[idx]) / HW and no backward runs in the
forward.  Only the target index needs a forward.  With ``y`` it is ``y``.  Without it the reference takes the argmax of the
main classifier over an eval-mode layer4 pass on the detached layer3 map (conv5 on conv4 for the first CAM, conv5_box on
conv4_box for the second), which reads the running statistics this step's train-mode pass has just updated and updates
none; in train mode that pass is rerun here under no_grad, and in eval mode it equals the forward already done, so the
first index is argmax(logits) and the second the main classifier on the pooled conv5_box.  GradCam's ``model.zero_grad()``
and the gradients of its backward are not reproduced: the reference's Example clears them with ``optimizer.zero_grad()``
before the loss's backward.
"""
import copy

import torch
import torch.nn as nn

from .. import ops, ops_mge, ops_resnet
from ..backbone.resnet import ResNetTrunk, resnet50
from ..registry import MODEL

BRANCHES = ('', '_box', '_box_2', '_gate')


class Classifier(nn.Module):
    """MGE.py:18-27 (parameter container)."""

    def __init__(self, in_panel, out_panel, bias=False):
        super().__init__()
        self.fc = nn.Linear(in_panel, out_panel, bias=bias)

    def forward(self, x):
        return ops.linear(x, self.fc.weight, self.fc.bias)


class LocalCamNet(nn.Module):
    """MGE.py:75-240.  ``layers`` sets the trunk's blocks per stage (tests use a shallow trunk); a ResNet-50 loads
    $HAWKEYE_RESNET50_PTH into all four trunks, as the reference's deep copies of one pretrained ResNet-50 do."""

    def __init__(self, config=None, layers=None):
        super().__init__()
        self.config = config
        self.num_classes = int(config.num_classes)
        self.box_thred = float(config.box_thred)
        self.image_size = int(config.image_size)
        ops.check_num_classes(self.num_classes)
        if self.image_size <= 0 or self.image_size % 32:
            raise ValueError(f'MGE_CNN: image_size={self.image_size} must be a positive multiple of 32')
        K = self.num_classes
        trunk = resnet50(pretrained=True) if layers is None else ResNetTrunk(tuple(layers))
        kids = list(trunk.children())
        self.conv4 = nn.Sequential(*kids[:7])
        self.conv5 = nn.Sequential(*list(kids[7]))
        self.pool = nn.AdaptiveAvgPool2d(1)
        self.classifier = Classifier(2048, K, bias=True)
        self.conv4_box = copy.deepcopy(self.conv4)
        self.conv5_box = copy.deepcopy(self.conv5)
        self.classifier_box = Classifier(2048, K, bias=True)
        self.conv4_box_2 = copy.deepcopy(self.conv4)
        self.conv5_box_2 = copy.deepcopy(self.conv5)
        self.classifier_box_2 = Classifier(2048, K, bias=True)
        self.conv6_1 = nn.Conv2d(1024, 10 * K, 1, 1, 1)
        self.conv6_2 = nn.Conv2d(1024, 10 * K, 1, 1, 1)
        self.conv6 = nn.Conv2d(1024, 10 * K, 1, 1, 1)
        self.cls_part_1 = Classifier(10 * K, K, bias=True)
        self.cls_part_2 = Classifier(10 * K, K, bias=True)
        self.cls_part = Classifier(10 * K, K, bias=True)
        self.cls_cat_1 = Classifier(2048 + 10 * K, K, bias=True)
        self.cls_cat_2 = Classifier(2048 + 10 * K, K, bias=True)
        self.cls_cat = Classifier(2048 + 10 * K, K, bias=True)
        self.pool_max = nn.AdaptiveMaxPool2d(1)
        self.cls_cat_a = Classifier(3 * (2048 + 10 * K), K, bias=True)     # never used by forward (MGE.py:119)
        self.conv4_gate = copy.deepcopy(self.conv4)
        self.conv5_gate = copy.deepcopy(self.conv5)
        self.cls_gate = nn.Sequential(Classifier(2048, 512, bias=True), Classifier(512, 3, bias=True))
        self.__dict__['_plans'] = {b: (ops_resnet.TrunkPlan(getattr(self, 'conv4' + b)),
                                       [ops_resnet.block_units(blk) for blk in getattr(self, 'conv5' + b)]) for b in BRANCHES}

    def trunk(self, x, branch):
        """conv4 and conv5 of ``branch`` on an NCHW image -> (NHWC layer3 map, NHWC layer4 map, pooled [N, 2048])."""
        plan, blocks = self._plans[branch]
        c4 = ops_resnet.resnet_trunk_nhwc(x, plan, self.training)
        c5 = ops_resnet.block_stack(c4, blocks, self.training)
        return c4, c5, ops.NHWCMeanFn.apply(c5)

    def experts(self, c4, pool, suffix):
        """The part head and the two classifiers after it -> (logits_max, logits_cat)."""
        conv6, cls_part, cls_cat = (getattr(self, n + suffix) for n in ('conv6', 'cls_part', 'cls_cat'))
        pooled, _ = ops_mge.part(c4, conv6)
        return cls_part(pooled), cls_cat(ops_mge.cat_l2n(pool, pooled))

    def cam_target(self, c4, pool, branch, logits, y):
        """-> (logits, targets) of one Grad-CAM's index: y when given; else the main classifier over layer4 in eval mode."""
        if y is not None:
            return None, y
        if branch == '' and not self.training:
            return logits, None
        with torch.no_grad():
            if self.training:                              # layer4 rerun on the running statistics, updating none
                pool = ops.NHWCMeanFn.apply(ops_resnet.block_stack(c4.detach(), self._plans[branch][1], False))
            return self.classifier(pool), None

    def forward(self, x, y=None, is_vis=False, vis_idx=None, gt_top=None):
        n, _, h, w = x.shape
        if h != self.image_size or w != self.image_size:
            raise ValueError(f'MGE_CNN: input {h}x{w}, the model is built for image_size {self.image_size}')
        S, W_main = self.image_size, self.classifier.fc.weight
        t1 = gt_top if is_vis and vis_idx == 1 else y
        t2 = gt_top if is_vis and vis_idx == 2 else y

        c4, c5, pool = self.trunk(x, '')
        logits = self.classifier(pool)
        logits_max, logits_cat = self.experts(c4, pool, '')
        z, t = self.cam_target(c4, pool, '', logits, t1)
        boxes = ops_mge.cam_box(c5, W_main, S, self.box_thred, logits=z, targets=t)
        input_box = ops_mge.crop(x, boxes, S)

        c4b, c5b, pool_b = self.trunk(input_box, '_box')
        logits_box = self.classifier_box(pool_b)
        logits_max_1, logits_cat_1 = self.experts(c4b, pool_b, '_1')
        z, t = self.cam_target(c4b, pool_b, '_box', None, t2)
        boxes_2 = ops_mge.cam_box(c5b, W_main, S, self.box_thred, logits=z, targets=t)
        input_box_2 = ops_mge.crop(input_box, boxes_2, S)

        c4b2, _, pool_b2 = self.trunk(input_box_2, '_box_2')
        logits_box_2 = self.classifier_box_2(pool_b2)
        logits_max_2, logits_cat_2 = self.experts(c4b2, pool_b2, '_2')

        _, _, pool_gate = self.trunk(x, '_gate')
        g1 = self.cls_gate[1].fc
        logits_gate, pr_gate = ops_mge.GateFn.apply(self.cls_gate[0](pool_gate), g1.weight, g1.bias, logits_cat, logits_cat_1,
                                                    logits_cat_2)
        logits_list = [logits, logits_max, logits_cat, logits_box, logits_max_1, logits_cat_1, logits_box_2, logits_max_2,
                       logits_cat_2, logits_gate]
        return {'logits': logits_list, 'pr_gate': pr_gate, 'boxes': torch.stack([boxes, boxes_2])}

    def get_params(self, prefix='extractor'):
        """MGE.py:225-240: the four trunks (conv5 before conv4 in each pair), or every other parameter."""
        extractor = [p for b in BRANCHES for m in ('conv5', 'conv4') for p in getattr(self, m + b).parameters()]
        if prefix in ['extractor', 'extract']:
            return extractor
        elif prefix in ['classifier']:
            ids = set(map(id, extractor))
            return filter(lambda p: id(p) not in ids, self.parameters())


@MODEL.register
def MGE_CNN(config):
    return LocalCamNet(config)
