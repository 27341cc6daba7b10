"""DCL (destruction and construction learning, Chen et al., CVPR 2019) with the reference's surface (model/methods/DCL.py).

Same constructor, attributes (``backbone`` = the ResNet-50 trunk, ``Convmask``, ``avgpool2``, ``avgpool``, ``classifier``,
``classifier_swap``) and ``state_dict``, so reference checkpoints load strictly.  ``forward`` returns the list
``[logits, swap_logits, mask]``.  The pool, Convmask, AvgPool2d(2) and tanh run as one head node (hk_dcl_head_*), and both
bias-free classifiers as one GEMM over a stacked weight; the two logit tensors are column views of that GEMM's output, which
``losses.DCLLoss`` reads without a copy.  At 448x448 the trunk map is 14x14 and the mask has 49 entries, one per cell of
the default 7x7 jigsaw.
"""
import torch.nn as nn

from .. import _lib, ops, ops_dcl
from ..backbone.resnet import resnet50
from ..registry import MODEL


@MODEL.register
class DCL(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.num_classes = config.num_classes
        self.cls_2 = config.cls_2
        self.cls_2xmul = config.cls_2xmul
        if not (self.cls_2 or self.cls_2xmul):
            raise _lib.HawkeyeLibError('DCL: set model.cls_2 (2-way swap classifier) or model.cls_2xmul (2 x num_classes); '
                                       'with neither there is no classifier_swap')
        ops.check_num_classes(self.num_classes)
        self.backbone = resnet50(pretrained=True)                # children()[:-2] of the reference ResNet, same keys
        self.Convmask = nn.Conv2d(2048, 1, 1, stride=1, padding=0, bias=True)
        self.avgpool2 = nn.AvgPool2d(2, stride=2)                # parameter-free; fused into the head kernel
        self.avgpool = nn.AdaptiveAvgPool2d(output_size=1)       # likewise
        self.classifier = nn.Linear(2048, self.num_classes, bias=False)
        # cls_2xmul wins when both are set, as in DCL.py:25-28
        self.classifier_swap = nn.Linear(2048, 2 * self.num_classes if self.cls_2xmul else 2, bias=False)

    def forward(self, x):
        x = self.backbone(x)
        pooled, mask = ops_dcl.DCLHeadFn.apply(x, self.Convmask.weight, self.Convmask.bias)
        logits = ops_dcl.StackedClassifierFn.apply(pooled, self.classifier.weight, self.classifier_swap.weight)
        K, K2 = self.classifier.weight.shape[0], self.classifier_swap.weight.shape[0]
        return [logits[:, :K], logits[:, K:K + K2], mask]

    def prediction(self, outputs):
        """The logits, plus both halves of the swap logits under cls_2xmul (Examples/DCL.py's validation)."""
        logits = outputs[0]
        if self.cls_2xmul:
            K = logits.shape[1]
            logits = logits + outputs[1][:, :K] + outputs[1][:, K:2 * K]
        return logits
