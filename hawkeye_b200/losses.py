"""Losses of the callers of the hot path that are not plain cross-entropy.

``MAMCLoss`` / ``NPairsLoss`` follow model/loss/MAMC_loss.py:6-90 (the criterion of OSMENet, Examples/OSMENet.py:32): row
normalisation, the anchor-similarity matrix and its adjoint on the library's kernels (hk_l2norm_rows_*, the 3xTF32 GEMM),
and the three N-pairs terms of every anchor plus their gradient in ONE launch (hk_npair_loss) instead of the reference's
Python loop over anchors.

``peer_learning_loss`` follows model/loss/peer_learning_loss.py:5-65 (co-teaching between two networks, Sun et al.,
ICCV 2021): samples on which the two networks DISAGREE are always kept; of the samples on which they agree, each network is
updated on the ``(1 - drop_rate)`` fraction with the smallest loss *under the other network*.  It works on two [N, K] logit
tensors (N = batch size), so it stays in PyTorch: a few microseconds next to a ~25 ms step, and not part of the kernels' path.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function


def peer_learning_loss(logits_1, logits_2, labels, drop_rate):
    """-> (loss_1, loss_2), each the mean cross-entropy of its network over the samples it is updated on."""
    pred_1 = logits_1.argmax(dim=1)          # argmax of softmax == argmax of logits (peer_learning_loss.py:15-21)
    pred_2 = logits_2.argmax(dim=1)
    agree = pred_1 == pred_2
    idx_dis = (~agree).nonzero(as_tuple=True)[0]
    idx_agr = agree.nonzero(as_tuple=True)[0]
    sel_1, sel_2 = idx_dis, idx_dis          # sample indices network 1 / 2 is updated on
    if idx_agr.numel() > 0:
        with torch.no_grad():                # ranking only (the reference sorts `.data`, :36-40)
            l1 = F.cross_entropy(logits_1[idx_agr], labels[idx_agr], reduction='none')
            l2 = F.cross_entropy(logits_2[idx_agr], labels[idx_agr], reduction='none')
        keep = int((1 - drop_rate) * idx_agr.numel())                    # :42
        small_1 = idx_agr[torch.argsort(l1)[:keep]]                      # low-loss samples according to network 1
        small_2 = idx_agr[torch.argsort(l2)[:keep]]
        sel_1 = torch.cat((idx_dis, small_2))                            # network 1 learns from network 2's selection (:48-51)
        sel_2 = torch.cat((idx_dis, small_1))
    return F.cross_entropy(logits_1[sel_1], labels[sel_1]), F.cross_entropy(logits_2[sel_2], labels[sel_2])


class NPairsLossFn(Function):
    """features [b, p, D], labels [b]  ->  scalar N-pairs loss (MAMC_loss.py:35-90)."""

    @staticmethod
    def forward(ctx, feats, labels):
        from . import _lib
        from .ops import _check_cuda, _f32c, gemm
        _check_cuda(feats, labels)
        b, p, D = feats.shape
        n = b * p
        if n % 4 or D % 4:
            raise _lib.HawkeyeLibError(f'NPairsLoss: batch x attentions = {n} and the feature size {D} must be multiples of 4 '
                                       '(16-byte TMA row pitch of the anchor-similarity GEMMs)')
        x = _f32c(feats).reshape(n, D)
        s = _lib.stream_ptr()
        dev = x.device
        xn, inv = torch.empty_like(x), torch.empty(n, device=dev, dtype=torch.float32)
        _lib.call('hk_l2norm_rows_fwd', x, xn, inv, n, D, s)                                        # :43
        prod = torch.empty(n, n, device=dev, dtype=torch.float32)
        gemm(xn, 0, D, 0, xn, 0, D, 0, prod, n, 0, n, n, D, exact=True)                              # :46 prod = F F^T
        cls = labels.to(torch.int32).repeat_interleave(p).contiguous()                              # :44
        part = torch.arange(p, device=dev, dtype=torch.int32).repeat(b).contiguous()                # :45
        acc = torch.zeros(1, device=dev, dtype=torch.float64)
        dprod = torch.empty_like(prod)
        _lib.call('hk_npair_loss', prod, cls, part, acc, dprod, n, s)                               # :57-90
        ctx.save_for_backward(xn, inv, dprod)
        ctx.shape = (b, p, D)
        return acc[0].float()

    @staticmethod
    def backward(ctx, g):
        from . import _lib
        from .ops import gemm
        xn, inv, dprod = ctx.saved_tensors
        b, p, D = ctx.shape
        n = b * p
        s = _lib.stream_ptr()
        # dF = (dprod + dprod^T) F : two products into the same buffer (the second accumulates through D / beta)
        t = torch.empty_like(xn)
        gemm(dprod, 0, n, 0, xn, 1, D, 0, t, D, 0, n, D, n, exact=True)
        dxn = torch.empty_like(xn)
        gemm(dprod, 1, n, 0, xn, 1, D, 0, dxn, D, 0, n, D, n, D=t, ldd=D, beta=1.0, exact=True)
        dx = torch.empty_like(xn)
        _lib.call('hk_l2norm_rows_bwd', xn, inv, dxn, dx, n, D, s)
        return (dx * g).reshape(b, p, D), None


class NPairsLoss(nn.Module):
    def forward(self, inputs, targets):
        return NPairsLossFn.apply(inputs, targets)


class MAMCLoss(nn.Module):
    """CrossEntropy(label_smoothing=0.1) on the logits + lambda_a x N-pairs loss on the per-attention features
    (MAMC_loss.py:6-21); ``inputs`` is the ``(pred, x_part)`` pair OSMENet returns."""

    def __init__(self, config):
        super().__init__()
        from . import ops
        self.lambda_a = config.lambda_a if 'lambda_a' in config else 0.5
        self.use_mamc = config.use_mamc if 'use_mamc' in config else True
        self.ce_loss = ops.CrossEntropyLS(0.1)
        self.npair_loss = NPairsLoss()

    def forward(self, inputs, targets):
        pred, x_part = inputs
        loss_ce = self.ce_loss(pred, targets)
        self.last_correct = self.ce_loss.last_correct
        if not self.use_mamc:
            return loss_ce
        return loss_ce + self.lambda_a * self.npair_loss(x_part, targets)


class APINetLoss(nn.Module):
    """model/loss/APINet_loss.py: CrossEntropy(label_smoothing=0.1) over cat(self_logits, other_logits) with targets
    cat(labels1, labels2, labels1, labels2), plus MarginRankingLoss(margin=0.05) between the softmax scores of the target under
    the self and the other features.  ``inputs`` is the 4-tuple APINet returns; ``target`` is unused, as in the reference.
    One cross-entropy kernel over the 8n rows and one ranking kernel (hk_apinet_rank_loss) that adds its term and gradient;
    ``last_correct`` is the top-1 count over the 8n rows, on the device."""

    def __init__(self, config=None):
        super().__init__()
        from .ops_apinet import RANK_MARGIN
        self.margin = RANK_MARGIN

    def forward(self, inputs, target=None):
        from .ops_apinet import APINetLossFn
        self_logits, other_logits, labels1, labels2 = inputs
        base = self_logits._base
        if (base is not None and base is other_logits._base and base.is_contiguous() and base.dim() == 2
                and self_logits.data_ptr() == base.data_ptr() and self_logits.shape[0] * 2 == base.shape[0]
                and other_logits.data_ptr() == base.data_ptr() + self_logits.numel() * base.element_size()):
            logits = base                    # APINet's two halves of one [8n, K] fc output: no copy
        else:
            logits = torch.cat([self_logits, other_logits], dim=0)
        targets = torch.cat([labels1, labels2, labels1, labels2], dim=0)
        loss, correct = APINetLossFn.apply(logits, targets, self.margin)
        self.last_correct = correct
        return loss


def dcl_stacked_logits(logits, swap_logits):
    """-> one [R, ld] tensor with ``logits`` in columns [0, K) and ``swap_logits`` in [K, K + K2).  When the two are DCL's
    own column views of one contiguous [R, Kp] classifier output — all its rows, its strides, adjacent columns — that output
    is returned as it is; anything else (a row slice of it, say) is concatenated into a new tensor."""
    base = logits._base
    R, K = logits.shape
    if (base is not None and base is swap_logits._base and base.dim() == 2 and base.is_contiguous()
            and base.shape[0] == R == swap_logits.shape[0] and base.shape[1] >= K + swap_logits.shape[1]
            and logits.stride() == base.stride() and swap_logits.stride() == base.stride()
            and logits.data_ptr() == base.data_ptr()
            and swap_logits.data_ptr() == base.data_ptr() + K * base.element_size()):
        return base
    return torch.cat([logits, swap_logits], dim=1)


class DCLLoss(nn.Module):
    """model/loss/DCL_loss.py: alpha CE(logits, labels) + beta CE(swap_logits, labels_swap) + gamma L1(mask, swap_law), both
    cross-entropies with label smoothing 0.1.  ``outputs`` is the list DCL returns; its two logit tensors are read in place
    when they are the column views of one stacked classifier output, as DCL makes them.  One hk_dcl_loss launch;
    ``last_correct`` is the top-1 count on the device (over the summed logits under cls_2xmul, Examples/DCL.py:104-107)."""

    def __init__(self, config):
        super().__init__()
        self.alpha, self.beta, self.gamma = config.alpha, config.beta, config.gamma

    def forward(self, outputs, labels, labels_swap, swap_law):
        from .ops_dcl import DCLLossFn
        logits, swap_logits, mask = outputs
        K, K2 = logits.shape[1], swap_logits.shape[1]
        loss, correct = DCLLossFn.apply(dcl_stacked_logits(logits, swap_logits), K, K2, labels, labels_swap, mask, swap_law,
                                        self.alpha, self.beta, self.gamma, K2 == 2 * K)
        self.last_correct = correct
        return loss
