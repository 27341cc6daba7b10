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


class ProtoTreeLoss(nn.Module):
    """Examples/ProtoTreeNet.py:109: F.nll_loss(torch.log(pred), labels) on the (pred, info) pair ProtoTreeNet returns, in one
    hk_prototree_nll launch.  ``last_correct`` is the top-1 count on the device; ``last`` keeps (pred, pa, labels) of the call
    for the derivative-free leaf update that follows the optimizer step (under CUDA-graph replay these are the graph's static
    tensors, refreshed by every replay)."""

    def forward(self, outputs, labels):
        from .ops_prototree import NLLFn
        pred, info = outputs
        loss, correct = NLLFn.apply(pred, labels)
        self.last_correct = correct
        self.last = (pred.detach(), info['pa_tensor'].dense, labels)
        return loss


class NTSLoss(nn.Module):
    """model/loss/NTS_loss.py: CE(raw_logits) + CE(concat_logits) + CE over the B*T part rows (each with label smoothing 0.1
    and its own mean) + ranking_loss(top_n_prob, list_loss(part_logits)) on the list NTSNet returns.  The cross-entropies
    run on hk_softmax_ce_ls, the list and ranking losses in one hk_nts_rank_loss launch with no per-row read-back (the
    reference reads every label to the host in list_loss).  ``last_correct`` is the top-1 count on concat_logits, the
    accuracy Examples/NTSNet.py reports.

    Under torchrun each rank runs on its own B_local images: with equal shards, the per-rank means and the ranking sum over
    B_local, averaged by the gradient all-reduce, are the objective the reference optimises under nn.DataParallel."""

    def __init__(self, config):
        super().__init__()
        from . import ops
        self.PROPOSAL_NUM = int(config.proposal_num)
        self.raw_ce, self.concat_ce, self.part_ce = (ops.CrossEntropyLS(0.1) for _ in range(3))

    def forward(self, outputs, targets):
        from .ops_nts import RankLossFn
        raw_logits, concat_logits, part_logits, _, top_n_prob = outputs
        B, T = targets.shape[0], self.PROPOSAL_NUM
        if top_n_prob.shape != (B, T):
            raise ValueError(f'NTSLoss: top_n_prob {tuple(top_n_prob.shape)}, expected ({B}, {T}) (criterion proposal_num)')
        part_rows = part_logits.reshape(B * T, -1)
        part_targets = targets.repeat_interleave(T)
        loss = self.raw_ce(raw_logits, targets) + RankLossFn.apply(part_rows, targets, top_n_prob)
        loss = loss + self.concat_ce(concat_logits, targets) + self.part_ce(part_rows, part_targets)
        self.last_correct = self.concat_ce.last_correct
        return loss


class APCNNLoss(nn.Module):
    """Examples/APCNN.py:49: the sum of the base criterion (cross-entropy with label smoothing 0.1, train.py:211-212) over the
    eight logit tensors of the 4-tuple APCNN returns, as one hk_softmax_ce_ls launch over the stacked [8N, K] rows: its mean
    over 8N rows times 8 is the sum of the eight means.  ``last_correct`` is the top-1 count on ``out_mean``, the accuracy
    Examples/APCNN.py reports, from the same kernel without a gradient."""

    def __init__(self, config=None):
        super().__init__()
        self.label_smoothing = 0.1

    def forward(self, outputs, targets):
        from .ops import CrossEntropyLSFn
        out_mean, out_list = outputs[0], outputs[1]
        loss, _ = CrossEntropyLSFn.apply(torch.cat(out_list, dim=0), targets.repeat(len(out_list)), self.label_smoothing)
        with torch.no_grad():
            _, self.last_correct = CrossEntropyLSFn.apply(out_mean.detach(), targets, self.label_smoothing)
        return loss * float(len(out_list))


class MGECNNLoss(nn.Module):
    """Examples/MGE_CNN.py:43-45: the mean of the base criterion (cross-entropy with label smoothing 0.1) over the ten logit
    tensors MGE_CNN returns, as one hk_softmax_ce_ls launch over the stacked [10N, K] rows: with equal row counts, the mean
    over 10N rows is the mean of the ten means.  ``last_correct`` is the top-1 count on logits_gate, the accuracy
    Examples/MGE_CNN.py reports, from the same kernel without a gradient."""

    def __init__(self, config=None):
        super().__init__()
        self.label_smoothing = 0.1

    def forward(self, outputs, targets):
        from .ops import CrossEntropyLSFn
        logits = outputs['logits']
        loss, _ = CrossEntropyLSFn.apply(torch.cat(logits, dim=0), targets.repeat(len(logits)), self.label_smoothing)
        with torch.no_grad():
            _, self.last_correct = CrossEntropyLSFn.apply(logits[-1].detach(), targets, self.label_smoothing)
        return loss


class CINLoss(nn.Module):
    """model/loss/CIN_loss.py with the reference's config keys, defaults and ``h`` (nn.Linear(channel * feature_size,
    r_channel), initialised by utils.initialize_weights; state_dict keys ``h.weight`` / ``h.bias``).  What the reference
    computes, reproduced here:
    - pair_label = target[:B/2] == target[B/2]: every label of the first half against the ONE label target[B/2], not the
      second half element by element;
    - L1 = sum over those pairs of ||h(Z_CCI_i) - h(Z_CCI_{B/2+i}) + 1e-6||^2 (nn.PairwiseDistance's eps);
    - the margin hinge with ``beta`` is computed and then overwritten by L1^2, so ``beta`` changes nothing;
    - loss = CE_ls0.1(Z, target) + alpha (L1 + L1^2); the cross-entropy alone when the output is not a tuple (eval mode).
    With the class-by-class batches of BalancedBatchSampler (n_classes x n_samples, 4 x 5 in configs/CIN.yaml), target[B/2]
    is a class of the second half only, no pair matches, the contrastive term is 0 and ``h`` gets a zero gradient (not
    None): the optimizer's weight decay still shrinks it every step, as in the reference.

    The projection runs on the pair differences (ops_cin.PairDiffProjFn) and the contrastive term with its gradient in one
    launch that builds the pair mask on the device (ops_cin.ContrastiveLossFn): no host read-back, where the reference's
    boolean indexing synchronises four times per step.  ``last_correct`` is the top-1 count of the cross-entropy kernel."""

    def __init__(self, config):
        super().__init__()
        from . import ops
        from .utils import initialize_weights
        self.alpha = config.alpha if 'alpha' in config else 2.0
        self.beta = config.beta if 'beta' in config else 0.5            # read by nothing: see the class docstring
        self.channel = config.channel if 'channel' in config else 2048
        self.feature_size = config.feature_size if 'feature_size' in config else 7 * 7
        self.r_channel = config.r_channel if 'r_channel' in config else 512
        if self.r_channel % 4:
            raise ValueError(f'CINLoss: r_channel={self.r_channel} must be a multiple of 4 (16-byte row pitch of the '
                             'projection gradients)')
        self.ce_loss = ops.CrossEntropyLS(0.1)
        self.h = nn.Linear(self.channel * self.feature_size, self.r_channel)
        self.apply(initialize_weights)

    def forward(self, output, target):
        from .ops_cin import ContrastiveLossFn, PairDiffProjFn
        if not isinstance(output, tuple):
            loss = self.ce_loss(output, target)
            self.last_correct = self.ce_loss.last_correct
            return loss
        Z, Z_CCI = output
        B = Z_CCI.shape[0]
        if Z_CCI[0].numel() != self.h.in_features:
            raise ValueError(f'CINLoss: Z_CCI {tuple(Z_CCI.shape)} has {Z_CCI[0].numel()} features per sample, the criterion '
                             f'channel x feature_size = {self.channel} x {self.feature_size} = {self.h.in_features} (a '
                             '448x448 input gives a 14x14 map: feature_size 196)')
        loss_ce = self.ce_loss(Z, target)
        self.last_correct = self.ce_loss.last_correct
        p = PairDiffProjFn.apply(Z_CCI.reshape(B, -1), self.h.weight, self.h.bias)
        return loss_ce + ContrastiveLossFn.apply(p, target, self.alpha)


class PairConfusionFn(Function):
    """CE_ls(logits, labels) + lambda_a * sum_{i < B/2} [y_i != y_{B/2+i}] ||z_i - z_{B/2+i}|| / B -> (loss, top-1 count),
    forward and gradient in one hk_pc_loss launch (pair_confusion.py:15-28).  Backward scales the kept gradient."""

    @staticmethod
    def forward(ctx, logits, labels, smoothing, lambda_a):
        from . import _lib
        from .ops import _check_cuda, _f32c
        _check_cuda(logits, labels)
        logits = _f32c(logits)
        labels = labels.contiguous().to(torch.int64)
        B, K = logits.shape
        loss = torch.empty(1, device=logits.device, dtype=torch.float32)
        dlogits = torch.empty_like(logits)
        correct = torch.empty(1, device=logits.device, dtype=torch.int32)
        _lib.call('hk_pc_loss', logits, labels, loss, dlogits, correct, B, K, float(smoothing), float(lambda_a), 1.0,
                  _lib.stream_ptr())
        ctx.save_for_backward(dlogits)
        ctx.mark_non_differentiable(correct)
        return loss[0], correct

    @staticmethod
    def backward(ctx, g, _g_correct=None):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None, None


class PairwiseConfusionLoss(nn.Module):
    """model/loss/pair_confusion.py: CrossEntropy(label_smoothing=0.1) + lambda_a x the Euclidean confusion of the pairs
    (i, B/2 + i) with different labels, ||z_i - z_{B/2+i}|| summed and divided by B; ``lambda_a`` from the criterion config,
    10 by default.  An odd batch raises before any launch, as in the reference.  One hk_pc_loss launch; ``last_correct`` is
    the top-1 count on the device, so the training step reads nothing back."""

    def __init__(self, config):
        super().__init__()
        self.lambda_a = config.lambda_a if 'lambda_a' in config else 10
        self.label_smoothing = 0.1

    def forward(self, features, labels):
        if features.shape[0] % 2 != 0:
            raise ValueError(f'PairwiseConfusionLoss: incorrect batch size {features.shape[0]} (it must be even: the two '
                             'halves of the batch are paired)')
        loss, correct = PairConfusionFn.apply(features, labels, self.label_smoothing, self.lambda_a)
        self.last_correct = correct
        return loss


class InterpPartsLoss(nn.Module):
    """model/loss/InterpParts_loss.py: CrossEntropy(logits) + coeff x ShapingLoss(assign) on the (logits, att, assign)
    triple Interp-Parts returns, with the reference's config keys and defaults (radius 2, std 0.4, num_parts 5, alpha 1,
    beta 0.001, coeff 0.5).  ``last_correct`` is the top-1 count on the device.

    The Beta prior depends only on (N, alpha, beta): it is computed once per batch size with scipy and kept on the device,
    so after the first call with a batch size the loss makes no host round trip (the reference recomputes it on the host at
    every call, because its ``prev_bs`` is never updated).  Under torchrun every rank all-gathers the [N_local, K]
    occupancies, so that the ranking and the prior cover the global batch, as under the reference's nn.DataParallel, which
    gathers assign onto one device; the local rows' gradient is then scaled by the world size, which undoes the 1 / world
    averaging of the gradient all-reduce."""

    def __init__(self, config):
        super().__init__()
        from . import ops, ops_interp_parts
        self.radius = int(config.radius if 'radius' in config else 2)
        self.std = config.std if 'std' in config else 0.4
        self.num_parts = config.num_parts if 'num_parts' in config else 5
        self.alpha = config.alpha if 'alpha' in config else 1
        self.beta = config.beta if 'beta' in config else 0.001
        self.coeff = config.coeff if 'coeff' in config else 0.5
        if self.radius < 0:
            raise ValueError(f'InterpPartsLoss: radius={self.radius} must be >= 0')
        ops_interp_parts.check_parts(self.num_parts)
        self.ce_loss = ops.CrossEntropyLS(0.0)
        self._taps = ops_interp_parts.gaussian_taps(self.radius, self.std)
        self._device_taps = {}
        self._priors = {}

    def prior(self, n, device):
        """[n] fp32 Beta prior quantiles on ``device``, computed on the host the first time only."""
        key = (n, self.alpha, self.beta, str(device))
        if key not in self._priors:
            from .ops_interp_parts import beta_prior
            self._priors[key] = beta_prior(n, self.alpha, self.beta).to(device)
        return self._priors[key]

    def taps(self, device):
        key = str(device)
        if key not in self._device_taps:
            self._device_taps[key] = self._taps.to(device)
        return self._device_taps[key]

    def shaping_loss(self, assign):
        from .ops_interp_parts import SHAPING_EPS, ShapingLossFn, occupancy
        if assign.shape[1] != self.num_parts:
            raise ValueError(f'InterpPartsLoss: assign has {assign.shape[1]} parts, the criterion num_parts={self.num_parts}')
        occ, _ = occupancy(assign, self.taps(assign.device), self.radius)
        occ_all, row0, world = occ.detach(), 0, 1
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            world = dist.get_world_size()
            occ_all = torch.empty(world * occ.shape[0], occ.shape[1], device=occ.device, dtype=occ.dtype)
            dist.all_gather_into_tensor(occ_all, occ.detach().contiguous())
            row0 = dist.get_rank() * occ.shape[0]
        return ShapingLossFn.apply(occ, occ_all, self.prior(occ_all.shape[0], occ.device), row0, world, SHAPING_EPS)

    def forward(self, output, target):
        logits, att, assign = output
        loss_ce = self.ce_loss(logits, target)
        self.last_correct = self.ce_loss.last_correct
        return loss_ce + self.coeff * self.shaping_loss(assign)
