"""Autograd bindings for APINet's attentive pairwise interaction (reference model/methods/APINet.py:28-119 and
model/loss/APINet_loss.py): pair mining on the device, the pair head (gather -> map1 -> dropout -> map2 -> attentive gate with
its four dropouts) as one autograd node, and the cross-entropy + margin-ranking loss.  Host plumbing only; all arithmetic is
in libhawkeye_b200.so."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, gemm, linear_fwd

# dropout call ids, in the reference's call order: drop(map1_out), then drop(f1_self), drop(f1_other), drop(f2_self),
# drop(f2_other) (the gate kernel uses GATE_CALL + 0..3)
MAP1_CALL, GATE_CALL = 0, 1
RANK_MARGIN = 0.05                      # nn.MarginRankingLoss(margin=0.05), APINet_loss.py:11


def mine_pairs(pool, labels):
    """get_pairs (APINet.py:76-113) on the device: -> (idx2, labels1, labels2), all int64 [2n]; idx2 = cat(intra, inter).
    No host round trip, so the step stays free of synchronisation and can be captured in a CUDA graph."""
    _check_cuda(pool, labels)
    pool = _f32c(pool)
    n, D = pool.shape
    labels = labels.contiguous().to(torch.int64)
    idx2 = torch.empty(2 * n, device=pool.device, dtype=torch.int64)
    lab = torch.empty(2, 2 * n, device=pool.device, dtype=torch.int64)
    _lib.call('hk_apinet_pairs', pool, labels, idx2, idx2[n:], lab[0], lab[1], n, D, _lib.stream_ptr())
    return idx2, lab[0], lab[1]


class PairHeadFn(Function):
    """pool [n, D], idx2 [2n]  ->  [8n, D] = [f1_self; f2_self; f1_other; f2_other] after dropout (APINet.py:36-61).

    mutual = [pool[idx1] | pool[idx2]] -> map1 -> dropout -> map2 = m;  g1 = sigmoid(m f1), g2 = sigmoid(m f2);  the four
    gated features.  ``seed`` is a device int64 (None when p == 0): the masks are a hash of it, recomputed in backward.
    Backward: the gate kernel writes dm and mutual's gate gradient, map1's dgrad accumulates onto the latter through the
    GEMM's addend, and the scatter folds both halves of dmutual back onto pool in a fixed order."""

    @staticmethod
    def forward(ctx, pool, idx2, w1, b1, w2, b2, seed, p):
        _check_cuda(pool, idx2, w1, b1, w2, b2)
        pool, w1, w2 = _f32c(pool), _f32c(w1), _f32c(w2)
        n, D = pool.shape
        dev, s = pool.device, _lib.stream_ptr()
        mutual = torch.empty(2 * n, 2 * D, device=dev, dtype=torch.float32)
        _lib.call('hk_apinet_gather', pool, idx2, mutual, n, D, s)
        h = linear_fwd(mutual, w1, b1)
        if p > 0:
            hd = torch.empty_like(h)
            _lib.call('hk_dropout_fwd', h, hd, h.numel(), float(p), seed, MAP1_CALL, s)
        else:
            hd = h
        m = linear_fwd(hd, w2, b2)
        out = torch.empty(8 * n, D, device=dev, dtype=torch.float32)
        _lib.call('hk_apinet_gate_fwd', m, mutual, out, 2 * n, D, float(p), seed, GATE_CALL, s)
        ctx.save_for_backward(idx2, mutual, hd, m, w1, w2, seed)
        ctx.p = float(p)
        ctx.has_bias = (b1 is not None, b2 is not None)
        return out

    @staticmethod
    def backward(ctx, dout):
        idx2, mutual, hd, m, w1, w2, seed = ctx.saved_tensors
        p = ctx.p
        dev, s = mutual.device, _lib.stream_ptr()
        R, F = mutual.shape                                   # 2n, 2D
        n, D, H = R // 2, F // 2, w1.shape[0]
        dout = _f32c(dout)
        dm = torch.empty_like(m)
        dmutual = torch.empty_like(mutual)
        _lib.call('hk_apinet_gate_bwd', m, mutual, dout, dm, dmutual, R, D, p, seed, GATE_CALL, s)
        # map2: dW2, db2 from dm and the (dropped-out) map1 output; d(dropout output) = dm . W2
        dw2 = torch.empty_like(w2)
        db2 = torch.empty(D, device=dev, dtype=torch.float32) if ctx.has_bias[1] else None
        _lib.call('hk_linear_wgrad', dm, hd, dw2, db2, R, H, D, s)
        dh = torch.empty(R, H, device=dev, dtype=torch.float32)
        _lib.call('hk_linear_dgrad', dm, w2, dh, R, H, D, s)
        if p > 0:
            dhd, dh = dh, torch.empty_like(dh)
            _lib.call('hk_dropout_bwd', dhd, dh, dh.numel(), p, seed, MAP1_CALL, s)
        dw1 = torch.empty_like(w1)
        db1 = torch.empty(H, device=dev, dtype=torch.float32) if ctx.has_bias[0] else None
        _lib.call('hk_linear_wgrad', dh, mutual, dw1, db1, R, F, H, s)
        # dmutual += dh . W1  (map1's dgrad, accumulated onto the gate's contribution)
        gemm(dh, 0, H, 0, w1, 1, F, 0, dmutual, F, 0, R, F, H, D=dmutual, ldd=F, beta=1.0)
        dpool = torch.empty(n, D, device=dev, dtype=torch.float32)
        _lib.call('hk_apinet_scatter', dmutual, idx2, dpool, n, D, s)
        return dpool, None, dw1, db1, dw2, db2, None, None


def pair_head(pool, idx2, map1, map2, p, seed):
    return PairHeadFn.apply(pool, idx2, map1.weight, map1.bias, map2.weight, map2.bias, seed, p)


class APINetLossFn(Function):
    """logits [8n, K] (rows r and r + 4n are a (self, other) pair), targets [8n] -> (CE(label_smoothing 0.1) + margin ranking
    loss, top-1 count).  One cross-entropy kernel over all rows, then the ranking kernel adds its term and its gradient."""

    @staticmethod
    def forward(ctx, logits, targets, margin):
        _check_cuda(logits, targets)
        logits = _f32c(logits)
        targets = targets.contiguous().to(torch.int64)
        B, K = logits.shape
        if B % 2:
            raise _lib.HawkeyeLibError(f'APINetLoss: {B} logit rows, expected an even number (self rows, then other rows)')
        dev, s = logits.device, _lib.stream_ptr()
        ce = torch.empty(1, device=dev, dtype=torch.float32)
        dlogits = torch.empty_like(logits)
        correct = torch.empty(1, device=dev, dtype=torch.int32)
        _lib.call('hk_softmax_ce_ls', logits, targets, ce, dlogits, correct, B, K, 0.1, 1.0, s)
        rank = torch.zeros(1, device=dev, dtype=torch.float64)
        _lib.call('hk_apinet_rank_loss', logits, targets, rank, dlogits, B // 2, K, float(margin), 1.0, s)
        ctx.save_for_backward(dlogits)
        ctx.mark_non_differentiable(correct)
        return ce[0] + rank[0].float(), correct

    @staticmethod
    def backward(ctx, g, _g_correct=None):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None
