"""Autograd bindings for DCL (reference model/methods/DCL.py:31-45 and model/loss/DCL_loss.py): the region-alignment head
(global average pool, 1x1 Convmask, AvgPool2d(2), tanh) as one node, the two bias-free classifiers as one stacked GEMM node,
and the loss.  Host plumbing only; all arithmetic is in libhawkeye_b200.so."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws, linear_fwd


class DCLHeadFn(Function):
    """x [N, C, H, W] (the trunk output), Convmask weight [1, C, 1, 1] and bias [1] -> (pooled [N, C], mask [N, Q])."""

    @staticmethod
    def forward(ctx, x, w, b):
        _check_cuda(x, w, b)
        x, w, b = _f32c(x), _f32c(w), _f32c(b)
        if x.dim() != 4 or w.numel() != x.shape[1] or b.numel() != 1:
            raise _lib.HawkeyeLibError(f'DCLHeadFn: x {tuple(x.shape)} needs a [N, C, H, W] map, a Convmask weight of C '
                                       f'elements (got {w.numel()}) and one bias (got {b.numel()})')
        N, C, H, W = x.shape
        dev = x.device
        pooled = torch.empty(N, C, device=dev, dtype=torch.float32)
        mask = torch.empty(N, (H // 2) * (W // 2), device=dev, dtype=torch.float32)
        ws = _ws(_lib.query('hk_dcl_head_workspace_bytes', N, C, H, W), dev)
        _lib.call('hk_dcl_head_fwd', x, w, b, pooled, mask, N, C, H, W, ws, ws.numel(), _lib.stream_ptr())
        ctx.save_for_backward(x, w, mask)
        ctx.w_shape = w.shape
        return pooled, mask

    @staticmethod
    def backward(ctx, dpooled, dmask):
        x, w, mask = ctx.saved_tensors
        N, C, H, W = x.shape
        dev = x.device
        dpooled = torch.zeros(N, C, device=dev) if dpooled is None else _f32c(dpooled)
        dmask = torch.zeros_like(mask) if dmask is None else _f32c(dmask)
        dx = torch.empty_like(x)
        dw = torch.empty(ctx.w_shape, device=dev, dtype=torch.float32)
        db = torch.empty(1, device=dev, dtype=torch.float32)
        ws = _ws(_lib.query('hk_dcl_head_workspace_bytes', N, C, H, W), dev)
        _lib.call('hk_dcl_head_bwd', x, w, mask, dpooled, dmask, dx, dw, db, N, C, H, W, ws, ws.numel(), _lib.stream_ptr())
        return dx, dw, db


def stacked_rows(K, K2):
    """Rows of the stacked classifier weight: K + K2 rounded up to a multiple of 4 (16-byte TMA row pitch of dlogits)."""
    return (K + K2 + 3) // 4 * 4


class StackedClassifierFn(Function):
    """pooled [R, F], classifier.weight [K, F], classifier_swap.weight [K2, F] -> logits [R, Kp] = pooled . [W; W2; 0]^T,
    Kp = stacked_rows(K, K2): one hk_linear_fwd without bias; backward one hk_linear_dgrad and one hk_linear_wgrad whose
    [Kp, F] weight gradient is split back into the two parameters."""

    @staticmethod
    def forward(ctx, x, w, w2):
        _check_cuda(x, w, w2)
        x, w, w2 = _f32c(x), _f32c(w), _f32c(w2)
        K, K2, F = w.shape[0], w2.shape[0], w.shape[1]
        ws = torch.zeros(stacked_rows(K, K2), F, device=x.device, dtype=torch.float32)
        ws[:K].copy_(w)
        ws[K:K + K2].copy_(w2)
        y = linear_fwd(x, ws, None)
        ctx.save_for_backward(x, ws)
        ctx.split = (K, K2)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, ws = ctx.saved_tensors
        K, K2 = ctx.split
        dy = _f32c(dy)
        R, F = x.shape
        Kp = ws.shape[0]
        s = _lib.stream_ptr()
        dx = dw = dw2 = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _lib.call('hk_linear_dgrad', dy, ws, dx, R, F, Kp, s)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dws = torch.empty_like(ws)
            _lib.call('hk_linear_wgrad', dy, x, dws, None, R, F, Kp, s)
            dw, dw2 = dws[:K], dws[K:K + K2]
        return dx, dw, dw2


def check_loss_shapes(logits, K, K2, labels, labels_swap, mask, law):
    """Every per-row input of DCLLossFn must have the logits' R rows, and the mask and the swap law the same width: the
    kernel indexes all of them by row.  Shapes are known on the host, so this costs no synchronisation."""
    if logits.dim() != 2 or K + K2 > logits.shape[1]:
        raise _lib.HawkeyeLibError(f'DCLLoss: logits {tuple(logits.shape)} do not hold {K} + {K2} columns')
    R = logits.shape[0]
    if mask.dim() != 2 or law.dim() != 2:
        raise _lib.HawkeyeLibError(f'DCLLoss: mask {tuple(mask.shape)} and swap_law {tuple(law.shape)} must be [rows, cells]')
    if mask.shape[1] != law.shape[1]:
        side = int(round(law.shape[1] ** 0.5))
        raise _lib.HawkeyeLibError(
            f'DCLLoss: the region-alignment mask has {mask.shape[1]} entries per image but swap_law has {law.shape[1]}: the '
            f'mask has one entry per 2x2 window of the trunk map (input size / 64 per side, so {64 * side}x{64 * side} inputs '
            f'for swap_num [{side}, {side}]); match the input size and swap_num')
    rows = dict(labels=labels.numel(), labels_swap=labels_swap.numel(), mask=mask.shape[0], swap_law=law.shape[0])
    if any(n != R for n in rows.values()):
        raise _lib.HawkeyeLibError(f'DCLLoss: {R} logit rows, but ' + ', '.join(f'{k} has {n}' for k, n in rows.items()))


class DCLLossFn(Function):
    """logits [R, ld] (classifier columns [0, K), classifier_swap columns [K, K + K2)), labels / labels_swap [R], mask / law
    [R, Q] -> (alpha CE + beta CE_swap + gamma L1, top-1 count).  One hk_dcl_loss launch writes the loss and both
    gradients; ``combine`` takes the top-1 count over the summed cls_2xmul logits (Examples/DCL.py:104-107)."""

    @staticmethod
    def forward(ctx, logits, K, K2, labels, labels_swap, mask, law, alpha, beta, gamma, combine):
        check_loss_shapes(logits, K, K2, labels, labels_swap, mask, law)
        _check_cuda(logits, labels, labels_swap, mask, law)
        logits, mask, law = _f32c(logits), _f32c(mask), _f32c(law)
        labels = labels.contiguous().to(torch.int64)
        labels_swap = labels_swap.contiguous().to(torch.int64)
        R, ld = logits.shape
        Q = mask.shape[1]
        dev = logits.device
        acc = torch.zeros(1, device=dev, dtype=torch.float64)
        dlogits = torch.empty_like(logits)
        dmask = torch.empty_like(mask)
        correct = torch.empty(1, device=dev, dtype=torch.int32)
        _lib.call('hk_dcl_loss', logits, ld, K, K2, labels, labels_swap, mask, law, R, Q, float(alpha), float(beta),
                  float(gamma), int(combine), acc, dlogits, dmask, correct, _lib.stream_ptr())
        ctx.save_for_backward(dlogits, dmask)
        ctx.mark_non_differentiable(correct)
        return acc[0].float(), correct

    @staticmethod
    def backward(ctx, g, _g_correct=None):
        dlogits, dmask = ctx.saved_tensors
        return dlogits * g, None, None, None, None, dmask * g, None, None, None, None, None
