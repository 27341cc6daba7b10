"""Autograd bindings for the channel-interaction module (reference model/methods/CIN.py:24-60): batched Gram and W.X
products on the wgmma GEMM, softmax(-G), the contrastive weight |W_SCI - w W_SCI_BA|, the residual add and OSME's
excitation gate (the 3x3 convolution is ops.Conv3x3Fn), and the pair-difference projection and contrastive term of CIN's
loss (model/loss/CIN_loss.py).  Host plumbing only; all arithmetic is in libhawkeye_b200.so."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, add_, gemm, linear_fwd


class GramFn(Function):
    """G = alpha * X X^T,  X [B, C, P] (P % 4 == 0; zero-padded columns are harmless)  ->  [B, C, C]       (CIN.py:31)"""

    @staticmethod
    def forward(ctx, x, alpha):
        _check_cuda(x)
        x = _f32c(x)
        B, C, P = x.shape
        g = torch.empty(B, C, C, device=x.device, dtype=torch.float32)
        # 3xTF32: G feeds exp(-G) with |G| in the tens — a 5e-4 relative TF32 error would be percents of the softmax
        gemm(x, 0, P, C * P, x, 0, P, C * P, g, C, C * C, C, C, P, B, alpha, exact=True)
        ctx.save_for_backward(x)
        ctx.alpha = alpha
        return g

    @staticmethod
    def backward(ctx, dg):
        (x,) = ctx.saved_tensors
        B, C, P = x.shape
        dg = _f32c(dg)
        dx = torch.empty_like(x)
        # dX = alpha (dG + dG^T) X : two products, the second accumulates onto the first
        gemm(dg, 0, C, C * C, x, 1, P, C * P, dx, P, C * P, C, P, C, B, ctx.alpha)
        gemm(dg, 1, C, C * C, x, 1, P, C * P, dx, P, C * P, C, P, C, B, ctx.alpha, D=dx, ldd=P, sD=C * P, beta=1.0)
        return dx, None


class WXFn(Function):
    """Y = W X,  W [B, C, C], X [B, C, P] -> [B, C, P]                                                   (CIN.py:34, :55)"""

    @staticmethod
    def forward(ctx, w, x):
        _check_cuda(w, x)
        w, x = _f32c(w), _f32c(x)
        B, C, P = x.shape
        y = torch.empty_like(x)
        gemm(w, 0, C, C * C, x, 1, P, C * P, y, P, C * P, C, P, C, B)
        ctx.save_for_backward(w, x)
        return y

    @staticmethod
    def backward(ctx, dy):
        w, x = ctx.saved_tensors
        B, C, P = x.shape
        dy = _f32c(dy)
        dw = dx = None
        if ctx.needs_input_grad[0]:
            dw = torch.empty_like(w)
            gemm(dy, 0, P, C * P, x, 0, P, C * P, dw, C, C * C, C, C, P, B)             # dW = dY X^T
        if ctx.needs_input_grad[1]:
            dx = torch.empty_like(x)
            gemm(w, 1, C, C * C, dy, 1, P, C * P, dx, P, C * P, C, P, C, B)             # dX = W^T dY
        return dw, dx


class SoftmaxNegFn(Function):
    """softmax(-g, dim=-1)                                                                              (CIN.py:32)"""

    @staticmethod
    def forward(ctx, g):
        _check_cuda(g)
        g = _f32c(g)
        w = torch.empty_like(g)
        _lib.call('hk_softmax_neg_rows_fwd', g, w, g.numel() // g.shape[-1], g.shape[-1], _lib.stream_ptr())
        ctx.save_for_backward(w)
        return w

    @staticmethod
    def backward(ctx, dw):
        (w,) = ctx.saved_tensors
        dg = torch.empty_like(w)
        _lib.call('hk_softmax_neg_rows_bwd', w, _f32c(dw), dg, w.numel() // w.shape[-1], w.shape[-1], _lib.stream_ptr())
        return dg


class CCIWeightFn(Function):
    """| W_SCI[b] - weight[b] W_SCI[(b + B/2) % B] |                                                    (CIN.py:50-53)"""

    @staticmethod
    def forward(ctx, w_sci, weight):
        _check_cuda(w_sci, weight)
        w_sci, weight = _f32c(w_sci), _f32c(weight)
        B = w_sci.shape[0]
        out = torch.empty_like(w_sci)
        _lib.call('hk_cci_weight_fwd', w_sci, weight, out, B, w_sci.numel() // B, _lib.stream_ptr())
        ctx.save_for_backward(w_sci, weight)
        return out

    @staticmethod
    def backward(ctx, d):
        w_sci, weight = ctx.saved_tensors
        B = w_sci.shape[0]
        d_sci = torch.empty_like(w_sci)
        d_w = torch.empty_like(weight)
        _lib.call('hk_cci_weight_bwd', w_sci, weight, _f32c(d), d_sci, d_w, B, w_sci.numel() // B, _lib.stream_ptr())
        return d_sci, d_w


class AddFn(Function):
    """a + b (residual, CIN.py:38,59) on hk_add_inplace"""

    @staticmethod
    def forward(ctx, a, b):
        return add_(_f32c(a).clone(), _f32c(b))

    @staticmethod
    def backward(ctx, g):
        return g, g


class PairDiffProjFn(Function):
    """P = h(z[:B/2]) - h(z[B/2:]) = (z[:B/2] - z[B/2:]) W^T,  z [B, F], W [R, F] -> [B/2, R]       (CIN_loss.py:36-41)

    The bias cancels, so the projection runs once, on the difference: half the GEMM, and TF32 rounds the difference instead
    of two nearly equal operands (a same-class pair), whose separate rounding would lose most of it.  ``bias`` is an input
    so that it receives its gradient, which is zero: a parameter that never accumulates one would keep the early-group
    all-reduce of engine.GradAllReduce from firing."""

    @staticmethod
    def forward(ctx, z, weight, bias):
        _check_cuda(z, weight, bias)
        z, weight = _f32c(z), _f32c(weight)
        B, F = z.shape
        d = torch.empty(B // 2, F, device=z.device, dtype=torch.float32)
        _lib.call('hk_cin_pair_diff_fwd', z, d, B, F, _lib.stream_ptr())
        ctx.save_for_backward(d, weight)
        ctx.B = B
        return linear_fwd(d, weight, None)

    @staticmethod
    def backward(ctx, dp):
        d, weight = ctx.saved_tensors
        dp = _f32c(dp)
        half, F = d.shape
        R = weight.shape[0]
        s = _lib.stream_ptr()
        dz = dw = db = None
        if ctx.needs_input_grad[0]:
            dd = torch.empty_like(d)
            _lib.call('hk_linear_dgrad', dp, weight, dd, half, F, R, s)
            dz = torch.empty(ctx.B, F, device=d.device, dtype=torch.float32)
            _lib.call('hk_cin_pair_diff_bwd', dd, dz, ctx.B, F, s)
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(weight)
            _lib.call('hk_linear_wgrad', dp, d, dw, None, half, F, R, s)
        if ctx.needs_input_grad[2]:
            db = torch.zeros(R, device=d.device, dtype=torch.float32)
        return dz, dw, db


class ContrastiveLossFn(Function):
    """alpha (L1 + L1^2) over the pairs i with labels[i] == labels[B/2], L1 = sum ||p_i + 1e-6||^2; p [B/2, R], labels [B].
    Forward and gradient in one hk_cin_contrastive_loss launch (CIN_loss.py:36-46)."""

    @staticmethod
    def forward(ctx, p, labels, alpha):
        _check_cuda(p, labels)
        p = _f32c(p)
        labels = labels.contiguous().to(torch.int64)
        B = labels.numel()
        if B % 2 or p.shape[0] != B // 2:
            raise _lib.HawkeyeLibError(f'CIN contrastive loss: {B} labels for {p.shape[0]} pairs (the batch must be even)')
        loss = torch.empty(1, device=p.device, dtype=torch.float32)
        dp = torch.empty_like(p)
        _lib.call('hk_cin_contrastive_loss', p, labels, loss, dp, B, p.shape[1], float(alpha), _lib.stream_ptr())
        ctx.save_for_backward(dp)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dp,) = ctx.saved_tensors
        return dp * g, None, None


class SEGateFn(Function):
    """sigmoid(m)[n, c] * x[n, c, :, :]  (OSME.py:19-23)"""

    @staticmethod
    def forward(ctx, x, m):
        _check_cuda(x, m)
        x, m = _f32c(x), _f32c(m)
        N, C = x.shape[:2]
        hw = x.numel() // (N * C)
        s = torch.empty_like(x)
        _lib.call('hk_se_gate_fwd', x, m, s, N * C, hw, _lib.stream_ptr())
        ctx.save_for_backward(x, m)
        return s

    @staticmethod
    def backward(ctx, ds):
        x, m = ctx.saved_tensors
        N, C = x.shape[:2]
        hw = x.numel() // (N * C)
        dx, dm = torch.empty_like(x), torch.empty_like(m)
        _lib.call('hk_se_gate_bwd', x, m, _f32c(ds), dx, dm, N * C, hw, _lib.stream_ptr())
        return dx, dm
