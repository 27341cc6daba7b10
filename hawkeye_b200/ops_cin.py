"""Autograd bindings for the channel-interaction module (reference model/methods/CIN.py:24-60): batched Gram and W.X
products on the wgmma GEMM, softmax(-G), the contrastive weight |W_SCI - w W_SCI_BA|, the 3x3 convolution on the
implicit-GEMM kernels (NCHW in / out), the residual add and OSME's excitation gate.  Host plumbing only; all arithmetic is in
libhawkeye_b200.so."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import (_check_cuda, _f32c, add_, conv3x3_dgrad, conv3x3_fwd, conv3x3_pack, conv3x3_wgrad, gemm, nchw_to_nhwc,
                  nhwc_to_nchw)


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


class Conv3x3NCHWFn(Function):
    """nn.Conv2d(C, C, 3, 1, 1) on an NCHW map (CIN.py:22,36,57): NHWC inside, wgmma implicit GEMM."""

    @staticmethod
    def forward(ctx, x, w, b):
        _check_cuda(x, w, b)
        xn = nchw_to_nhwc(_f32c(x))
        wf, wd = conv3x3_pack(_f32c(w), True)
        y = nhwc_to_nchw(conv3x3_fwd(xn, wf, b, relu=False))
        ctx.save_for_backward(xn, wd)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        xn, wd = ctx.saved_tensors
        g = nchw_to_nhwc(_f32c(dy))
        cin, cout = xn.shape[-1], g.shape[-1]
        dw = torch.empty(cout, cin, 3, 3, device=g.device, dtype=torch.float32)
        db = torch.empty(cout, device=g.device, dtype=torch.float32) if ctx.has_bias else None
        conv3x3_wgrad(xn, g, dw, db)
        dx = nhwc_to_nchw(conv3x3_dgrad(g, wd)) if ctx.needs_input_grad[0] else None
        return dx, dw, db


class AddFn(Function):
    """a + b (residual, CIN.py:38,59) on hk_add_inplace"""

    @staticmethod
    def forward(ctx, a, b):
        return add_(_f32c(a).clone(), _f32c(b))

    @staticmethod
    def backward(ctx, g):
        return g, g


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
