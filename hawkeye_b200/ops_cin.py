"""Autograd bindings for the channel-interaction module (reference model/methods/CIN.py:24-60): batched Gram and W.X
products on the wgmma GEMM, softmax(-G), the contrastive weight |W_SCI - w W_SCI_BA|, the 3x3 convolution on the
implicit-GEMM kernels (NCHW in / out), and the classifier's spatial mean.  Host plumbing only; all arithmetic is in
libhawkeye_b200.so."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws


def _gemm(A, a_mn, lda, sA, B, b_mn, ldb, sB, C, ldc, sC, M, N, K, batch, alpha=1.0, D=None, ldd=0, sD=0, beta=0.0,
          exact=False):
    _lib.call('hk_gemm_3xtf32' if exact else 'hk_gemm_tf32', A, int(a_mn), lda, sA, B, int(b_mn), ldb, sB, C, ldc, sC, 0, M, N, K, batch, float(alpha), None,
              0.0, D, ldd, sD, float(beta), None, 0, _lib.stream_ptr())


class GramFn(Function):
    """G = alpha * X X^T,  X [B, C, P] (P % 4 == 0; zero-padded columns are harmless)  ->  [B, C, C]       (CIN.py:31)"""

    @staticmethod
    def forward(ctx, x, alpha):
        _check_cuda(x)
        x = _f32c(x)
        B, C, P = x.shape
        g = torch.empty(B, C, C, device=x.device, dtype=torch.float32)
        # 3xTF32: G feeds exp(-G) with |G| in the tens — a 5e-4 relative TF32 error would be percents of the softmax
        _gemm(x, 0, P, C * P, x, 0, P, C * P, g, C, C * C, C, C, P, B, alpha, exact=True)
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
        _gemm(dg, 0, C, C * C, x, 1, P, C * P, dx, P, C * P, C, P, C, B, ctx.alpha)
        _gemm(dg, 1, C, C * C, x, 1, P, C * P, dx, P, C * P, C, P, C, B, ctx.alpha, D=dx, ldd=P, sD=C * P, beta=1.0)
        return dx, None


class WXFn(Function):
    """Y = W X,  W [B, C, C], X [B, C, P] -> [B, C, P]                                                   (CIN.py:34, :55)"""

    @staticmethod
    def forward(ctx, w, x):
        _check_cuda(w, x)
        w, x = _f32c(w), _f32c(x)
        B, C, P = x.shape
        y = torch.empty_like(x)
        _gemm(w, 0, C, C * C, x, 1, P, C * P, y, P, C * P, C, P, C, B)
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
            _gemm(dy, 0, P, C * P, x, 0, P, C * P, dw, C, C * C, C, C, P, B)            # dW = dY X^T
        if ctx.needs_input_grad[1]:
            dx = torch.empty_like(x)
            _gemm(w, 1, C, C * C, dy, 1, P, C * P, dx, P, C * P, C, P, C, B)            # dX = W^T dY
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
        x, w = _f32c(x), _f32c(w)
        s = _lib.stream_ptr()
        N, C, H, W = x.shape
        cout = w.shape[0]
        xn = torch.empty(N, H, W, C, device=x.device, dtype=torch.float32)
        _lib.call('hk_nchw_to_nhwc', x, xn, N, H * W, C, s)
        wf = torch.empty(9 * cout * C, device=x.device, dtype=torch.float32)
        wd = torch.empty(9 * cout * C, device=x.device, dtype=torch.float32)
        _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, C, s)
        yn = torch.empty(N, H, W, cout, device=x.device, dtype=torch.float32)
        _lib.call('hk_conv3x3_fwd', xn, wf, b, yn, N, H, W, C, cout, 0, s)
        y = torch.empty(N, cout, H, W, device=x.device, dtype=torch.float32)
        _lib.call('hk_nhwc_to_nchw', yn, y, N, H * W, cout, s)
        ctx.save_for_backward(xn, wd)
        ctx.shape = (N, C, H, W, cout)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        xn, wd = ctx.saved_tensors
        N, C, H, W, cout = ctx.shape
        s = _lib.stream_ptr()
        dev = dy.device
        dy = _f32c(dy)
        g = torch.empty(N, H, W, cout, device=dev, dtype=torch.float32)
        _lib.call('hk_nchw_to_nhwc', dy, g, N, H * W, cout, s)
        dw = torch.empty(cout, C, 3, 3, device=dev, dtype=torch.float32)
        db = torch.empty(cout, device=dev, dtype=torch.float32) if ctx.has_bias else None
        ws = _ws(_lib.query('hk_conv3x3_wgrad_workspace_bytes', C, cout), dev)
        _lib.call('hk_conv3x3_wgrad', xn, g, dw, db, N, H, W, C, cout, ws, ws.numel(), s)
        dx = None
        if ctx.needs_input_grad[0]:
            dxn = torch.empty(N, H, W, C, device=dev, dtype=torch.float32)
            _lib.call('hk_conv3x3_dgrad', g, wd, None, dxn, N, H, W, C, cout, s)
            dx = torch.empty(N, C, H, W, device=dev, dtype=torch.float32)
            _lib.call('hk_nhwc_to_nchw', dxn, dx, N, H * W, C, s)
        return dx, dw, db


class RowMeanFn(Function):
    """AdaptiveAvgPool1d(1) over the last dimension (CIN.py:71): [..., P] -> [...]"""

    @staticmethod
    def forward(ctx, x):
        _check_cuda(x)
        x = _f32c(x)
        P = x.shape[-1]
        y = torch.empty(x.shape[:-1], device=x.device, dtype=torch.float32)
        _lib.call('hk_row_mean_fwd', x, y, x.numel() // P, P, P, _lib.stream_ptr())
        ctx.P = P
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _f32c(dy)
        dx = torch.empty(*dy.shape, ctx.P, device=dy.device, dtype=torch.float32)
        _lib.call('hk_row_mean_bwd', dy, dx, dy.numel(), ctx.P, ctx.P, _lib.stream_ptr())
        return dx


class AddFn(Function):
    """a + b (residual, CIN.py:38,59) on hk_add_inplace"""

    @staticmethod
    def forward(ctx, a, b):
        out = _f32c(a).clone()
        _lib.call('hk_add_inplace', out, _f32c(b), out.numel(), _lib.stream_ptr())
        return out

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


class ReluFn(Function):
    @staticmethod
    def forward(ctx, x):
        x = _f32c(x)
        y = torch.empty_like(x)
        _lib.call('hk_relu_fwd', x, y, x.numel(), _lib.stream_ptr())
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        dx = torch.empty_like(y)
        _lib.call('hk_relu_bwd', y, _f32c(dy), dx, y.numel(), _lib.stream_ptr())
        return dx
