"""torch.autograd bindings of the C-ABI kernels (host plumbing only: memory, streams, autograd edges).

Every op here calls ``libhawkeye_b200.so`` through ``_lib.call``; there is no PyTorch-eager fallback.
PyTorch owns all device buffers (caching allocator) incl. workspaces and saved-for-backward tensors.
"""
import torch
from torch.autograd import Function

from . import _lib

# Parity tests only: when set to a list, forward passes append the decisions they took at the non-smooth points of the
# path, in execution order — ('relu', y NHWC) after every ReLU, ('pool2', x NHWC) before every 2x2 max-pool,
# ('pool3', argmax u8 NHWC, input shape) for the ResNet stem pool, ('ssqrt', bins) for CBCNN's signed square root —
# so that a CPU oracle can be evaluated on the same branch of the piecewise-smooth function (oracle.hop_oracle.MaskTape).
CAPTURE = None


def _grad_ready(p):
    g = getattr(p, 'grad', None)
    return (g is not None and p.requires_grad and g.is_cuda and g.dtype == torch.float32 and g.is_contiguous()
            and g.shape == p.shape and not p._backward_hooks and not getattr(p, '_post_accumulate_grad_hooks', None))


def _check_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.HawkeyeLibError('hawkeye_b200 ops need CUDA tensors (there is no CPU fallback)')


def _f32c(t):
    if t.dtype != torch.float32:
        raise _lib.HawkeyeLibError(f'hawkeye_b200 ops are fp32 (got {t.dtype})')
    return t.contiguous()


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def wants_grad(x, params):
    """Save-for-backward decision, taken from what requires grad at call time (grad mode is always off inside
    Function.forward, so callers decide before ``apply``; freezing / unfreezing parameters after construction just works)."""
    return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))


# ----------------------------------------------------------------------------------------------------------
# shared host bindings: GEMM, linear forward, NCHW <-> NHWC, 3x3 convolution on NHWC maps
# ----------------------------------------------------------------------------------------------------------
def gemm(A, a_mn, lda, sA, B, b_mn, ldb, sB, C, ldc, sC, M, N, K, batch=1, alpha=1.0, alpha_vec=None, diag=0.0, D=None,
         ldd=0, sD=0, beta=0.0, beta_vec=None, relu=False, trans_c=False, exact=False):
    """C[b] = alpha*alpha_vec * A[b].B[b] + diag*I + beta*beta_vec * D[b] (then ReLU; C^T stored if trans_c) on the wgmma
    GEMM, with raw leading dimensions and batch strides (0 = shared across the batch).  A is [M,K] (or [K,M] if a_mn),
    B is [N,K] (or [K,N] if b_mn).  ``exact`` runs 3xTF32 whatever the library's precision mode."""
    _lib.call('hk_gemm_3xtf32' if exact else 'hk_gemm_tf32', A, int(a_mn), lda, sA, B, int(b_mn), ldb, sB, C, ldc, sC,
              int(trans_c), M, N, K, batch, float(alpha), alpha_vec, float(diag), D, ldd, sD, float(beta), beta_vec,
              int(relu), _lib.stream_ptr())


def linear_fwd(x, w, b):
    """y = x w^T + b: x [B, F], w [N, F], b [N] or None -> [B, N]"""
    B, F = x.shape
    N = w.shape[0]
    y = torch.empty(B, N, device=x.device, dtype=torch.float32)
    ws = _ws(_lib.query('hk_linear_fwd_workspace_bytes', B, F, N), x.device)
    _lib.call('hk_linear_fwd', x, w, b, y, B, F, N, ws, ws.numel(), _lib.stream_ptr())
    return y


def nchw_to_nhwc(x):
    N, C, H, W = x.shape
    y = torch.empty(N, H, W, C, device=x.device, dtype=torch.float32)
    _lib.call('hk_nchw_to_nhwc', x, y, N, H * W, C, _lib.stream_ptr())
    return y


def nhwc_to_nchw(x):
    N, H, W, C = x.shape
    y = torch.empty(N, C, H, W, device=x.device, dtype=torch.float32)
    _lib.call('hk_nhwc_to_nchw', x, y, N, H * W, C, _lib.stream_ptr())
    return y


def conv3x3_pack(w, dgrad):
    """[Cout, Cin, 3, 3] weights -> (w_fwd [9, Cout, Cin], w_dgrad [9, Cin, Cout] with flipped taps, or None unless dgrad)"""
    cout, cin = w.shape[:2]
    wf = torch.empty(9, cout, cin, device=w.device, dtype=torch.float32)
    wd = torch.empty(9, cin, cout, device=w.device, dtype=torch.float32) if dgrad else None
    _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, _lib.stream_ptr())
    return wf, wd


def conv3x3_fwd(x, wf, b, relu, stride=1):
    """padding-1 3x3 conv (+ bias) (+ ReLU) of an NHWC map with packed weights -> NHWC [N, H/stride, W/stride, Cout]"""
    N, H, W, cin = x.shape
    cout = wf.shape[1]
    y = torch.empty(N, H // stride, W // stride, cout, device=x.device, dtype=torch.float32)
    _lib.call('hk_conv3x3_fwd' if stride == 1 else 'hk_conv3x3_s2_fwd', x, wf, b, y, N, H, W, cin, cout, int(relu),
              _lib.stream_ptr())
    return y


def conv3x3_wgrad(x, g, dw, db=None, accumulate=False):
    """dw [Cout, Cin, 3, 3] (and db [Cout]) of a stride-1 3x3 conv from its NHWC input and the (ReLU-masked) NHWC output
    gradient, written or, with ``accumulate``, added onto"""
    N, H, W, cin = x.shape
    cout = g.shape[-1]
    ws = _ws(_lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout), x.device)
    _lib.call('hk_conv3x3_wgrad_acc', x, g, dw, db, N, H, W, cin, cout, ws, ws.numel(), int(accumulate), _lib.stream_ptr())


def conv3x3_dgrad(g, wd, mask=None):
    """input gradient of a stride-1 3x3 conv from the NHWC output gradient and the packed w_dgrad, times (mask > 0) if given"""
    N, H, W, cout = g.shape
    cin = wd.shape[1]
    dx = torch.empty(N, H, W, cin, device=g.device, dtype=torch.float32)
    _lib.call('hk_conv3x3_dgrad', g, wd, mask, dx, N, H, W, cin, cout, _lib.stream_ptr())
    return dx


# ----------------------------------------------------------------------------------------------------------
# layers the methods share: in-place add, image crops, means, ReLU
# ----------------------------------------------------------------------------------------------------------
def add_(a, b):
    """a += b (contiguous fp32 tensors of one size) -> a"""
    _lib.call('hk_add_inplace', a, b, a.numel(), _lib.stream_ptr())
    return a


def crop(images, boxes, size, pad):
    """Bilinear (align_corners=True) crops without a gradient: images NCHW [B, C, H, W], boxes int32 [B, T, 4] as (y0, x0,
    y1, x1), end exclusive, in the image zero-padded by ``pad`` on every side -> NCHW [B*T, C, size, size]."""
    _check_cuda(images, boxes)
    images = _f32c(images.detach())
    B, C, H, W = images.shape
    T = boxes.shape[1]
    out = torch.empty(B * T, C, size, size, device=images.device, dtype=torch.float32)
    _lib.call('hk_nts_crop', images, boxes.contiguous(), out, B, T, C, H, W, pad, size, _lib.stream_ptr())
    return out


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


class NHWCMeanFn(Function):
    """NHWC [N, H, W, C] -> [N, C] spatial mean (AP-CNN's global-pooling branch, MGE-CNN's pooled layer4)."""

    @staticmethod
    def forward(ctx, x):
        _check_cuda(x)
        x = _f32c(x)
        N, H, W, C = x.shape
        y = torch.empty(N, C, device=x.device, dtype=torch.float32)
        ws = _ws(_lib.query('hk_apcnn_pool_workspace_bytes', N, H * W, C), x.device)
        _lib.call('hk_apcnn_pool', x, y, N, H * W, C, 1.0 / (H * W), ws, ws.numel(), _lib.stream_ptr())
        ctx.shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        N, H, W, C = ctx.shape
        dx = torch.empty(N, H, W, C, device=dy.device, dtype=torch.float32)
        _lib.call('hk_apcnn_bcast', None, _f32c(dy), dx, N, H * W, C, 1.0 / (H * W), _lib.stream_ptr())
        return dx


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


# ----------------------------------------------------------------------------------------------------------
# BCNN bilinear pooling (reference model/methods/BCNN.py:8-27)
# ----------------------------------------------------------------------------------------------------------
class BilinearPoolFn(Function):
    @staticmethod
    def forward(ctx, x):
        _check_cuda(x)
        x = _f32c(x)
        B, C, H, W = x.shape
        hw = H * W
        y = torch.empty(B, C * C, device=x.device, dtype=torch.float32)
        ws = _ws(_lib.query('hk_bilinear_pool_fwd_workspace_bytes', B, C, hw), x.device)
        _lib.call('hk_bilinear_pool_fwd', x, y, None, B, C, hw, ws, ws.numel(), _lib.stream_ptr())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        B, C, H, W = x.shape
        hw = H * W
        dy = _f32c(dy)
        dx = torch.empty_like(x)
        ws = _ws(_lib.query('hk_bilinear_pool_bwd_workspace_bytes', B, C, hw), x.device)
        _lib.call('hk_bilinear_pool_bwd', x, dy, dx, B, C, hw, ws, ws.numel(), _lib.stream_ptr())
        return dx


def bilinear_pool(x):
    return BilinearPoolFn.apply(x)


# ----------------------------------------------------------------------------------------------------------
# nn.Linear as skinny tensor-core GEMMs (BCNN.py:42)
# ----------------------------------------------------------------------------------------------------------
class LinearFn(Function):
    @staticmethod
    def forward(ctx, x, w, b):
        _check_cuda(x, w, b)
        x, w = _f32c(x), _f32c(w)
        y = linear_fwd(x, w, b)
        ctx.save_for_backward(x, w)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = _f32c(dy)
        B, F = x.shape
        N = w.shape[0]
        s = _lib.stream_ptr()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _lib.call('hk_linear_dgrad', dy, w, dx, B, F, N, s)
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            db = torch.empty(N, device=x.device, dtype=torch.float32) if ctx.has_bias else None
            _lib.call('hk_linear_wgrad', dy, x, dw, db, B, F, N, s)
        return dx, dw, db


def linear(x, w, b):
    return LinearFn.apply(x, w, b)


def check_num_classes(n):
    """The classifier's dgrad / wgrad GEMMs take dlogits [B, num_classes] through TMA, whose row pitch must be a multiple
    of 16 bytes: fail at model construction with a clear message instead of in the first backward."""
    if int(n) % 4 != 0:
        raise _lib.HawkeyeLibError(f'num_classes={n}: hawkeye_b200 classifiers need num_classes % 4 == 0 (16-byte TMA row '
                                   'pitch of the logit gradients); pad the label space to the next multiple of 4')


# ----------------------------------------------------------------------------------------------------------
# CrossEntropyLoss(label_smoothing) (train.py:211-212)
# ----------------------------------------------------------------------------------------------------------
class CrossEntropyLSFn(Function):
    @staticmethod
    def forward(ctx, logits, labels, smoothing):
        _check_cuda(logits, labels)
        logits = _f32c(logits)
        labels = labels.contiguous().to(torch.int64)
        B, K = logits.shape
        loss = torch.empty(1, device=logits.device, dtype=torch.float32)
        dlogits = torch.empty_like(logits)
        correct = torch.empty(1, device=logits.device, dtype=torch.int32)
        _lib.call('hk_softmax_ce_ls', logits, labels, loss, dlogits, correct, B, K, float(smoothing), 1.0,
                  _lib.stream_ptr())
        ctx.save_for_backward(dlogits)
        ctx.mark_non_differentiable(correct)
        return loss[0], correct

    @staticmethod
    def backward(ctx, g, _g_correct=None):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None


class CrossEntropyLS(torch.nn.Module):
    """Drop-in for ``torch.nn.CrossEntropyLoss(label_smoothing=...)`` (mean reduction) on the fused kernel."""

    def __init__(self, label_smoothing=0.1):
        super().__init__()
        self.label_smoothing = label_smoothing

    def forward(self, logits, labels):
        loss, correct = CrossEntropyLSFn.apply(logits, labels, self.label_smoothing)
        self.last_correct = correct      # [1] int32 on device: top-1 hits of this batch (same kernel, no extra pass)
        return loss


# ----------------------------------------------------------------------------------------------------------
# VGG-style backbone (reference model/backbone/vgg.py:56-70), whole feature stack as ONE autograd node
# ----------------------------------------------------------------------------------------------------------
def _vgg_layers(cfg):
    """-> [(cout, pool_after)]: one entry per conv, 'M' folded into the conv it follows."""
    layers = []
    for v in cfg:
        if v != 'M':
            layers.append((int(v), False))
        elif layers and not layers[-1][1]:
            layers[-1] = (layers[-1][0], True)
        else:
            raise _lib.HawkeyeLibError('VGG cfg: every max-pool must follow a conv')
    if not layers[-1][1]:
        raise _lib.HawkeyeLibError('VGG cfg must end with a max-pool (reference BCNN keeps the last pool)')
    return layers


class VGGFeaturesFn(Function):
    """x NCHW image -> NCHW feature map.  Internally NHWC; convs are wgmma implicit GEMMs.

    params = (w0, b0, w1, b1, ...) in the reference layout [Cout,Cin,3,3] / [Cout].
    """

    @staticmethod
    def forward(ctx, x, cfg, save, *params):
        _check_cuda(x, *params)
        x = _f32c(x)
        s = _lib.stream_ptr()
        dev = x.device
        N, cin0, H, W = x.shape
        if cin0 != 3:
            raise _lib.HawkeyeLibError('VGG features expect a 3-channel NCHW image')
        layers = _vgg_layers(cfg)
        records = []   # per conv layer, for backward
        cur, C = x, 3
        # conv + ReLU + max-pool in one kernel (the pre-pool map is never written) where a pool follows a conv; the
        # unfused pair stays for the 3xTF32 mode (its passes chain through the full map), for activation capture and
        # for odd map sizes
        fuse_ok = not _lib.get_precise() and CAPTURE is None
        for li, (cout, pool) in enumerate(layers):
            w, b = _f32c(params[2 * li]), params[2 * li + 1]
            rec = dict(inp=cur, H=H, W=W)
            fused = pool and li > 0 and fuse_ok and H % 2 == 0 and W % 2 == 0
            if li == 0:
                y = torch.empty(N, H, W, cout, device=dev, dtype=torch.float32)
                ws0 = _ws(_lib.query('hk_conv3x3_first_fwd_workspace_bytes', N, H, W, cout), dev)
                _lib.call('hk_conv3x3_first_fwd', x, w, b, y, N, H, W, cout, ws0, ws0.numel(), s)
                rec['x27'] = ws0 if save else None
            else:
                wf, rec['wd'] = conv3x3_pack(w, save)
                if not fused:
                    y = conv3x3_fwd(cur, wf, b, relu=True)
            if not fused and CAPTURE is not None:
                CAPTURE.append(('relu', y))
            if pool:
                last = li == len(layers) - 1
                Ho, Wo = H // 2, W // 2
                out = torch.empty((N, cout, Ho, Wo) if last else (N, Ho, Wo, cout), device=dev, dtype=torch.float32)
                # one byte per pooled element (arg-max position + ReLU mask) is all the backward needs
                code = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.uint8) if save else None
                if fused:
                    _lib.call('hk_conv3x3_fwd_pool', cur, wf, b, out, code, N, H, W, C, cout, int(last), s)
                elif save:
                    _lib.call('hk_maxpool2x2_fwd_idx', y, out, code, N, H, W, cout, int(last), s)
                else:
                    _lib.call('hk_maxpool2x2_fwd', y, out, N, H, W, cout, int(last), s)
                if CAPTURE is not None:
                    CAPTURE.append(('pool2', y))
                rec.update(code=code, last=last)
                y, H, W = out, Ho, Wo
            records.append(rec)
            cur, C = y, cout
        ctx.layers, ctx.records, ctx.nparams = layers, (records if save else None), len(params)
        ctx.params = params if save else None    # the nn.Parameters themselves: backward accumulates into their .grad
        return cur

    @staticmethod
    def backward(ctx, dfeat):
        if ctx.records is None:
            return (None, None, None) + (None,) * ctx.nparams
        s = _lib.stream_ptr()
        g = _f32c(dfeat)
        grads = [None] * ctx.nparams
        for li in reversed(range(len(ctx.layers))):
            rec, (cout, pool) = ctx.records[li], ctx.layers[li]
            N, H, W = g.shape[0], rec['H'], rec['W']
            if pool:
                dx = torch.empty(N, H, W, cout, device=g.device, dtype=torch.float32)
                _lib.call('hk_maxpool2x2_bwd_idx', rec['code'], g, dx, N, H, W, cout, int(rec['last']), s)
                g = dx
            # Accumulate straight into the parameters' .grad buffers when they exist (the Trainer keeps them as views of
            # one flat buffer): same semantics as autograd's own accumulation, without the temporaries and the 26 `add`
            # launches.  Otherwise (first backward, .grad is None) return fresh tensors and let autograd install them.
            pw, pb = ctx.params[2 * li], ctx.params[2 * li + 1]
            direct = _grad_ready(pw) and _grad_ready(pb)
            if direct:
                dw, db = pw.grad, pb.grad
            else:
                dw = torch.empty(pw.shape, device=g.device, dtype=torch.float32)
                db = torch.empty(cout, device=g.device, dtype=torch.float32)
                grads[2 * li], grads[2 * li + 1] = dw, db
            if li == 0:
                ws = _ws(_lib.query('hk_conv3x3_first_wgrad_workspace_bytes', N, H, W, cout), g.device)
                _lib.call('hk_conv3x3_first_wgrad_acc', rec['x27'], g, dw, db, N, H, W, cout, ws, ws.numel(), int(direct), s)
            else:
                conv3x3_wgrad(rec['inp'], g, dw, db, accumulate=direct)
                # the input is a ReLU output unless a pool came in between (the pool's code carries that mask)
                g = conv3x3_dgrad(g, rec['wd'], mask=None if ctx.layers[li - 1][1] else rec['inp'])
        ctx.records = ctx.params = None
        return (None, None, None) + tuple(grads)


def vgg_features(x, cfg, params):
    return VGGFeaturesFn.apply(x, tuple(cfg), wants_grad(x, params), *params)


# ----------------------------------------------------------------------------------------------------------
# GEMM with the arguments derived from the operands' shapes (tests)
# ----------------------------------------------------------------------------------------------------------
def gemm_tf32(A, B, a_mn=False, b_mn=False, M=None, N=None, K=None, alpha=1.0, diag=0.0, D=None, beta=0.0,
              alpha_vec=None, beta_vec=None, trans_c=False, relu=False, out=None):
    """Batched C = alpha*A.B + diag*I + beta*D on the wgmma GEMM.  A: [b,M,K] (or [b,K,M] if a_mn),
    B: [b,N,K] (K-major, i.e. C = A.B^T layout) or [b,K,N] if b_mn.  2-D operands are shared across the batch."""
    _check_cuda(A, B)
    A, B = _f32c(A), _f32c(B)
    batch = max(A.shape[0] if A.dim() == 3 else 1, B.shape[0] if B.dim() == 3 else 1)
    a2, b2 = A.shape[-2:], B.shape[-2:]
    M_ = a2[1] if a_mn else a2[0]
    K_ = a2[0] if a_mn else a2[1]
    N_ = b2[1] if b_mn else b2[0]
    M, N, K = M or M_, N or N_, K or K_
    sA = a2[0] * a2[1] if A.dim() == 3 else 0
    sB = b2[0] * b2[1] if B.dim() == 3 else 0
    if out is None:
        out = torch.empty((batch, N, M) if trans_c else (batch, M, N), device=A.device, dtype=torch.float32)
    ldc = out.shape[-1]
    sD = ldd = 0
    if D is not None:
        D = _f32c(D)
        ldd = D.shape[-1] if D.shape[-2] != 1 else 0
        sD = D.shape[-2] * D.shape[-1] if D.dim() == 3 else 0
    gemm(A, a_mn, a2[1], sA, B, b_mn, b2[1], sB, out, ldc, out.shape[-2] * out.shape[-1], M, N, K, batch, alpha, alpha_vec,
         diag, D, ldd, sD, beta, beta_vec, relu, trans_c)
    return out


# ----------------------------------------------------------------------------------------------------------
# CBCNN compact bilinear pooling (reference model/methods/CBCNN.py:38-164)
# ----------------------------------------------------------------------------------------------------------
def count_sketch_hashes(input_dim, output_dim):
    """(h1, s1, h2, s2) int64 numpy arrays, bit-identical to CBCNN.py:76-91 (numpy legacy MT19937, seeds 1/3/5/7;
    ``RandomState(seed)`` is the same stream as ``np.random.seed(seed)`` without clobbering the global RNG)."""
    import numpy as np
    h1 = np.random.RandomState(1).randint(output_dim, size=input_dim)
    s1 = 2 * np.random.RandomState(3).randint(2, size=input_dim) - 1
    h2 = np.random.RandomState(5).randint(output_dim, size=input_dim)
    s2 = 2 * np.random.RandomState(7).randint(2, size=input_dim) - 1
    return h1.astype(np.int64), s1.astype(np.int64), h2.astype(np.int64), s2.astype(np.int64)


class CompactBilinearPoolFn(Function):
    @staticmethod
    def forward(ctx, x, h1, h2, s1, s2, d):
        _check_cuda(x, h1, h2, s1, s2)
        x = _f32c(x)
        B, C, H, W = x.shape
        y = torch.empty(B, d, device=x.device, dtype=torch.float32)
        pre = torch.empty(B, d, device=x.device, dtype=torch.float32)
        _lib.call('hk_cbp_fwd', x, h1, h2, s1, s2, y, pre, B, C, H * W, d, _lib.stream_ptr())
        if CAPTURE is not None:
            CAPTURE.append(('ssqrt', pre))
        ctx.save_for_backward(x, pre, h1, h2, s1, s2)
        ctx.d = d
        return y

    @staticmethod
    def backward(ctx, dy):
        x, pre, h1, h2, s1, s2 = ctx.saved_tensors
        B, C, H, W = x.shape
        d = ctx.d
        dx = torch.empty_like(x)
        ws = _ws(_lib.query('hk_cbp_bwd_workspace_bytes', B, C, d), x.device)
        _lib.call('hk_cbp_bwd', x, pre, _f32c(dy), h1, h2, s1, s2, dx, B, C, H * W, d, ws, ws.numel(),
                  _lib.stream_ptr())
        return dx, None, None, None, None, None


# ----------------------------------------------------------------------------------------------------------
# Fast MPN-COV pooling head (reference model/methods/MPNCOV.py:105-242)
# ----------------------------------------------------------------------------------------------------------
class CovpoolFn(Function):
    """Covpool (MPNCOV.py:105-134): [B,C,H,W] -> [B,C,C]."""

    @staticmethod
    def forward(ctx, x):
        _check_cuda(x)
        x = _f32c(x)
        B, C, H, W = x.shape
        cov = torch.empty(B, C, C, device=x.device, dtype=torch.float32)
        xc = torch.empty(B, C, (H * W + 3) // 4 * 4, device=x.device, dtype=torch.float32)   # centred rows, 16-byte pitch
        _lib.call('hk_covpool_fwd', x, cov, xc, B, C, H * W, _lib.stream_ptr())
        ctx.save_for_backward(xc)
        ctx.shape = x.shape
        return cov

    @staticmethod
    def backward(ctx, g):
        (xc,) = ctx.saved_tensors
        B, C, H, W = ctx.shape
        dx = torch.empty(B, C, H, W, device=g.device, dtype=torch.float32)
        _lib.call('hk_covpool_bwd', xc, _f32c(g), dx, B, C, H * W, _lib.stream_ptr())
        return dx


class SqrtmFn(Function):
    """Sqrtm (MPNCOV.py:137-202): coupled Newton-Schulz forward + the reference's own backward recurrence."""

    @staticmethod
    def forward(ctx, x, iterN):
        _check_cuda(x)
        x = _f32c(x)
        B, n, _ = x.shape
        y = torch.empty_like(x)
        saved = torch.empty(_lib.query('hk_sqrtm_saved_floats', B, n, iterN), device=x.device, dtype=torch.float32)
        ws = _ws(_lib.query('hk_sqrtm_fwd_workspace_bytes', B, n), x.device)
        _lib.call('hk_sqrtm_fwd', x, y, saved, B, n, iterN, ws, ws.numel(), _lib.stream_ptr())
        ctx.save_for_backward(x, y, saved)
        ctx.iterN = iterN
        return y

    @staticmethod
    def backward(ctx, g):
        x, y, saved = ctx.saved_tensors
        B, n, _ = x.shape
        gx = torch.empty_like(x)
        ws = _ws(_lib.query('hk_sqrtm_bwd_workspace_bytes', B, n), x.device)
        _lib.call('hk_sqrtm_bwd', x, y, _f32c(g), saved, gx, B, n, ctx.iterN, ws, ws.numel(), _lib.stream_ptr())
        return gx, None


class TriuvecFn(Function):
    """Triuvec (MPNCOV.py:205-230): [B,n,n] -> [B, n(n+1)/2, 1]."""

    @staticmethod
    def forward(ctx, x):
        _check_cuda(x)
        x = _f32c(x)
        B, n, _ = x.shape
        y = torch.empty(B, n * (n + 1) // 2, 1, device=x.device, dtype=torch.float32)
        _lib.call('hk_triuvec_fwd', x, y, B, n, _lib.stream_ptr())
        ctx.n = n
        return y

    @staticmethod
    def backward(ctx, g):
        B, n = g.shape[0], ctx.n
        dx = torch.empty(B, n, n, device=g.device, dtype=torch.float32)
        _lib.call('hk_triuvec_bwd', _f32c(g), dx, B, n, _lib.stream_ptr())
        return dx


def CovpoolLayer(var):
    return CovpoolFn.apply(var)


def SqrtmLayer(var, iterN):
    return SqrtmFn.apply(var, iterN)


def TriuvecLayer(var):
    return TriuvecFn.apply(var)
