"""torch.autograd bindings of the C-ABI kernels (host plumbing only: memory, streams, autograd edges).

Every op here calls ``libhawkeye_b200.so`` through ``_lib.call``; there is no PyTorch-eager fallback.
PyTorch owns all device buffers (caching allocator) incl. workspaces and saved-for-backward tensors.
"""
import os

import torch
from torch.autograd import Function

from . import _lib

VGG16_D = (64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M')

# Parity tests only: when set to a list, forward passes append the decisions they took at the non-smooth points of the
# path, in execution order — ('relu', y NHWC) after every ReLU, ('pool2', x NHWC) before every 2x2 max-pool,
# ('pool3', argmax u8 NHWC, input shape) for the ResNet stem pool, ('ssqrt', bins) for CBCNN's signed square root —
# so that a CPU oracle can be evaluated on the same branch of the piecewise-smooth function (oracle.hop_oracle.MaskTape).
CAPTURE = None

# Backbone weight/bias gradients are accumulated by the wgrad kernels directly into an existing ``param.grad`` (see
# VGGFeaturesFn.backward).  Set to False to make every backward return fresh gradient tensors to autograd instead.
ACCUMULATE_INTO_GRAD = True
# conv3x3 + ReLU + MaxPool2d(2,2) as one kernel (hk_conv3x3_fwd_pool) wherever VGG has a pool after a conv
FUSE_CONV_POOL = os.environ.get('HK_FUSE_CONV_POOL', '1') != '0'


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
        B, F = x.shape
        N = w.shape[0]
        y = torch.empty(B, N, device=x.device, dtype=torch.float32)
        ws = _ws(_lib.query('hk_linear_fwd_workspace_bytes', B, F, N), x.device)
        _lib.call('hk_linear_fwd', x, w, b, y, B, F, N, ws, ws.numel(), _lib.stream_ptr())
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
def _vgg_plan(cfg):
    """-> list of ('conv', cout) / ('pool',) entries."""
    return [('pool',) if v == 'M' else ('conv', int(v)) for v in cfg]


class VGGFeaturesFn(Function):
    """x NCHW image -> NCHW feature map.  Internally NHWC; convs are wgmma implicit GEMMs.

    params = (w0, b0, w1, b1, ...) in the reference layout [Cout,Cin,3,3] / [Cout].
    """

    @staticmethod
    def forward(ctx, x, cfg, train_backbone, *params):
        _check_cuda(x, *params)
        x = _f32c(x)
        s = _lib.stream_ptr()
        dev = x.device
        N, cin0, H, W = x.shape
        if cin0 != 3:
            raise _lib.HawkeyeLibError('VGG features expect a 3-channel NCHW image')
        plan = _vgg_plan(cfg)
        if plan[-1][0] != 'pool':
            raise _lib.HawkeyeLibError('VGG cfg must end with a max-pool (reference BCNN keeps the last pool)')
        save = bool(train_backbone)   # decided by the caller: grad mode is always off inside Function.forward
        records = []   # per layer: dict for backward
        cur, C, li = None, 3, 0
        # conv + ReLU + max-pool in one kernel (the pre-pool map is never written) whenever a pool follows a conv; the
        # unfused pair stays for the 3xTF32 mode (its passes chain through the full map) and for activation capture
        fuse_pool = FUSE_CONV_POOL and not _lib.get_precise() and CAPTURE is None
        skip_pool = False
        for idx, ent in enumerate(plan):
            if ent[0] == 'conv':
                cout = ent[1]
                w, b = _f32c(params[2 * li]), params[2 * li + 1]
                fused = fuse_pool and li > 0 and idx + 1 < len(plan) and plan[idx + 1][0] == 'pool' and H % 2 == 0 and W % 2 == 0
                y = None if fused else torch.empty(N, H, W, cout, device=dev, dtype=torch.float32)
                if li == 0:
                    ws0 = _ws(_lib.query('hk_conv3x3_first_fwd_workspace_bytes', N, H, W, cout), dev)
                    _lib.call('hk_conv3x3_first_fwd', x, w, b, y, N, H, W, cout, ws0, ws0.numel(), s)
                    rec = dict(kind='conv0', inp=None, out=y, H=H, W=W, cin=3, cout=cout, x27=ws0 if save else None)
                else:
                    wf = torch.empty(9 * cout * C, device=dev, dtype=torch.float32)
                    wd = torch.empty(9 * cout * C, device=dev, dtype=torch.float32) if save else None
                    _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, C, s)
                    rec = dict(kind='conv', inp=cur, out=y, wd=wd, H=H, W=W, cin=C, cout=cout,
                               inp_is_relu=(records[-1]['kind'] != 'pool'))
                    if fused:
                        last = idx + 1 == len(plan) - 1
                        Ho, Wo = H // 2, W // 2
                        out = torch.empty((N, cout, Ho, Wo) if last else (N, Ho, Wo, cout), device=dev, dtype=torch.float32)
                        code = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.uint8) if save else None
                        _lib.call('hk_conv3x3_fwd_pool', cur, wf, b, out, code, N, H, W, C, cout, 1 if last else 0, s)
                        records.append(rec)
                        records.append(dict(kind='pool', code=code, H=H, W=W, C=cout, last=last))
                        cur, C, H, W = out, cout, Ho, Wo
                        li += 1
                        skip_pool = True
                        continue
                    _lib.call('hk_conv3x3_fwd', cur, wf, b, y, N, H, W, C, cout, 1, s)
                records.append(rec)
                if CAPTURE is not None:
                    CAPTURE.append(('relu', y))
                cur, C = y, cout
                li += 1
            else:
                if skip_pool:       # already done by the conv before it
                    skip_pool = False
                    continue
                last = idx == len(plan) - 1
                Ho, Wo = H // 2, W // 2
                out = torch.empty((N, C, Ho, Wo) if last else (N, Ho, Wo, C), device=dev, dtype=torch.float32)
                code = None
                if save:     # one byte per pooled element (arg-max position + ReLU mask) is all the backward needs
                    code = torch.empty(N, Ho, Wo, C, device=dev, dtype=torch.uint8)
                    _lib.call('hk_maxpool2x2_fwd_idx', cur, out, code, N, H, W, C, 1 if last else 0, s)
                else:
                    _lib.call('hk_maxpool2x2_fwd', cur, out, N, H, W, C, 1 if last else 0, s)
                if CAPTURE is not None:
                    CAPTURE.append(('pool2', cur))
                records.append(dict(kind='pool', code=code, H=H, W=W, C=C, last=last))
                cur, H, W = out, Ho, Wo
        if save:
            ctx.records = records
            ctx.x = x
            ctx.N = N
            ctx.params = params      # the nn.Parameters themselves: backward accumulates into their .grad when it can
        else:
            ctx.records = None
        ctx.nparams = len(params)
        return cur

    @staticmethod
    def backward(ctx, dfeat):
        if ctx.records is None:
            return (None, None, None) + (None,) * ctx.nparams
        s = _lib.stream_ptr()
        N = ctx.N
        dev = dfeat.device
        g = _f32c(dfeat)
        grads = [None] * ctx.nparams
        li = ctx.nparams // 2
        for rec in reversed(ctx.records):
            if rec['kind'] == 'pool':
                dx = torch.empty(N, rec['H'], rec['W'], rec['C'], device=dev, dtype=torch.float32)
                _lib.call('hk_maxpool2x2_bwd_idx', rec['code'], g, dx, N, rec['H'], rec['W'], rec['C'],
                          1 if rec['last'] else 0, s)
                rec['code'] = None
                g = dx
                continue
            li -= 1
            H, W, cin, cout = rec['H'], rec['W'], rec['cin'], rec['cout']
            # Accumulate straight into the parameters' .grad buffers when they exist (the Trainer keeps them as views of
            # one flat buffer): same semantics as autograd's own accumulation, without the temporaries and the 26 `add`
            # launches.  Otherwise (first backward, .grad is None) return fresh tensors and let autograd install them.
            pw, pb = ctx.params[2 * li], ctx.params[2 * li + 1]
            direct = ACCUMULATE_INTO_GRAD and _grad_ready(pw) and _grad_ready(pb)
            if direct:
                dw, db, acc = pw.grad, pb.grad, 1
            else:
                dw = torch.empty(cout, cin, 3, 3, device=dev, dtype=torch.float32)
                db = torch.empty(cout, device=dev, dtype=torch.float32)
                acc = 0
            if rec['kind'] == 'conv0':
                ws = _ws(_lib.query('hk_conv3x3_first_wgrad_workspace_bytes', N, H, W, cout), dev)
                _lib.call('hk_conv3x3_first_wgrad_acc', rec['x27'], g, dw, db, N, H, W, cout, ws, ws.numel(), acc, s)
            else:
                ws = _ws(_lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout), dev)
                _lib.call('hk_conv3x3_wgrad_acc', rec['inp'], g, dw, db, N, H, W, cin, cout, ws, ws.numel(), acc, s)
                dx = torch.empty_like(rec['inp'])
                mask = rec['inp'] if rec['inp_is_relu'] else None
                _lib.call('hk_conv3x3_dgrad', g, rec['wd'], mask, dx, N, H, W, cin, cout, s)
                g = dx
            if not direct:
                grads[2 * li], grads[2 * li + 1] = dw, db
            rec['out'] = None
        ctx.records = None
        ctx.params = None
        return (None, None, None) + tuple(grads)


def vgg_features(x, cfg, params, train_backbone=True):
    """``train_backbone`` is kept for call compatibility; whether activations are saved for backward is decided from what
    actually requires grad at call time (so freezing / unfreezing the backbone after construction just works)."""
    save = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
    return VGGFeaturesFn.apply(x, tuple(cfg), save, *params)


# ----------------------------------------------------------------------------------------------------------
# raw helpers used by tests / other heads
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
    _lib.call('hk_gemm_tf32', A, int(a_mn), a2[1], sA, B, int(b_mn), b2[1], sB, out, ldc, out.shape[-2] * out.shape[-1],
              int(trans_c), M, N, K, batch, float(alpha), alpha_vec, float(diag), D, ldd, sD, float(beta), beta_vec,
              int(relu), _lib.stream_ptr())
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
