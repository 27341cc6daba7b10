"""Autograd bindings of CrossX (reference model/methods/CrossX.py, model/loss/CrossX_loss.py) on the hk_crossx_* kernels.

An excitation block (the last bottleneck of layer3 and of layer4) runs as two nodes around its gate MLPs:
``MEConvFn`` (conv1 .. bn3 on the ResNet units, no residual, no ReLU: ``c``, its spatial mean ``z`` and the residual)
and ``MEFn`` (the main output relu(c + r) and the P parts relu(c g_p + r), hk_crossx_me_*).  The backward of ``MEConvFn``
receives dc, dz and dr together: the squeeze's gradient dz / HW is added to dc in one more pass over it, and dr
goes into conv1's data-gradient GEMM epilogue, so neither takes an extra autograd sum.

Part maps are [N, H, W, P, C].  ``UltiFn`` applies each conv2_p (1x1, 2048 -> 1024) to its slice of the layer4 parts and
takes the parts' spatial means as [N, P, 2048]; ``FuseFn`` adds the upsampled conv2 outputs to the layer3 parts and takes
their global max as [N, P, 1024].
"""
import torch
from torch.autograd import Function

from . import _lib, ops as _ops
from .ops import _check_cuda, _f32c, _ws, gemm, nhwc_channel_sum


class MEConvFn(Function):
    """NHWC x through conv1/bn1/relu, conv2/bn2/relu, conv3/bn3 of a bottleneck without downsample -> (c, mean_hw c [N, C],
    the residual x).  ``units`` = (u1, u2, u3) with u3 built without ReLU."""

    @staticmethod
    def forward(ctx, x, units, save, training, *params):
        _check_cuda(x)
        x = _f32c(x)
        recs, cur = [], x
        for i, u in enumerate(units):
            w, g, b = params[3 * i:3 * i + 3]
            cur, r = u.forward(cur, _f32c(w), g, b, None, save, training)
            recs.append(r)
        N, H, W, C = cur.shape
        z = nhwc_channel_sum(cur, N, H * W, C, 1.0 / (H * W))
        ctx.units, ctx.recs, ctx.shape = units, (recs if save else None), cur.shape
        return cur, z, x

    @staticmethod
    def backward(ctx, dc, dz, dr):
        if ctx.recs is None:
            return (None,) * (4 + 9)
        N, H, W, C = ctx.shape
        dev = ctx.recs[0]['w'].device
        if dz is not None:   # dc + dz / HW at every pixel: one read of dc and one write
            g = torch.empty(ctx.shape, device=dev, dtype=torch.float32)
            _lib.call('hk_apcnn_bcast', None if dc is None else _f32c(dc), _f32c(dz), g, N, H * W, C, 1.0 / (H * W),
                      _lib.stream_ptr())
            dc = g
        dc = _f32c(dc) if dc is not None else torch.zeros(ctx.shape, device=dev, dtype=torch.float32)
        u1, u2, u3 = ctx.units
        r1, r2, r3 = ctx.recs
        d2, _, dw3, dg3, db3 = u3.backward(r3, dc)
        d1, _, dw2, dg2, db2 = u2.backward(r2, d2)
        dx, _, dw1, dg1, db1 = u1.backward(r1, d1, addend=None if dr is None else _f32c(dr))
        ctx.recs = None
        return (dx, None, None, None, dw1, dg1, db1, dw2, dg2, db2, dw3, dg3, db3)


class MEFn(Function):
    """(c, r [N, H, W, C], gate logits m [N, P, C]) -> (relu(c + r), parts [N, H, W, P, C]), or the parts alone when
    ``main`` is False (layer4's main output is discarded by the reference)."""

    @staticmethod
    def forward(ctx, c, r, m, main):
        _check_cuda(c, r, m)
        c, r, m = _f32c(c), _f32c(r), _f32c(m)
        N, H, W, C = c.shape
        P = m.shape[1]
        out = torch.empty_like(c) if main else None
        parts = torch.empty(N, H, W, P, C, device=c.device, dtype=torch.float32)
        _lib.call('hk_crossx_me_fwd', c, r, m, out, parts, N, H * W, P, C, _lib.stream_ptr())
        ctx.save_for_backward(c, r, m)
        ctx.main = main
        return (out, parts) if main else parts

    @staticmethod
    def backward(ctx, *grads):
        c, r, m = ctx.saved_tensors
        dout, dparts = grads if ctx.main else (None, grads[0])
        N, H, W, C = c.shape
        P = m.shape[1]
        dc, dr, dm = torch.empty_like(c), torch.empty_like(r), torch.empty_like(m)
        ws = _ws(_lib.query('hk_crossx_me_bwd_workspace_bytes', N, H * W, P, C), c.device)
        _lib.call('hk_crossx_me_bwd', c, r, m, None if dout is None else _f32c(dout), _f32c(dparts), dc, dr, dm, N, H * W,
                  P, C, ws, ws.numel(), _lib.stream_ptr())
        return dc, dr, dm, None


def excite(x, units, mlps, main, training):
    """One excitation block on NHWC x: ``units`` (u1, u2, u3) and ``mlps`` the P ``nn.Sequential(Linear, ReLU, Linear,
    Sigmoid)`` of its MELayer -> (relu(c + r), parts) or the parts alone (``main`` False)."""
    params = [p for u in units for p in u.params()]
    c, z, r = MEConvFn.apply(x, units, _ops.wants_grad(x, params), training, *params)
    gates = [_ops.linear(_ops.ActFn.apply(_ops.linear(z, q[0].weight, q[0].bias), False), q[2].weight, q[2].bias)
             for q in mlps]
    return MEFn.apply(c, r, torch.stack(gates, 1), main)


class UltiFn(Function):
    """layer4 parts [N, h, w, P, C4] and the conv2 weights [C3, C4, 1, 1] of each part -> (the parts' spatial means
    [N, P, C4], conv2_p(part p) [N, h, w, C3] for each p).  The 1x1 convolutions read their slice of the parts in place
    (row stride P C4)."""

    @staticmethod
    def forward(ctx, parts, *wts):
        _check_cuda(parts, *wts)
        parts = _f32c(parts)
        N, h, w, P, C4 = parts.shape
        rows = N * h * w
        mean = torch.empty(N, P, C4, device=parts.device, dtype=torch.float32)
        ws = _ws(_lib.query('hk_apcnn_pool_workspace_bytes', N, h * w, P * C4), parts.device)
        _lib.call('hk_apcnn_pool', parts, mean, N, h * w, P * C4, 1.0 / (h * w), ws, ws.numel(), _lib.stream_ptr())
        outs = []
        wts = [_f32c(wt) for wt in wts]
        for p, wt in enumerate(wts):
            C3 = wt.shape[0]
            y = torch.empty(N, h, w, C3, device=parts.device, dtype=torch.float32)
            gemm(parts[..., p, :], 0, P * C4, 0, wt, 0, C4, 0, y, C3, 0, rows, C3, C4)
            outs.append(y)
        ctx.save_for_backward(parts, *wts)
        return (mean,) + tuple(outs)

    @staticmethod
    def backward(ctx, dmean, *douts):
        parts, *wts = ctx.saved_tensors
        N, h, w, P, C4 = parts.shape
        rows = N * h * w
        dconv = torch.empty_like(parts)                 # the 1x1 convolutions' share of dparts
        dws = []
        for p, (wt, dy) in enumerate(zip(wts, douts)):
            if dy is None:
                dconv[..., p, :].zero_()
                dws.append(None)
                continue
            dy = _f32c(dy)
            C3 = wt.shape[0]
            gemm(dy, 0, C3, 0, wt, 1, C4, 0, dconv[..., p, :], P * C4, 0, rows, C4, C3)          # dX = dY W
            dw = torch.empty_like(wt)
            gemm(dy, 1, C3, 0, parts[..., p, :], 1, P * C4, 0, dw, C4, 0, C3, C4, rows)          # dW = dY^T X
            dws.append(dw)
        if dmean is None:
            return (dconv,) + tuple(dws)
        dparts = torch.empty_like(parts)                # + dmean / hw at every pixel
        _lib.call('hk_apcnn_bcast', dconv, _f32c(dmean), dparts, N, h * w, P * C4, 1.0 / (h * w), _lib.stream_ptr())
        return (dparts,) + tuple(dws)


class FuseFn(Function):
    """layer3 parts [N, H, W, P, C] and R_p [N, H/2, W/2, C] -> (global max of each part [N, P, C], S_p = part_p +
    nearest-2x(R_p) for each p)."""

    @staticmethod
    def forward(ctx, parts, *Rs):
        _check_cuda(parts, *Rs)
        parts = _f32c(parts)
        N, H, W, P, C = parts.shape
        pmax = torch.empty(N, P, C, device=parts.device, dtype=torch.float32)
        pidx = torch.empty(N, P, C, device=parts.device, dtype=torch.int32)
        s = _lib.stream_ptr()
        Ss = []
        for p, R in enumerate(Rs):
            S = torch.empty(N, H, W, C, device=parts.device, dtype=torch.float32)
            _lib.call('hk_crossx_fuse_fwd', parts, _f32c(R), S, pmax, pidx, N, H, W, P, C, p, s)
            Ss.append(S)
        ctx.save_for_backward(pidx)
        ctx.shape = parts.shape
        return (pmax,) + tuple(Ss)

    @staticmethod
    def backward(ctx, dmax, *dSs):
        (pidx,) = ctx.saved_tensors
        N, H, W, P, C = ctx.shape
        s = _lib.stream_ptr()
        dmax = torch.zeros(N, P, C, device=pidx.device, dtype=torch.float32) if dmax is None else _f32c(dmax)
        dparts = torch.empty(ctx.shape, device=pidx.device, dtype=torch.float32)
        dRs = []
        for p, dS in enumerate(dSs):
            dS = _f32c(dS) if dS is not None else torch.zeros(N, H, W, C, device=pidx.device, dtype=torch.float32)
            dR = torch.empty(N, H // 2, W // 2, C, device=pidx.device, dtype=torch.float32)
            _lib.call('hk_crossx_fuse_bwd', dS, dmax, pidx, dparts, dR, N, H, W, P, C, p, s)
            dRs.append(dR)
        return (dparts,) + tuple(dRs)


def reg_sums(fu, fp, fc):
    """Features [N, P, Cu], [N, P, Cp], [N, P, Cp] -> s: the batch sums of their L2-normalised rows, (s_u, s_p, s_c)
    concatenated into one buffer [P (Cu + 2 Cp)]."""
    N, P, Cu = fu.shape
    Cp = fp.shape[2]
    s = torch.empty(P * (Cu + 2 * Cp), device=fu.device, dtype=torch.float32)
    _lib.call('hk_crossx_reg_sums', fu, fp, fc, s, N, P, Cu, Cp, _lib.stream_ptr())
    return s


class CrossXLossFn(Function):
    """(xf, xp, xc, fu, fp, fc, labels) -> (loss, top-1 count) on hk_crossx_reg_sums + hk_crossx_loss; ``reduce_s``
    (optional) sums s over the ranks in place between the two launches, ``world`` ranks of equal batches."""

    @staticmethod
    def forward(ctx, xf, xp, xc, fu, fp, fc, labels, smoothing, gammas, world, reduce_s):
        _check_cuda(xf, xp, xc, fu, fp, fc, labels)
        xf, xp, xc, fu, fp, fc = (_f32c(t) for t in (xf, xp, xc, fu, fp, fc))
        labels = labels.contiguous().to(torch.int64)
        N, K = xf.shape
        _, P, Cu = fu.shape
        Cp = fp.shape[2]
        s = reg_sums(fu, fp, fc)
        if reduce_s is not None:
            reduce_s(s)
        loss = torch.empty(1, device=xf.device, dtype=torch.float32)
        correct = torch.empty(1, device=xf.device, dtype=torch.int32)
        grads = [torch.empty_like(t) for t in (xf, xp, xc, fu, fp, fc)]
        _lib.call('hk_crossx_loss', xf, xp, xc, labels, fu, fp, fc, s, loss, *grads, correct, N, K, P, Cu, Cp,
                  float(smoothing), *(float(g) for g in gammas), N * world, float(world), _lib.stream_ptr())
        ctx.save_for_backward(*grads)
        ctx.mark_non_differentiable(correct)
        return loss[0], correct

    @staticmethod
    def backward(ctx, g, _g_correct=None):
        return tuple(d * g for d in ctx.saved_tensors) + (None,) * 5
