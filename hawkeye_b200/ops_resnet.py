"""ResNet-50 v1.5 trunk (reference model/backbone/resnet.py:89-252) and the MPN-COV dimension-reduction block
(MPNCOV.py:64-69) as explicit forward/backward pipelines over the C-ABI kernels.  NHWC fp32 inside.

conv unit = convolution (wgmma GEMM / implicit GEMM) -> train-mode BatchNorm (+ residual) (+ ReLU).
"""
import torch
from torch.autograd import Function

from . import _lib, ops as _ops
from .ops import _check_cuda, _f32c, _ws

BN_EPS = 1e-5


def _gemm(A, a_mn, lda, B, b_mn, ldb, C, ldc, M, N, K, relu=0, D=None):
    """C = A.B (+ D, same layout as C: the residual-gradient add rides in the GEMM epilogue instead of a separate pass)"""
    _lib.call('hk_gemm_tf32', A, int(a_mn), lda, 0, B, int(b_mn), ldb, 0, C, ldc, 0, 0, M, N, K, 1, 1.0, None, 0.0, D,
              ldc if D is not None else 0, 0, 1.0 if D is not None else 0.0, None, relu, _lib.stream_ptr())


class Unit:
    """One conv + BN (+residual) (+ReLU).  kind in {'stem','1x1','1x1s2','3x3','3x3s2'}."""

    def __init__(self, kind, conv, bn, relu):
        self.kind, self.conv, self.bn, self.relu = kind, conv, bn, relu

    def params(self):
        return [self.conv.weight, self.bn.weight, self.bn.bias]

    # ---- forward: x NHWC [N,H,W,Cin] (stem: NCHW image) -> y NHWC
    def forward(self, x, w, gamma, beta, residual, save, training=True):
        s = _lib.stream_ptr()
        dev = x.device
        rec = {}
        cout = w.shape[0]
        if self.kind == 'stem':
            N, _, H, W = x.shape
            Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
            P = N * Ho * Wo
            x147 = torch.empty(P, 160, device=dev, dtype=torch.float32)
            w147 = torch.empty(cout, 160, device=dev, dtype=torch.float32)
            _lib.call('hk_stem_im2col', x, x147, N, H, W, s)
            _lib.call('hk_pack_stem_weights', w, w147, cout, s)
            c = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.float32)
            _gemm(x147, 0, 160, w147, 0, 160, c, cout, P, cout, 160)
            rec['xin'] = x147
        else:
            N, H, W, cin = x.shape
            if self.kind in ('1x1', '1x1s2'):
                xin = x
                if self.kind == '1x1s2':
                    xin = torch.empty(N, (H + 1) // 2, (W + 1) // 2, cin, device=dev, dtype=torch.float32)
                    _lib.call('hk_subsample2', x, xin, N, H, W, cin, s)
                    rec['full_hw'] = (H, W)
                Ho, Wo = xin.shape[1], xin.shape[2]
                P = N * Ho * Wo
                c = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.float32)
                _gemm(xin, 0, cin, w, 0, cin, c, cout, P, cout, cin)
                rec['xin'] = xin
            else:
                wf = torch.empty(9 * cout * cin, device=dev, dtype=torch.float32)
                wd = torch.empty(9 * cout * cin, device=dev, dtype=torch.float32) if save else None
                _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, s)
                if self.kind == '3x3':
                    Ho, Wo = H, W
                    c = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.float32)
                    _lib.call('hk_conv3x3_fwd', x, wf, None, c, N, H, W, cin, cout, 0, s)
                else:
                    Ho, Wo = H // 2, W // 2
                    c = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.float32)
                    _lib.call('hk_conv3x3_s2_fwd', x, wf, None, c, N, H, W, cin, cout, 0, s)
                    rec['full_hw'] = (H, W)
                rec['xin'], rec['wd'] = x, wd
            P = N * Ho * Wo
        y = torch.empty_like(c)
        bn = self.bn
        if training:
            mean = torch.empty(cout, device=dev, dtype=torch.float32)
            invstd = torch.empty(cout, device=dev, dtype=torch.float32)
            ws = _ws(_lib.query('hk_bn_workspace_bytes', P, cout), dev)
            _lib.call('hk_bn_fwd', c, gamma, beta, residual, y, mean, invstd, bn.running_mean, bn.running_var,
                      float(bn.momentum), float(bn.eps), P, cout, int(self.relu), ws, ws.numel(), s)
            bn.num_batches_tracked += 1
        else:
            mean = bn.running_mean
            invstd = torch.rsqrt(bn.running_var + bn.eps)
            _lib.call('hk_bn_apply', c, mean, invstd, gamma, beta, residual, y, P, cout, int(self.relu), s)
        if _ops.CAPTURE is not None and self.relu:
            _ops.CAPTURE.append(('relu', y))
        if save:
            rec.update(c=c, y=y if self.relu else None, mean=mean, invstd=invstd, P=P, cout=cout, w=w, gamma=gamma, beta=beta,
                       shape=(N, Ho, Wo), has_res=residual is not None)
            return y, rec
        return y, None

    # ---- backward: dy NHWC -> (dx NHWC or None, dres or None, dw, dgamma, dbeta)
    def backward(self, rec, dy, need_dx=True, addend=None):
        """addend (optional, same shape as dx): added to dx — inside the dgrad GEMM's epilogue for 1x1 convs"""
        s = _lib.stream_ptr()
        dev = dy.device
        P, cout = rec['P'], rec['cout']
        N, Ho, Wo = rec['shape']
        dc = torch.empty(N, Ho, Wo, cout, device=dev, dtype=torch.float32)
        dres = torch.empty_like(dc) if rec['has_res'] else None
        dgamma = torch.empty(cout, device=dev, dtype=torch.float32)
        dbeta = torch.empty(cout, device=dev, dtype=torch.float32)
        ws = _ws(_lib.query('hk_bn_workspace_bytes', P, cout), dev)
        # BN + ReLU without a residual: the mask is recomputed from x (hk_bn_bwd_ex), y is not read
        mask_beta = rec['beta'] if (self.relu and not rec['has_res'] and rec.get('train_stats', True)) else None
        _lib.call('hk_bn_bwd_ex', rec['c'], rec['y'], dy, rec['gamma'], mask_beta, rec['mean'], rec['invstd'], dc, dres,
                  dgamma, dbeta, P, cout, int(self.relu), ws, ws.numel(), s)
        w, xin = rec['w'], rec['xin']
        dx = None
        if self.kind == 'stem':
            dwm = torch.empty(cout, 160, device=dev, dtype=torch.float32)
            wsb = _ws(_lib.query('hk_matconv_wgrad_workspace_bytes', P, 160, cout), dev)
            _lib.call('hk_matconv_wgrad', xin, dc, dwm, P, 160, cout, wsb, wsb.numel(), s)
            dw = dwm[:, :147].reshape(w.shape).contiguous()
        elif self.kind in ('1x1', '1x1s2'):
            cin = xin.shape[-1]
            dw = torch.empty(cout, cin, 1, 1, device=dev, dtype=torch.float32)
            wsb = _ws(_lib.query('hk_matconv_wgrad_workspace_bytes', P, cin, cout), dev)
            _lib.call('hk_matconv_wgrad', xin, dc, dw, P, cin, cout, wsb, wsb.numel(), s)
            if need_dx:
                dxs = torch.empty_like(xin)
                fused = addend if (addend is not None and self.kind == '1x1') else None
                _gemm(dc, 0, cout, w, 1, cin, dxs, cin, P, cin, cout, D=fused)   # dX = dC . W (+ addend)  (W [Cout,Cin] as the MN-major B)
                if fused is not None:
                    addend = None
                if self.kind == '1x1s2':
                    H, W = rec['full_hw']
                    dx = torch.empty(N, H, W, cin, device=dev, dtype=torch.float32)
                    _lib.call('hk_upsample2_zero', dxs, dx, N, H, W, cin, s)
                else:
                    dx = dxs
        else:
            cin = xin.shape[-1]
            H, W = (Ho, Wo) if self.kind == '3x3' else rec['full_hw']
            g = dc
            if self.kind == '3x3s2':                    # adjoint of the stride: zero-insert dC to the input resolution
                g = torch.empty(N, H, W, cout, device=dev, dtype=torch.float32)
                _lib.call('hk_upsample2_zero', dc, g, N, H, W, cout, s)
            dw = torch.empty(cout, cin, 3, 3, device=dev, dtype=torch.float32)
            wsb = _ws(_lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout), dev)
            _lib.call('hk_conv3x3_wgrad', xin, g, dw, None, N, H, W, cin, cout, wsb, wsb.numel(), s)
            if need_dx:
                dx = torch.empty(N, H, W, cin, device=dev, dtype=torch.float32)
                _lib.call('hk_conv3x3_dgrad', g, rec['wd'], None, dx, N, H, W, cin, cout, s)
        if addend is not None and dx is not None:
            dx = _add(dx, addend)
        return dx, dres, dw, dgamma, dbeta


def _add(a, b):
    _lib.call('hk_add_inplace', a, b, a.numel(), _lib.stream_ptr())
    return a


class TrunkPlan:
    """Flattened description of a ResNet trunk module: stem unit, max-pool, list of bottleneck blocks."""

    def __init__(self, trunk):
        self.stem = Unit('stem', trunk[0], trunk[1], True)
        self.blocks = []
        for layer in list(trunk)[4:]:
            for blk in layer:
                s2 = blk.stride == 2
                u1 = Unit('1x1', blk.conv1, blk.bn1, True)
                u2 = Unit('3x3s2' if s2 else '3x3', blk.conv2, blk.bn2, True)
                u3 = Unit('1x1', blk.conv3, blk.bn3, True)
                ds = None
                if blk.downsample is not None:
                    ds = Unit('1x1s2' if s2 else '1x1', blk.downsample[0], blk.downsample[1], False)
                self.blocks.append((u1, u2, u3, ds))

    def units(self):
        us = [self.stem]
        for u1, u2, u3, ds in self.blocks:
            us += [u1, u2, u3] + ([ds] if ds is not None else [])
        return us

    def params(self):
        return [p for u in self.units() for p in u.params()]


class ResNetTrunkFn(Function):
    """NCHW image -> NCHW feature map [N, 2048, H/32, W/32]."""

    @staticmethod
    def forward(ctx, x, plan, save, training, *params):
        _check_cuda(x)
        x = _f32c(x)
        s = _lib.stream_ptr()
        it = iter(range(0, len(params), 3))
        pget = lambda: (lambda i: (_f32c(params[i]), params[i + 1], params[i + 2]))(next(it))
        recs = []
        w, g, b = pget()
        y, r = plan.stem.forward(x, w, g, b, None, save, training)
        N, H, W, C = y.shape
        Hp, Wp = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
        p = torch.empty(N, Hp, Wp, C, device=x.device, dtype=torch.float32)
        am = torch.empty(N, Hp, Wp, C, device=x.device, dtype=torch.uint8) if save else None
        _lib.call('hk_maxpool3x3s2_fwd', y, p, am, N, H, W, C, s)
        if _ops.CAPTURE is not None:
            _ops.CAPTURE.append(('pool3', am, (N, H, W, C)))
        recs.append(('stem', r, (tuple(y.shape), am) if save else None))
        cur = p
        for (u1, u2, u3, ds) in plan.blocks:
            w, g, b = pget()
            a1, r1 = u1.forward(cur, w, g, b, None, save, training)
            w, g, b = pget()
            a2, r2 = u2.forward(a1, w, g, b, None, save, training)
            w3, g3, b3 = pget()
            rd = None
            identity = cur
            if ds is not None:
                w, g, b = pget()
                identity, rd = ds.forward(cur, w, g, b, None, save, training)
            out, r3 = u3.forward(a2, w3, g3, b3, identity, save, training)
            recs.append(('block', (r1, r2, r3, rd), None))
            cur = out
        N, H, W, C = cur.shape
        feat = torch.empty(N, C, H, W, device=x.device, dtype=torch.float32)
        _lib.call('hk_nhwc_to_nchw', cur, feat, N, H * W, C, s)
        ctx.plan, ctx.recs, ctx.nparams = plan, (recs if save else None), len(params)
        return feat

    @staticmethod
    def backward(ctx, dfeat):
        if ctx.recs is None:
            return (None,) * (4 + ctx.nparams)
        plan, recs = ctx.plan, ctx.recs
        s = _lib.stream_ptr()
        dfeat = _f32c(dfeat)
        N, C, H, W = dfeat.shape
        g = torch.empty(N, H, W, C, device=dfeat.device, dtype=torch.float32)
        _lib.call('hk_nchw_to_nhwc', dfeat, g, N, H * W, C, s)
        grads = []   # collected in reverse unit order, each (dw, dgamma, dbeta)
        for (u1, u2, u3, ds), (_, (r1, r2, r3, rd), _) in zip(reversed(plan.blocks), reversed(recs[1:])):
            d2, dres, dw3, dg3, db3 = u3.backward(r3, g)
            d1, _, dw2, dg2, db2 = u2.backward(r2, d2)
            # the identity branch's gradient (dres, or the downsample unit's dx) is added inside u1's dgrad GEMM epilogue
            extra = None
            if ds is not None:
                dxd, _, dwd, dgd, dbd = ds.backward(rd, dres)
                extra = (dwd, dgd, dbd)
            dx, _, dw1, dg1, db1 = u1.backward(r1, d1, addend=dxd if ds is not None else dres)
            blk = [(dw1, dg1, db1), (dw2, dg2, db2), (dw3, dg3, db3)]
            if extra is not None:
                blk.append(extra)
            grads = blk + grads
            g = dx
        _, r0, (yshape, am) = recs[0]
        N, H, W, C = yshape
        dy0 = torch.empty(N, H, W, C, device=dfeat.device, dtype=torch.float32)
        _lib.call('hk_maxpool3x3s2_bwd', am, g, dy0, N, H, W, C, s)
        _, _, dw0, dg0, db0 = plan.stem.backward(r0, dy0, need_dx=False)
        grads = [(dw0, dg0, db0)] + grads
        ctx.recs = None
        flat = [t for trip in grads for t in trip]
        return (None, None, None, None) + tuple(flat)


def resnet_trunk(x, trunk_module):
    plan = trunk_module._plan
    params = plan.params()
    training = trunk_module.training
    save = _wants_grad(x, params, training, 'ResNet trunk')
    return ResNetTrunkFn.apply(x, plan, save, training, *params)


def _wants_grad(x, params, training, what):
    """Save-for-backward decision, taken from what requires grad at call time.  Gradients through EVAL-mode BatchNorm
    (running statistics) are not on the reference's training path and have no kernel here: asking for them is an error,
    never a silent None."""
    want = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
    if want and not training:
        raise _lib.HawkeyeLibError(f'{what}: backward through eval-mode BatchNorm is not implemented — call .train(), '
                                   'or run under torch.no_grad() / with all inputs and parameters frozen')
    return want


class DRBlockFn(Function):
    """MPNCOV.conv_dr_block (MPNCOV.py:64-69): 1x1 conv (no bias) + BN + ReLU, NCHW in / NCHW out."""

    @staticmethod
    def forward(ctx, x, unit, save, training, w, gamma, beta):
        _check_cuda(x)
        x = _f32c(x)
        s = _lib.stream_ptr()
        N, C, H, W = x.shape
        xn = torch.empty(N, H, W, C, device=x.device, dtype=torch.float32)
        _lib.call('hk_nchw_to_nhwc', x, xn, N, H * W, C, s)
        y, rec = unit.forward(xn, _f32c(w), gamma, beta, None, save, training)
        out = torch.empty(N, y.shape[-1], H, W, device=x.device, dtype=torch.float32)
        _lib.call('hk_nhwc_to_nchw', y, out, N, H * W, y.shape[-1], s)
        ctx.unit, ctx.rec = unit, rec
        return out

    @staticmethod
    def backward(ctx, dout):
        if ctx.rec is None:
            return (None,) * 7
        s = _lib.stream_ptr()
        dout = _f32c(dout)
        N, C, H, W = dout.shape
        g = torch.empty(N, H, W, C, device=dout.device, dtype=torch.float32)
        _lib.call('hk_nchw_to_nhwc', dout, g, N, H * W, C, s)
        dx, _, dw, dg, db = ctx.unit.backward(ctx.rec, g)
        cin = dx.shape[-1]
        dxn = torch.empty(N, cin, H, W, device=dout.device, dtype=torch.float32)
        _lib.call('hk_nhwc_to_nchw', dx, dxn, N, H * W, cin, s)
        ctx.rec = None
        return dxn, None, None, None, dw, dg, db
