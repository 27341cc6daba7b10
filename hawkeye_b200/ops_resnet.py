"""ResNet-50 v1.5 trunk (reference model/backbone/resnet.py:89-252) and the MPN-COV dimension-reduction block
(MPNCOV.py:64-69) as explicit forward/backward pipelines over the C-ABI kernels, NHWC fp32 inside, and the same BatchNorm
over [P, C] rows for the methods' heads (RowBatchNormFn).

conv unit = convolution (wgmma GEMM / implicit GEMM) -> BatchNorm (+ residual) (+ ReLU).  BatchNorm runs on the batch
statistics in train mode and on the running statistics in eval mode; both have a backward (eval mode: the statistics are
constants, hk_bn_bwd_frozen).
"""
import torch
from torch.autograd import Function

from . import _lib, ops as _ops
from .ops import (_check_cuda, _f32c, _ws, add_, conv3x3_dgrad, conv3x3_fwd, conv3x3_pack, conv3x3_wgrad, gemm,
                  nchw_to_nhwc, nhwc_to_nchw)

BN_EPS = 1e-5


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
            gemm(x147, 0, 160, 0, w147, 0, 160, 0, c, cout, 0, P, cout, 160)
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
                gemm(xin, 0, cin, 0, w, 0, cin, 0, c, cout, 0, P, cout, cin)
                rec['xin'] = xin
            else:
                wf, rec['wd'] = conv3x3_pack(w, save)
                c = conv3x3_fwd(x, wf, None, relu=False, stride=2 if self.kind == '3x3s2' else 1)
                Ho, Wo = c.shape[1:3]
                rec['xin'] = x
            P = N * Ho * Wo
        y, mean, invstd = bn_forward(c, P, cout, gamma, beta, residual, self.bn, training, self.relu, s)
        if _ops.CAPTURE is not None and self.relu:
            _ops.CAPTURE.append(('relu', y))
        if save:
            rec.update(c=c, y=y if self.relu else None, mean=mean, invstd=invstd, P=P, cout=cout, w=w, gamma=gamma, beta=beta,
                       shape=(N, Ho, Wo), has_res=residual is not None, frozen=not training)
            return y, rec
        return y, None

    # ---- backward: dy NHWC -> (dx NHWC or None, dres or None, dw, dgamma, dbeta)
    def backward(self, rec, dy, need_dx=True, addend=None):
        """addend (optional, same shape as dx): added to dx — inside the dgrad GEMM's epilogue for 1x1 convs"""
        s = _lib.stream_ptr()
        dev = dy.device
        P, cout = rec['P'], rec['cout']
        N, Ho, Wo = rec['shape']
        # BN + ReLU without a residual: the mask is recomputed from x (hk_bn_bwd_ex), y is not read
        mask_beta = rec['beta'] if (self.relu and not rec['has_res']) else None
        dc, dres, dgamma, dbeta = bn_backward(rec['c'], rec['y'], dy, rec['gamma'], mask_beta, rec['mean'], rec['invstd'],
                                              rec['has_res'], self.relu, rec['frozen'], P, cout, s)
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
                # dX = dC . W (+ addend, in the epilogue)  (W [Cout,Cin] as the MN-major B)
                fuse = addend is not None and self.kind == '1x1'
                gemm(dc, 0, cout, 0, w, 1, cin, 0, dxs, cin, 0, P, cin, cout, D=addend if fuse else None,
                     ldd=cin if fuse else 0, beta=1.0 if fuse else 0.0)
                if fuse:
                    addend = None
                if self.kind == '1x1s2':
                    H, W = rec['full_hw']
                    dx = torch.empty(N, H, W, cin, device=dev, dtype=torch.float32)
                    _lib.call('hk_upsample2_zero', dxs, dx, N, H, W, cin, s)
                else:
                    dx = dxs
        else:
            _, H, W, cin = xin.shape
            g = dc
            if self.kind == '3x3s2':                    # adjoint of the stride: zero-insert dC to the input resolution
                g = torch.empty(N, H, W, cout, device=dev, dtype=torch.float32)
                _lib.call('hk_upsample2_zero', dc, g, N, H, W, cout, s)
            dw = torch.empty(cout, cin, 3, 3, device=dev, dtype=torch.float32)
            conv3x3_wgrad(xin, g, dw)
            if need_dx:
                dx = conv3x3_dgrad(g, rec['wd'])
        if addend is not None and dx is not None:
            dx = add_(dx, addend)
        return dx, dres, dw, dgamma, dbeta


def bn_forward(x, P, C, gamma, beta, residual, bn, training, relu, s):
    """BatchNorm of x as [P, C] rows (+ residual) (+ ReLU) with the parameters gamma, beta and the statistics of the
    nn.BatchNorm ``bn`` -> (y, mean, invstd).  Train mode normalises with the batch statistics, updates the running ones and
    counts ``num_batches_tracked``; eval mode normalises with the running statistics."""
    y = torch.empty_like(x)
    if training:
        mean = torch.empty(C, device=x.device, dtype=torch.float32)
        invstd = torch.empty(C, device=x.device, dtype=torch.float32)
        ws = _ws(_lib.query('hk_bn_workspace_bytes', P, C), x.device)
        _lib.call('hk_bn_fwd', x, gamma, beta, residual, y, mean, invstd, bn.running_mean, bn.running_var,
                  float(bn.momentum), float(bn.eps), P, C, int(relu), ws, ws.numel(), s)
        bn.num_batches_tracked += 1
    else:
        mean = bn.running_mean
        invstd = torch.rsqrt(bn.running_var + bn.eps)
        _lib.call('hk_bn_apply', x, mean, invstd, gamma, beta, residual, y, P, C, int(relu), s)
    return y, mean, invstd


def bn_backward(x, y, dy, gamma, mask_beta, mean, invstd, has_res, relu, frozen, P, C, s):
    """The backward of bn_forward from its input x, output y (read for the ReLU mask unless ``mask_beta`` lets the kernel
    recompute it from x) and (mean, invstd) -> (dx, dresidual or None, dgamma, dbeta).  ``frozen`` (eval mode) holds the
    statistics constant."""
    dx = torch.empty_like(x)
    dres = torch.empty_like(dx) if has_res else None
    dgamma = torch.empty(C, device=x.device, dtype=torch.float32)
    dbeta = torch.empty(C, device=x.device, dtype=torch.float32)
    ws = _ws(_lib.query('hk_bn_workspace_bytes', P, C), x.device)
    _lib.call('hk_bn_bwd_frozen' if frozen else 'hk_bn_bwd_ex', x, y, dy, gamma, mask_beta, mean, invstd, dx, dres, dgamma,
              dbeta, P, C, int(relu), ws, ws.numel(), s)
    return dx, dres, dgamma, dbeta


def block_units(blk):
    """(u1, u2, u3, ds) units of one bottleneck block: ResNet's Bottleneck (3x3 middle conv, v1.5 stride on it) or a
    Bottleneck1x1 (Interp_Parts.py:212-248, every conv 1x1); the middle unit's kind follows ``conv2.kernel_size``."""
    s2 = blk.stride == 2
    mid = ('3x3s2' if s2 else '3x3') if tuple(blk.conv2.kernel_size) == (3, 3) else ('1x1s2' if s2 else '1x1')
    ds = None
    if blk.downsample is not None:
        ds = Unit('1x1s2' if s2 else '1x1', blk.downsample[0], blk.downsample[1], False)
    return (Unit('1x1', blk.conv1, blk.bn1, True), Unit(mid, blk.conv2, blk.bn2, True), Unit('1x1', blk.conv3, blk.bn3, True),
            ds)


def block_params(blocks):
    return [p for b in blocks for u in b if u is not None for p in u.params()]


def blocks_forward(cur, blocks, pget, save, training):
    """NHWC [N, H, W, C] through the bottleneck blocks -> (NHWC output, per-block records for blocks_backward).
    ``pget()`` yields each unit's (weight, gamma, beta) in the order of ``block_params``."""
    recs = []
    for (u1, u2, u3, ds) in blocks:
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
        recs.append((r1, r2, r3, rd))
        cur = out
    return cur, recs


def blocks_backward(g, blocks, recs):
    """NHWC output gradient -> (NHWC input gradient, [(dw, dgamma, dbeta)] in the order of ``block_params``)."""
    grads = []   # collected in reverse unit order, each (dw, dgamma, dbeta)
    for (u1, u2, u3, ds), (r1, r2, r3, rd) in zip(reversed(blocks), reversed(recs)):
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
    return g, grads


class TrunkPlan:
    """Flattened description of a ResNet trunk: stem unit, max-pool, list of bottleneck blocks.  ``trunk`` is indexable as
    conv1, bn1, relu, maxpool, then the layers (a ResNetTrunk, or the same modules in a list)."""

    def __init__(self, trunk):
        self.stem = Unit('stem', trunk[0], trunk[1], True)
        self.blocks = [block_units(blk) for layer in list(trunk)[4:] for blk in layer]

    def units(self):
        us = [self.stem]
        for u1, u2, u3, ds in self.blocks:
            us += [u1, u2, u3] + ([ds] if ds is not None else [])
        return us

    def params(self):
        return [p for u in self.units() for p in u.params()]


def _param_iter(params):
    it = iter(range(0, len(params), 3))
    return lambda: (lambda i: (_f32c(params[i]), params[i + 1], params[i + 2]))(next(it))


class ResNetTrunkFn(Function):
    """NCHW image -> NCHW feature map [N, 2048, H/32, W/32]; with ``nhwc`` the NHWC map [N, H/32, W/32, 2048] as the last
    block writes it (and its gradient arrives in NHWC)."""

    @staticmethod
    def forward(ctx, x, plan, save, training, nhwc, *params):
        _check_cuda(x)
        x = _f32c(x)
        s = _lib.stream_ptr()
        pget = _param_iter(params)
        w, g, b = pget()
        y, r = plan.stem.forward(x, w, g, b, None, save, training)
        N, H, W, C = y.shape
        Hp, Wp = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
        p = torch.empty(N, Hp, Wp, C, device=x.device, dtype=torch.float32)
        am = torch.empty(N, Hp, Wp, C, device=x.device, dtype=torch.uint8) if save else None
        _lib.call('hk_maxpool3x3s2_fwd', y, p, am, N, H, W, C, s)
        if _ops.CAPTURE is not None:
            _ops.CAPTURE.append(('pool3', am, (N, H, W, C)))
        cur, brecs = blocks_forward(p, plan.blocks, pget, save, training)
        ctx.plan, ctx.nparams, ctx.nhwc = plan, len(params), nhwc
        ctx.recs = ((r, tuple(y.shape), am), brecs) if save else None
        return cur if nhwc else nhwc_to_nchw(cur)

    @staticmethod
    def backward(ctx, dfeat):
        if ctx.recs is None:
            return (None,) * (5 + ctx.nparams)
        plan, ((r0, yshape, am), brecs) = ctx.plan, ctx.recs
        s = _lib.stream_ptr()
        g = _f32c(dfeat) if ctx.nhwc else nchw_to_nhwc(_f32c(dfeat))
        g, grads = blocks_backward(g, plan.blocks, brecs)
        N, H, W, C = yshape
        dy0 = torch.empty(N, H, W, C, device=dfeat.device, dtype=torch.float32)
        _lib.call('hk_maxpool3x3s2_bwd', am, g, dy0, N, H, W, C, s)
        _, _, dw0, dg0, db0 = plan.stem.backward(r0, dy0, need_dx=False)
        grads = [(dw0, dg0, db0)] + grads
        ctx.recs = None
        flat = [t for trip in grads for t in trip]
        return (None, None, None, None, None) + tuple(flat)


class BlockStackFn(Function):
    """NHWC map [N, H, W, C] through a stack of bottleneck blocks (Interp-Parts' post_block and the Bottleneck1x1 pair of
    attconv, on P = N*K rows of 1x1 maps) -> NHWC output."""

    @staticmethod
    def forward(ctx, x, blocks, save, training, *params):
        _check_cuda(x)
        out, recs = blocks_forward(_f32c(x), blocks, _param_iter(params), save, training)
        ctx.blocks, ctx.nparams, ctx.recs = blocks, len(params), (recs if save else None)
        return out

    @staticmethod
    def backward(ctx, dout):
        if ctx.recs is None:
            return (None,) * (4 + ctx.nparams)
        dx, grads = blocks_backward(_f32c(dout), ctx.blocks, ctx.recs)
        ctx.recs = None
        return (dx, None, None, None) + tuple(t for trip in grads for t in trip)


def block_stack(x, blocks, training):
    """x NHWC through ``blocks`` (a list of block_units) with the units' own parameters."""
    params = block_params(blocks)
    return BlockStackFn.apply(x, blocks, _ops.wants_grad(x, params), training, *params)


def resnet_trunk(x, trunk_module):
    plan = trunk_module._plan
    params = plan.params()
    training = trunk_module.training
    save = _ops.wants_grad(x, params)
    return ResNetTrunkFn.apply(x, plan, save, training, False, *params)


def resnet_trunk_nhwc(x, plan, training):
    """The trunk of ``plan`` on an NCHW image -> its NHWC output map, without the NCHW transpose."""
    params = plan.params()
    return ResNetTrunkFn.apply(x, plan, _ops.wants_grad(x, params), training, True, *params)


class DRBlockFn(Function):
    """MPNCOV.conv_dr_block (MPNCOV.py:64-69): 1x1 conv (no bias) + BN + ReLU, NCHW in / NCHW out."""

    @staticmethod
    def forward(ctx, x, unit, save, training, w, gamma, beta):
        _check_cuda(x)
        y, rec = unit.forward(nchw_to_nhwc(_f32c(x)), _f32c(w), gamma, beta, None, save, training)
        ctx.unit, ctx.rec = unit, rec
        return nhwc_to_nchw(y)

    @staticmethod
    def backward(ctx, dout):
        if ctx.rec is None:
            return (None,) * 7
        dx, _, dw, dg, db = ctx.unit.backward(ctx.rec, nchw_to_nhwc(_f32c(dout)))
        ctx.rec = None
        return nhwc_to_nchw(dx), None, None, None, dw, dg, db


class RowBatchNormFn(Function):
    """nn.BatchNorm over [P, C] rows (Interp-Parts' groupingbn on the pooled features, Interp_Parts.py:365; AP-CNN's
    BatchNorm1d heads) on bn_forward / bn_backward."""

    @staticmethod
    def forward(ctx, x, gamma, beta, bn, training):
        _check_cuda(x, gamma, beta)
        x = _f32c(x)
        P, C = x.shape
        if training and P < 2:
            raise _lib.HawkeyeLibError(f'BatchNorm over rows: train mode needs more than one row (got {P})')
        y, mean, invstd = bn_forward(x, P, C, gamma, beta, None, bn, training, False, _lib.stream_ptr())
        ctx.save_for_backward(x, gamma, mean, invstd)
        ctx.frozen = not training
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, invstd = ctx.saved_tensors
        P, C = x.shape
        dx, _, dgamma, dbeta = bn_backward(x, None, _f32c(dy), gamma, None, mean, invstd, False, False, ctx.frozen, P, C,
                                           _lib.stream_ptr())
        return dx, dgamma, dbeta, None, None
