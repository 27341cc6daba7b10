"""Autograd bindings for Interp-Parts (reference model/methods/Interp_Parts.py, model/loss/InterpParts_loss.py): the grouping
unit, the part attention with the attention-weighted part sum, the blurred part occupancy and the shaping loss.  Host
plumbing only: shapes are checked here before any launch, all arithmetic is in libhawkeye_b200.so.

The shaping loss's gradient reaches the grouping unit without a dense d assign: the grouping node has a third output, a
zero [N, K] ``sink`` that the occupancy node takes as an input, and the gradient that arrives on the sink is the per-(n, k)
coefficient of the one blurred maximum.  The occupancy node leaves its argmax on the grouping node's ``ShapingTap``, and the
grouping backward spreads the coefficient through the Gaussian taps (hk_ip_group_bwd).  ``grouping`` attaches the
(tap, sink) pair to the assign tensor it returns, so the loss needs nothing but assign.
"""
import numpy as np
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws

MAX_PARTS = 32             # hk_ip_group_*: one register per part
SHAPING_EPS = 1e-5         # InterpParts_loss.py:83


def check_parts(K):
    if not 1 <= int(K) <= MAX_PARTS:
        raise _lib.HawkeyeLibError(f'Interp-Parts: num_parts={K} is outside the supported 1..{MAX_PARTS}')


def check_radius(radius, H, W):
    if radius < 0 or 2 * radius >= H or 2 * radius >= W:
        raise _lib.HawkeyeLibError(f'Interp-Parts shaping loss: radius={radius} leaves no "valid" blurred output on a '
                                   f'{H}x{W} assignment map (needs 2 * radius < min(H, W))')


def gaussian_taps(radius, std):
    """GaussianKernel (InterpParts_loss.py:34-59) as the reference builds it: fp32 taps exp(-(i^2 + j^2) / (2 std^2)),
    normalised by their fp32 sum; [1.0] for radius 0 (no blur)."""
    size = 2 * radius + 1
    weight = torch.ones(size, size)
    for i in range(-radius, radius + 1):
        for j in range(-radius, radius + 1):
            weight[i + radius][j + radius] = np.exp(-(i * i + j * j) / (2 * std * std))
    return (weight / weight.sum()).reshape(-1)


def beta_prior(n, alpha, beta):
    """update_prior_dist (InterpParts_loss.py:62-80): the Beta(alpha, beta) quantiles at the fp32 grid (2i + 1) / (2n),
    i = 0..n-1, as fp32 [n] (on the host: scipy)."""
    from scipy import stats
    grid = (torch.arange(1., 2 * n, 2.).float() / (2 * n)).numpy()
    return torch.tensor(stats.beta.ppf(grid, a=alpha, b=beta)).float()


class ShapingTap:
    """What the occupancy node leaves for the grouping backward: the argmax [N, K], the Gaussian taps and the radius."""

    def __init__(self):
        self.argmax = self.gauss = None
        self.radius = 0


class GroupingFn(Function):
    """x NHWC [N, H, W, C], centres [K, C, 1, 1], smooth_factor [K] -> (out [N, K, C] (the normalised residual codes, the
    reference's outputs_t transposed), assign [N, K, H, W], sink [N, K] zeros), Interp_Parts.py:56-122."""

    @staticmethod
    def forward(ctx, x, centres, smooth, tap):
        _check_cuda(x, centres, smooth)
        x, centres, smooth = _f32c(x), _f32c(centres), _f32c(smooth)
        if x.dim() != 4 or centres.dim() not in (2, 4) or centres.shape[1] != x.shape[3] or smooth.shape != centres.shape[:1]:
            raise _lib.HawkeyeLibError(f'GroupingUnit: map {tuple(x.shape)}, centres {tuple(centres.shape)} and smooth factor '
                                       f'{tuple(smooth.shape)} are not an NHWC [N, H, W, C] map, [K, C, 1, 1] and [K]')
        N, H, W, C = x.shape
        K = centres.shape[0]
        check_parts(K)
        if C % 4:
            raise _lib.HawkeyeLibError(f'GroupingUnit: C={C} channels must be a multiple of 4')
        dev = x.device
        e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        assign, dist, out, qx, ssum, nrm = e(N, K, H, W), e(N, K, H * W), e(N, K, C), e(N, K, C), e(N, K), e(N, K)
        ws = _ws(_lib.query('hk_ip_group_workspace_bytes', N, H * W, K, C), dev)
        _lib.call('hk_ip_group_fwd', x, centres, smooth, assign, dist, out, qx, ssum, nrm, N, H * W, K, C, ws, ws.numel(),
                  _lib.stream_ptr())
        sink = torch.zeros(N, K, device=dev, dtype=torch.float32)
        ctx.save_for_backward(x, centres, smooth, assign, dist, qx, ssum, nrm)
        ctx.tap = tap
        ctx.set_materialize_grads(False)
        return out, assign, sink

    @staticmethod
    def backward(ctx, dout, dassign, dsink):
        x, centres, smooth, assign, dist, qx, ssum, nrm = ctx.saved_tensors
        N, H, W, C = x.shape
        K = centres.shape[0]
        dev = x.device
        dout = torch.zeros(N, K, C, device=dev) if dout is None else _f32c(dout)
        tap = ctx.tap
        coef = _f32c(dsink) if (dsink is not None and tap is not None and tap.argmax is not None) else None
        dx = torch.empty_like(x)
        dcen = torch.empty_like(centres)
        dsmooth = torch.empty_like(smooth)
        ws = _ws(_lib.query('hk_ip_group_workspace_bytes', N, H * W, K, C), dev)
        _lib.call('hk_ip_group_bwd', x, centres, smooth, assign, dist, qx, ssum, nrm, dout,
                  None if dassign is None else _f32c(dassign), tap.argmax if coef is not None else None, coef,
                  tap.gauss if coef is not None else None, tap.radius if coef is not None else 0, dx, dcen, dsmooth, N, H, W,
                  K, C, ws, ws.numel(), _lib.stream_ptr())
        return dx, dcen, dsmooth, None


def grouping(x, centres, smooth):
    """GroupingFn with its shaping tap attached to the returned assign (``assign._ip_tap = (tap, sink)``)."""
    tap = ShapingTap()
    out, assign, sink = GroupingFn.apply(x, centres, smooth, tap)
    if sink.requires_grad:
        assign._ip_tap = (tap, sink)
    return out, assign


class OccupancyFn(Function):
    """assign [N, K, H, W] -> (occ [N, K], argmax [N, K] int32): the maximum of the "valid" Gaussian blur of each map and its
    first position (InterpParts_loss.py:114-124).  The gradient of occ leaves through ``sink`` (see the module docstring)."""

    @staticmethod
    def forward(ctx, assign, sink, gauss, radius, tap):
        _check_cuda(assign, gauss)
        assign = _f32c(assign)
        if assign.dim() != 4:
            raise _lib.HawkeyeLibError(f'Interp-Parts occupancy: assign {tuple(assign.shape)} is not [N, K, H, W]')
        N, K, H, W = assign.shape
        check_radius(radius, H, W)
        if gauss.numel() != (2 * radius + 1) ** 2:
            raise _lib.HawkeyeLibError(f'Interp-Parts occupancy: {gauss.numel()} Gaussian taps for radius {radius}')
        occ = torch.empty(N, K, device=assign.device, dtype=torch.float32)
        argmax = torch.empty(N, K, device=assign.device, dtype=torch.int32)
        _lib.call('hk_ip_occupancy', assign, _f32c(gauss), occ, argmax, N, K, H, W, radius, _lib.stream_ptr())
        if tap is not None:
            tap.argmax, tap.gauss, tap.radius = argmax, _f32c(gauss), radius
        ctx.mark_non_differentiable(argmax)
        return occ, argmax

    @staticmethod
    def backward(ctx, docc, _dargmax=None):
        return None, docc, None, None, None


def occupancy(assign, gauss, radius):
    """-> (occ, argmax) of ``assign``.  A differentiable assign must be the grouping unit's own (it carries the tap that
    takes the gradient back); any assign without gradients is accepted."""
    tap = getattr(assign, '_ip_tap', None)
    if tap is None or tap[0] is None:
        if assign.requires_grad and torch.is_grad_enabled():
            raise _lib.HawkeyeLibError('Interp-Parts occupancy: a differentiable assign must come from the grouping unit '
                                       '(ops_interp_parts.grouping), whose backward takes the shaping gradient')
        return OccupancyFn.apply(assign.detach(), None, gauss, radius, None)
    return OccupancyFn.apply(assign.detach(), tap[1], gauss, radius, tap[0])


class ShapingLossFn(Function):
    """occ [N, K] (this rank's rows), occ_all [R, K] (every rank's rows, this rank's at row0), prior [R] -> the shaping loss
    (InterpParts_loss.py:125-138) over the R rows; the gradient of this rank's rows, times ``world``."""

    @staticmethod
    def forward(ctx, occ, occ_all, prior, row0, world, eps):
        _check_cuda(occ, occ_all, prior)
        occ_all, prior = _f32c(occ_all), _f32c(prior)
        if (occ.dim() != 2 or occ_all.dim() != 2 or occ_all.shape[1] != occ.shape[1] or prior.shape != occ_all.shape[:1]
                or not 0 <= row0 <= occ_all.shape[0] - occ.shape[0]):
            raise _lib.HawkeyeLibError(f'Interp-Parts shaping loss: occ {tuple(occ.shape)}, gathered {tuple(occ_all.shape)}, '
                                       f'prior {tuple(prior.shape)}, row0 {row0}')
        R, K = occ_all.shape
        loss = torch.empty(1, device=occ.device, dtype=torch.float32)
        docc = torch.empty_like(occ_all)
        _lib.call('hk_ip_shaping_loss', occ_all, prior, loss, docc, R, K, float(eps), _lib.stream_ptr())
        ctx.save_for_backward(docc)
        ctx.rows, ctx.world = (row0, occ.shape[0]), world
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        docc, = ctx.saved_tensors
        r0, n = ctx.rows
        return docc[r0:r0 + n] * (g * ctx.world), None, None, None, None, None


class AttentionPoolFn(Function):
    """attconv[2:5] + softmax over the parts + the attention-weighted part sum (Interp_Parts.py:289-291,:349-361):
    f [P, C] (the Bottleneck1x1 pair's output, P = N K), post [P, D] (post_block's output), the 1-channel conv (w [1, C, 1, 1],
    b [1]) and BatchNorm(1) ``bn`` -> (pooled [N, D], att [N, K])."""

    @staticmethod
    def forward(ctx, f, post, w, b, gamma, beta, bn, training, N, K):
        _check_cuda(f, post, w, b, gamma, beta)
        f, post, w, b = _f32c(f), _f32c(post), _f32c(w), _f32c(b)
        P = N * K
        if f.dim() != 2 or post.dim() != 2 or f.shape[0] != P or post.shape[0] != P or w.numel() != f.shape[1]:
            raise _lib.HawkeyeLibError(f'Interp-Parts attention: features {tuple(f.shape)}, post-block output '
                                       f'{tuple(post.shape)} and conv weight {tuple(w.shape)} for N={N}, K={K}')
        if training and P < 2:
            raise _lib.HawkeyeLibError('Interp-Parts attention: BatchNorm in train mode needs more than one value '
                                       f'(N={N}, K={K})')
        C, D = f.shape[1], post.shape[1]
        dev = f.device
        conv = torch.empty(P, device=dev, dtype=torch.float32)
        att = torch.empty(N, K, device=dev, dtype=torch.float32)
        stats = torch.empty(2, device=dev, dtype=torch.float32)
        pooled = torch.empty(N, D, device=dev, dtype=torch.float32)
        _lib.call('hk_ip_att_fwd', f, w, b, gamma, beta, bn.running_mean, bn.running_var, float(bn.momentum), float(bn.eps),
                  int(training), post, conv, att, stats, pooled, N, K, C, D, _lib.stream_ptr())
        if training:
            bn.num_batches_tracked += 1
        ctx.save_for_backward(f, w, gamma, beta, conv, att, stats, post)
        ctx.training, ctx.NK = bool(training), (N, K)
        ctx.set_materialize_grads(False)
        return pooled, att

    @staticmethod
    def backward(ctx, dpooled, datt):
        f, w, gamma, beta, conv, att, stats, post = ctx.saved_tensors
        N, K = ctx.NK
        P, C = f.shape
        D = post.shape[1]
        dev = f.device
        dpooled = torch.zeros(N, D, device=dev) if dpooled is None else _f32c(dpooled)
        df, dpost = torch.empty_like(f), torch.empty_like(post)
        dw = torch.empty(w.shape, device=dev, dtype=torch.float32)
        db, dgamma, dbeta = (torch.empty(1, device=dev, dtype=torch.float32) for _ in range(3))
        scratch = torch.empty(P, device=dev, dtype=torch.float32)
        _lib.call('hk_ip_att_bwd', f, w, gamma, beta, conv, att, stats, post, dpooled,
                  None if datt is None else _f32c(datt), int(ctx.training), df, dw, db, dgamma, dbeta, dpost, scratch, N, K,
                  C, D, _lib.stream_ptr())
        return df, dpost, dw, db, dgamma, dbeta, None, None, None, None

