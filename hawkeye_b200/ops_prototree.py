"""Autograd bindings for ProtoTree (reference model/methods/ProtoTree/ and Examples/ProtoTreeNet.py): the 1x1 neck as one
GEMM node, the prototype distance with its global min-pool, the soft decision tree, the NLL of its output and the
derivative-free leaf update.  Host plumbing only: shapes are checked here before any launch, all arithmetic is in
libhawkeye_b200.so.

Tree layout: height H, 2^H - 1 branches, 2^H leaves, nodes numbered in pre-order as the reference numbers them
(prototree.py:275-287).  Prototype row k belongs to the k-th branch in pre-order and leaf row j to the j-th leaf from the left.
"""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws, gemm, nchw_to_nhwc, nhwc_to_nchw

MAX_HEIGHT = 12            # hk_prototree_*: one float per node of the tree in shared memory


def check_height(height):
    if not 1 <= int(height) <= MAX_HEIGHT:
        raise _lib.HawkeyeLibError(f'ProtoTree: height={height} is outside the supported 1..{MAX_HEIGHT}')


class NeckFn(Function):
    """Trunk map [N, C, H, W] (NCHW) and the neck's 1x1 weight [D, C, 1, 1] -> pre-activation [N, H*W, D]
    (position-major, the layout hk_prototree_dist_fwd reads).  One hk_gemm_tf32; backward one dgrad GEMM and one
    hk_matconv_wgrad."""

    @staticmethod
    def forward(ctx, feat, w):
        _check_cuda(feat, w)
        feat, w = _f32c(feat), _f32c(w)
        if feat.dim() != 4 or w.dim() != 4 or w.shape[1] != feat.shape[1] or w.shape[2:] != (1, 1):
            raise _lib.HawkeyeLibError(f'ProtoTree neck: map {tuple(feat.shape)} and weight {tuple(w.shape)} are not a '
                                       '[N, C, H, W] map and a [D, C, 1, 1] convolution')
        N, C, H, W = feat.shape
        D = w.shape[0]
        x = nchw_to_nhwc(feat)
        w2 = w.view(D, C)
        c = torch.empty(N, H * W, D, device=feat.device, dtype=torch.float32)
        gemm(x, 0, C, 0, w2, 0, C, 0, c, D, 0, N * H * W, D, C)
        ctx.save_for_backward(x, w2)
        ctx.w_shape = w.shape
        return c

    @staticmethod
    def backward(ctx, dc):
        x, w2 = ctx.saved_tensors
        N, H, W, C = x.shape
        D = w2.shape[0]
        M = N * H * W
        dc = _f32c(dc)
        s = _lib.stream_ptr()
        dfeat = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            gemm(dc, 0, D, 0, w2, 1, C, 0, dx, C, 0, M, C, D)
            dfeat = nhwc_to_nchw(dx)
        if ctx.needs_input_grad[1]:
            dw = torch.empty(ctx.w_shape, device=x.device, dtype=torch.float32)
            ws = _ws(_lib.query('hk_matconv_wgrad_workspace_bytes', M, C, D), x.device)
            _lib.call('hk_matconv_wgrad', x, dc, dw, M, C, D, ws, ws.numel(), s)
        return dfeat, dw


class PrototypeDistanceFn(Function):
    """x [N, HW, D], prototypes [P, D, 1, 1] (or [P, D]) -> mind [N, P]: the smallest L2 distance of each prototype to any
    position (l2conv.py:24-63 + the global min-pool of prototree.py:115).  ``act``: x is the neck's pre-activation and
    the sigmoid is applied on load; otherwise x holds the features themselves."""

    @staticmethod
    def forward(ctx, x, protos, act):
        _check_cuda(x, protos)
        x, protos = _f32c(x), _f32c(protos)
        if x.dim() != 3 or protos.dim() not in (2, 4) or protos.shape[1] != x.shape[2] or protos.shape[2:] not in ((), (1, 1)):
            raise _lib.HawkeyeLibError(f'PrototypeDistance: features {tuple(x.shape)} and prototypes {tuple(protos.shape)} '
                                       'are not [N, HW, D] and [P, D, 1, 1]')
        N, HW, D = x.shape
        P = protos.shape[0]
        z = torch.empty_like(x) if act else x
        mind = torch.empty(N, P, device=x.device, dtype=torch.float32)
        argmin = torch.empty(N, P, device=x.device, dtype=torch.int32)
        _lib.call('hk_prototree_dist_fwd', x, protos, z if act else None, mind, argmin, N, HW, D, P, int(act),
                  _lib.stream_ptr())
        ctx.save_for_backward(z, protos, mind, argmin)
        ctx.act = bool(act)
        ctx.mark_non_differentiable(argmin)
        return mind, argmin

    @staticmethod
    def backward(ctx, dmind, _dargmin=None):
        z, protos, mind, argmin = ctx.saved_tensors
        N, HW, D = z.shape
        P = protos.shape[0]
        dx = torch.empty_like(z)
        dp = torch.empty_like(protos)
        _lib.call('hk_prototree_dist_bwd', z, protos, mind, argmin, _f32c(dmind), dx, dp, N, HW, D, P, int(ctx.act),
                  _lib.stream_ptr())
        return dx, dp, None


class RouteFn(Function):
    """mind [N, P] and the leaf parameters theta [L, K] -> (pred [N, K], ps [N, P], pa [N, 2L - 1]).  ps (by branch rank) and
    pa (by node index) are the routing probabilities the reference reports in ``info``; they carry no gradient here."""

    @staticmethod
    def forward(ctx, mind, theta, height):
        _check_cuda(mind, theta)
        mind, theta = _f32c(mind), _f32c(theta)
        check_height(height)
        P, L = (1 << height) - 1, 1 << height
        if mind.dim() != 2 or mind.shape[1] != P or theta.dim() != 2 or theta.shape[0] != L:
            raise _lib.HawkeyeLibError(f'ProtoTree of height {height}: needs {P} distances per row and {L} leaf rows, got '
                                       f'mind {tuple(mind.shape)} and leaves {tuple(theta.shape)}')
        N, K = mind.shape[0], theta.shape[1]
        dev = mind.device
        sm = torch.empty(L, K, device=dev, dtype=torch.float32)
        ps = torch.empty(N, P, device=dev, dtype=torch.float32)
        pa = torch.empty(N, 2 * L - 1, device=dev, dtype=torch.float32)
        pred = torch.empty(N, K, device=dev, dtype=torch.float32)
        _lib.call('hk_prototree_route_fwd', mind, theta, sm, ps, pa, pred, N, height, K, _lib.stream_ptr())
        ctx.save_for_backward(ps, pa, sm)
        ctx.height = height
        ctx.mark_non_differentiable(ps, pa)
        return pred, ps, pa

    @staticmethod
    def backward(ctx, dpred, _dps=None, _dpa=None):
        ps, pa, sm = ctx.saved_tensors
        N, K = ps.shape[0], sm.shape[1]
        dpred = torch.zeros(N, K, device=ps.device) if dpred is None else _f32c(dpred)
        dmind = torch.empty_like(ps)
        dtheta = torch.empty_like(sm) if ctx.needs_input_grad[1] else None
        _lib.call('hk_prototree_route_bwd', ps, pa, sm, dpred, dmind, dtheta, N, ctx.height, K, _lib.stream_ptr())
        return dmind, dtheta, None


class NLLFn(Function):
    """pred [N, K], labels [N] -> (F.nll_loss(torch.log(pred), labels), top-1 count), Examples/ProtoTreeNet.py:109.  One
    hk_prototree_nll launch writes the loss and its gradient."""

    @staticmethod
    def forward(ctx, pred, labels):
        _check_cuda(pred, labels)
        pred = _f32c(pred)
        if pred.dim() != 2 or labels.numel() != pred.shape[0]:
            raise _lib.HawkeyeLibError(f'ProtoTree NLL: pred {tuple(pred.shape)} and {labels.numel()} labels')
        labels = labels.contiguous().to(torch.int64)
        N, K = pred.shape
        loss = torch.empty(1, device=pred.device, dtype=torch.float32)
        dpred = torch.empty_like(pred)
        correct = torch.empty(1, device=pred.device, dtype=torch.int32)
        _lib.call('hk_prototree_nll', pred, labels, loss, dpred, correct, N, K, _lib.stream_ptr())
        ctx.save_for_backward(dpred)
        ctx.mark_non_differentiable(correct)
        return loss[0], correct

    @staticmethod
    def backward(ctx, g, _g_correct=None):
        dpred, = ctx.saved_tensors
        return dpred * g, None


def leaf_update(theta, theta0, pa, pred, labels, num_batches, reduce=None):
    """The derivative-free leaf update of Examples/ProtoTreeNet.py:116-132, in place on theta [L, K], from one step's pa
    [N, 2L - 1], pred [N, K] and labels [N] and the epoch-start snapshot theta0.  ``reduce`` (optional) is called on the
    [L, K] update sum before it is applied: data-parallel ranks pass an all-reduce, so that the update covers the global
    batch as under the reference's nn.DataParallel and every rank's leaves stay identical."""
    _check_cuda(theta, theta0, pa, pred, labels)
    L, K = theta.shape
    height = L.bit_length() - 1
    N = pred.shape[0]
    if (L != 1 << height or theta0.shape != theta.shape or pa.shape != (N, 2 * L - 1) or pred.shape[1] != K
            or labels.numel() != N):
        raise _lib.HawkeyeLibError(f'ProtoTree leaf update: leaves {tuple(theta.shape)}, snapshot {tuple(theta0.shape)}, '
                                   f'pa {tuple(pa.shape)}, pred {tuple(pred.shape)}, {labels.numel()} labels')
    check_height(height)
    if not (theta.is_contiguous() and theta.dtype == torch.float32):
        raise _lib.HawkeyeLibError('ProtoTree leaf update: the leaf parameters must be one contiguous fp32 tensor')
    s = _lib.stream_ptr()
    update = torch.empty_like(theta)
    _lib.call('hk_prototree_leaf_update_sum', theta, _f32c(pa), _f32c(pred), labels.contiguous().to(torch.int64), update, N,
              height, K, s)
    if reduce is not None:
        reduce(update)
    _lib.call('hk_prototree_leaf_update_apply', theta, _f32c(theta0), update, height, K, float(num_batches),
              _lib.stream_ptr())
