"""Autograd bindings for MGE-CNN (reference model/methods/MGE_CNN/MGE.py, grad_cam.py): the conv6* part head, the CAM
boxes and their crops, the detached concatenation and the gate.  Host plumbing only; all arithmetic is in
libhawkeye_b200.so.

The reference computes each Grad-CAM with a full autograd backward inside its forward and builds the zoomed inputs in a
Python loop over the images, with nonzero() and a host-side test of the box corners (MGE.py:48-72, :145-190).  Here the
CAM weights are the closed form of that backward and the boxes stay on the device, so a training step never
synchronises."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws, crop as _crop

CAT_SCALE = 10.0            # pool_cat* = cat(10 l2n(pool), 10 l2n(pool_conv6)), MGE.py:136


class PartFn(Function):
    """pool_max(relu(conv6(x))) on the NHWC layer3 map: x [N, H, W, C], w [O, C, 1, 1], b [O] -> pooled [N, O].  x gets no
    gradient (the reference detaches it); the weight gradient reaches only the winning pixel of each (image, channel)."""

    @staticmethod
    def forward(ctx, x, w, b):
        _check_cuda(x, w, b)
        x, w2 = _f32c(x), _f32c(w).reshape(w.shape[0], -1)
        N, H, W, C = x.shape
        O = w2.shape[0]
        if w2.shape[1] != C:
            raise _lib.HawkeyeLibError(f'MGE part head: weight {tuple(w.shape)} on a map of {C} channels')
        pooled = torch.empty(N, O, device=x.device, dtype=torch.float32)
        pos = torch.empty(N, O, device=x.device, dtype=torch.int32)
        ws = _ws(_lib.query('hk_mge_part_workspace_bytes', N, H, W, O), x.device)
        _lib.call('hk_mge_part_fwd', x, w2, _f32c(b), pooled, pos, N, H, W, C, O, ws, ws.numel(), _lib.stream_ptr())
        ctx.save_for_backward(x, pos, pooled)
        ctx.wshape = w.shape
        ctx.mark_non_differentiable(pos)
        return pooled, pos

    @staticmethod
    def backward(ctx, dpooled, _dpos):
        x, pos, pooled = ctx.saved_tensors
        N, H, W, C = x.shape
        O = pooled.shape[1]
        dw = torch.empty(ctx.wshape, device=x.device, dtype=torch.float32)
        db = torch.empty(O, device=x.device, dtype=torch.float32)
        _lib.call('hk_mge_part_bwd', x, pos, pooled, _f32c(dpooled), dw, db, N, H, W, C, O, _lib.stream_ptr())
        return None, dw, db


def part(x_nhwc, conv):
    """``conv`` is one of conv6, conv6_1, conv6_2 -> pooled [N, O] (and the winning positions, for tests)."""
    return PartFn.apply(x_nhwc.detach(), conv.weight, conv.bias)


def cam_box(feat_nhwc, w_main, image_size, rate, logits=None, targets=None):
    """The crop boxes of get_bbox (MGE.py:48-72) with the closed-form Grad-CAM weights: feat [N, h, w, C] (layer4's map),
    w_main [K, C] (the main classifier's weight), the CAM's target from ``targets`` (int64 [N]) or else the argmax of
    ``logits`` [N, K] -> int32 [N, 4] (y0, x0, y1, x1), end exclusive, the whole image for a degenerate box."""
    _check_cuda(feat_nhwc, w_main, logits, targets)
    feat, w_main = _f32c(feat_nhwc.detach()), _f32c(w_main.detach())
    N, h, w, C = feat.shape
    K = w_main.shape[0]
    if targets is not None:
        targets = targets.detach().contiguous().to(torch.int64)
        logits = None
    else:
        logits = _f32c(logits.detach())
    boxes = torch.empty(N, 4, device=feat.device, dtype=torch.int32)
    _lib.call('hk_mge_cam_box', logits, targets, w_main, feat, boxes, N, K, C, h, w, int(image_size), float(rate),
              _lib.stream_ptr())
    return boxes


def crop(images, boxes, image_size):
    """input_box of get_bbox: images NCHW [N, 3, S, S], boxes int32 [N, 4] -> NCHW [N, 3, S, S], each box resized to S x S
    (bilinear, align_corners=True) without a gradient: one box per image, no padding."""
    return _crop(images, boxes.reshape(-1, 1, 4), int(image_size), 0)


def cat_l2n(a, b, scale=CAT_SCALE):
    """cat(scale a / ||a||, scale b / ||b||) per row, of detached inputs (no gradient): [N, Da], [N, Db] -> [N, Da + Db]."""
    _check_cuda(a, b)
    a, b = _f32c(a.detach()), _f32c(b.detach())
    N, Da = a.shape
    out = torch.empty(N, Da + b.shape[1], device=a.device, dtype=torch.float32)
    _lib.call('hk_mge_cat_l2n', a, b, out, N, Da, b.shape[1], float(scale), _lib.stream_ptr())
    return out


class GateFn(Function):
    """cls_gate[1], the softmax and the gated sum (MGE.py:209-213): h [N, F] (cls_gate[0]'s output), w2 [3, F], b2 [3] and
    the three cat logits [N, K] -> (logits_gate [N, K], pr_gate [N, 3]).  The cat logits are constants here (detached in
    the reference); h, w2 and b2 get gradients."""

    @staticmethod
    def forward(ctx, h, w2, b2, c0, c1, c2):
        _check_cuda(h, w2, b2, c0, c1, c2)
        h, w2 = _f32c(h), _f32c(w2)
        cs = [_f32c(c.detach()) for c in (c0, c1, c2)]
        N, F = h.shape
        K = cs[0].shape[1]
        if w2.shape != (3, F) or any(c.shape != (N, K) for c in cs):
            raise _lib.HawkeyeLibError(f'MGE gate: h {tuple(h.shape)}, w2 {tuple(w2.shape)}, logits {[tuple(c.shape) for c in cs]}')
        pr = torch.empty(N, 3, device=h.device, dtype=torch.float32)
        out = torch.empty(N, K, device=h.device, dtype=torch.float32)
        _lib.call('hk_mge_gate_fwd', h, w2, _f32c(b2), cs[0], cs[1], cs[2], pr, out, N, F, K, _lib.stream_ptr())
        ctx.save_for_backward(h, w2, pr, *cs)
        ctx.set_materialize_grads(False)
        return out, pr

    @staticmethod
    def backward(ctx, dout, dpr):
        h, w2, pr, c0, c1, c2 = ctx.saved_tensors
        N, F = h.shape
        K = c0.shape[1]
        if dout is None:
            dout = torch.zeros(N, K, device=h.device, dtype=torch.float32)
        dz = torch.empty(N, 3, device=h.device, dtype=torch.float32)
        dh = torch.empty_like(h) if ctx.needs_input_grad[0] else None
        dw2 = torch.empty_like(w2) if ctx.needs_input_grad[1] or ctx.needs_input_grad[2] else None
        db2 = torch.empty(3, device=h.device, dtype=torch.float32) if dw2 is not None else None
        _lib.call('hk_mge_gate_bwd', h, w2, pr, c0, c1, c2, _f32c(dout), None if dpr is None else _f32c(dpr), dz, dh, dw2, db2,
                  N, F, K, _lib.stream_ptr())
        return dh, dw2, db2, None, None, None
