"""Autograd bindings for AP-CNN (reference model/methods/APCNN.py): the feature pyramid's pieces, the pyramid attention
with its pooled outputs, the ROI selection, the ROI-guided refinement and the heads' vector ops.  Host plumbing only; all
arithmetic is in libhawkeye_b200.so.

The reference loops over the images on the host for the NMS (:458-474) and for the crops (:486-518), reading counts and
indices back for every image; here the per-image counts stay on the device next to fixed-shape boxes, so a training step
never synchronises."""
import numpy as np
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws, nhwc_channel_sum

STRIDES = (8, 16, 32)            # get_att_roi calls, :567-569
ANCHOR_SIZES = (64, 128, 256)
TOPK = (5, 3, 1)
IOU_THRESH = 0.05
ROI_OFFSETS = (0, 5, 8)          # first row of each level in the [N, 9, 4] box tensor
DROP_P3, DROP_P4 = 0.3, 0.6      # get_roi_crop_feat, :495 and :500


def suppression_table():
    """uint8 [3, 15, 15]: 1 where a candidate at cell offset (dy, dx) = (i - 7, j - 7) from a pick survives it.  The boxes
    of a level are equal squares of side ``size`` centred ``stride`` apart, so the outcome depends on the offset alone; it
    is computed with nms_pytorch's own float32 arithmetic (nms.py:26, :67-90: areas without +1, keep iff IoU < thresh).
    Offsets of 8 cells or more do not overlap and always survive."""
    out = np.ones((3, 15, 15), dtype=np.uint8)
    f = np.float32
    for l, (stride, size) in enumerate(zip(STRIDES, ANCHOR_SIZES)):
        area = f(size) * f(size)
        for i in range(15):
            for j in range(15):
                w = max(f(0), f(size) - f(abs(j - 7) * stride))
                h = max(f(0), f(size) - f(abs(i - 7) * stride))
                inter = f(w * h)
                iou = f(inter / f(f(area - inter) + area))
                out[l, i, j] = 1 if iou < f(IOU_THRESH) else 0
    return out


def central_windows(h3, w3, num_classes):
    """int32 [3, 4] (y0, y1, x0, x1) of each level's central window, with the reference's int(0.2 h) arithmetic (:451-454)."""
    lo, hi = (0.2, 0.8) if num_classes == 200 else (0.1, 0.9)
    return np.array([[int(lo * (h3 >> l)), int(hi * (h3 >> l)), int(lo * (w3 >> l)), int(hi * (w3 >> l))] for l in range(3)],
                    dtype=np.int32)


def roi_to_reference(boxes, counts):
    """The reference's roi_list from the fixed-shape tensors: three float [R_l, 5] tensors (image index, x1, y1, x2, y2),
    images in order, without the sixth column (the gate value of the pick) the reference's rows carry and never read.
    Reads the counts on the host: for tests and visualisation, not for the training step."""
    boxes, counts = boxes.detach().cpu(), counts.detach().cpu()
    out = []
    for l in range(3):
        rows = [torch.cat([torch.full((int(counts[n, l]), 1), float(n)), boxes[n, ROI_OFFSETS[l]:ROI_OFFSETS[l] + int(counts[n, l])]], 1)
                for n in range(boxes.shape[0])]
        out.append(torch.cat(rows, 0))
    return out


class BcastAddFn(Function):
    """a [N, H, W, C] + b [N, C] on every pixel (x_master + x_gpb, :197)."""

    @staticmethod
    def forward(ctx, a, b):
        _check_cuda(a, b)
        a, b = _f32c(a), _f32c(b)
        N, H, W, C = a.shape
        y = torch.empty_like(a)
        _lib.call('hk_apcnn_bcast', a, b, y, N, H * W, C, 1.0, _lib.stream_ptr())
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _f32c(dy)
        N, H, W, C = dy.shape
        return dy, nhwc_channel_sum(dy, N, H * W, C, 1.0)


class LateralFn(Function):
    """nearest-2x(top) + lat (:221-230); the backward is the 2x2 sum for top and the identity for lat."""

    @staticmethod
    def forward(ctx, top, lat):
        _check_cuda(top, lat)
        top, lat = _f32c(top), _f32c(lat)
        N, h, w, C = top.shape
        if tuple(lat.shape) != (N, 2 * h, 2 * w, C):
            raise _lib.HawkeyeLibError(f'APCNN lateral add: {tuple(lat.shape)} is not twice {tuple(top.shape)}')
        out = torch.empty_like(lat)
        _lib.call('hk_apcnn_lateral_fwd', top, lat, out, N, h, w, C, _lib.stream_ptr())
        ctx.shape = top.shape
        return out

    @staticmethod
    def backward(ctx, dout):
        dout = _f32c(dout)
        N, h, w, C = ctx.shape
        dtop = torch.empty(N, h, w, C, device=dout.device, dtype=torch.float32)
        _lib.call('hk_apcnn_lateral_bwd', dout, dtop, N, h, w, C, _lib.stream_ptr())
        return dtop, dout


class AttentionFn(Function):
    """F NHWC [N, H, W, 256], the SpatialGate's ConvTranspose2d weight [256, 1, 3, 3] and bias [1] ->
    (gate [N, H, W], mean_hw F [N, 256], mean_hw(gate F) [N, 256]).  The gate is not differentiable as an output."""

    @staticmethod
    def forward(ctx, F, w, b):
        _check_cuda(F, w, b)
        F, w = _f32c(F), _f32c(w)
        N, H, W, C = F.shape
        dev = F.device
        gate = torch.empty(N, H, W, device=dev, dtype=torch.float32)
        pf = torch.empty(N, C, device=dev, dtype=torch.float32)
        psf = torch.empty(N, C, device=dev, dtype=torch.float32)
        ws = _ws(_lib.query('hk_apcnn_att_workspace_bytes', N, H, W), dev)
        _lib.call('hk_apcnn_att_fwd', F, w, b, gate, pf, psf, N, H, W, C, ws, ws.numel(), _lib.stream_ptr())
        ctx.save_for_backward(F, w, gate)
        ctx.mark_non_differentiable(gate)
        ctx.set_materialize_grads(False)
        return gate, pf, psf

    @staticmethod
    def backward(ctx, _dgate, dpf, dpsf):
        F, w, gate = ctx.saved_tensors
        N, H, W, C = F.shape
        dev = F.device
        if dpsf is None:
            dpsf = torch.zeros(N, C, device=dev, dtype=torch.float32)
        dF = torch.empty_like(F)
        dw = torch.empty_like(w)
        db = torch.empty(1, device=dev, dtype=torch.float32)
        ws = _ws(_lib.query('hk_apcnn_att_workspace_bytes', N, H, W), dev)
        _lib.call('hk_apcnn_att_bwd', F, w, gate, None if dpf is None else _f32c(dpf), _f32c(dpsf), dF, dw, db, N, H, W, C, ws,
                  ws.numel(), _lib.stream_ptr())
        return dF, dw, db


class MixFn(Function):
    """z, pm, psf [3, N, C] (conv2 outputs of the three ChannelGates, mean F, mean gate F) -> v [3, N, C], the pooled attended
    maps mean_hw((gate_l + ch_l) F_l) with the bottom-up averaging of the channel gates (:256-266)."""

    @staticmethod
    def forward(ctx, z, pm, psf):
        _check_cuda(z, pm, psf)
        z, pm, psf = _f32c(z), _f32c(pm), _f32c(psf)
        _, N, C = z.shape
        v, ch = torch.empty_like(z), torch.empty_like(z)
        _lib.call('hk_apcnn_mix_fwd', z, pm, psf, v, ch, N, C, _lib.stream_ptr())
        ctx.save_for_backward(z, pm, ch)
        return v

    @staticmethod
    def backward(ctx, dv):
        z, pm, ch = ctx.saved_tensors
        dv = _f32c(dv)
        _, N, C = z.shape
        dz, dpm = torch.empty_like(z), torch.empty_like(z)
        _lib.call('hk_apcnn_mix_bwd', z, pm, ch, dv, dz, dpm, N, C, _lib.stream_ptr())
        return dz, dpm, dv


def roi_select(gates, windows, keep, img_h, img_w):
    """The three gates [N, H_l, W_l] -> (boxes fp32 [N, 9, 4], counts int32 [N, 3]); ``windows`` a host int32 [3, 4] tensor,
    ``keep`` the device copy of suppression_table().  No gradient."""
    g3, g4, g5 = (_f32c(g.detach()) for g in gates)
    _check_cuda(g3, g4, g5, keep)
    N, H3, W3 = g3.shape
    if tuple(g4.shape) != (N, H3 // 2, W3 // 2) or tuple(g5.shape) != (N, H3 // 4, W3 // 4) or H3 % 4 or W3 % 4:
        raise _lib.HawkeyeLibError(f'APCNN ROI selection: gates {tuple(g3.shape)}, {tuple(g4.shape)}, {tuple(g5.shape)} are not a '
                                   'stride-2 chain')
    boxes = torch.empty(N, 9, 4, device=g3.device, dtype=torch.float32)
    counts = torch.empty(N, 3, device=g3.device, dtype=torch.int32)
    _lib.call('hk_apcnn_roi', g3, g4, g5, windows, keep, boxes, counts, N, H3, W3, img_h, img_w, _lib.stream_ptr())
    return boxes, counts


class RefineFn(Function):
    """get_roi_crop_feat (:478-531) on the NHWC layer2 map: x [N, H, W, C], boxes, counts, draws [N, 2] or None (eval mode)."""

    @staticmethod
    def forward(ctx, x, boxes, counts, draws):
        _check_cuda(x, boxes, counts, draws)
        x = _f32c(x)
        N, H, W, C = x.shape
        y = torch.empty_like(x)
        meta = torch.empty(N, 12, device=x.device, dtype=torch.int32)
        _lib.call('hk_apcnn_refine_fwd', x, boxes, counts, None if draws is None else _f32c(draws), y, meta, N, H, W, C,
                  _lib.stream_ptr())
        ctx.save_for_backward(meta)
        return y

    @staticmethod
    def backward(ctx, dy):
        (meta,) = ctx.saved_tensors
        dy = _f32c(dy)
        N, H, W, C = dy.shape
        dx = torch.empty_like(dy)
        _lib.call('hk_apcnn_refine_bwd', dy, meta, dx, N, H, W, C, _lib.stream_ptr())
        return dx, None, None, None


def mask_cat(gates):
    g3, g4, g5 = (_f32c(g.detach()) for g in gates)
    N, H3, W3 = g3.shape
    out = torch.empty(N, 3, H3, W3, device=g3.device, dtype=torch.float32)
    _lib.call('hk_apcnn_mask_cat', g3, g4, g5, out, N, H3, W3, _lib.stream_ptr())
    return out
