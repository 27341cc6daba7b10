"""Autograd bindings for NTS-Net (reference model/methods/NTS_Net/NTSNet.py, anchors.py, model/loss/NTS_loss.py): the
navigator (proposal net, NMS and the gather of the kept scores) as one autograd node, the part crops, the trunk's dropout
and the ranking loss.  Host plumbing only; all arithmetic is in libhawkeye_b200.so.

The reference copies the proposal scores to the host for a numpy NMS and builds the part images with B x topN separate
F.interpolate calls (NTSNet.py:33-48); here both stay on the device, so a training step never synchronises."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, add_, conv3x3_dgrad, conv3x3_fwd, conv3x3_pack, conv3x3_wgrad, crop as _crop

PAD = 224                   # NTSNet.pad_side: the anchors live in the image zero-padded by 224 on every side (:26-27, :31)
PART_SIZE = 224             # every part image is resized to 224 x 224 (:43-48)
TIDY = (6, 6, 9)            # tidy1..3 outputs (ProposalNet, :70-72)
DROP_IMAGES, DROP_PARTS = 0, 1     # dropout call ids of the two trunk passes


def _down_fwd(x, wf, b, stride2):
    """relu(conv3x3(x) + b) at stride 1, or at stride 2 with ceil-mode output: the stride-1 map subsampled at the even
    positions, which is exactly nn.Conv2d(3, stride 2, padding 1) for even and odd maps alike."""
    y = conv3x3_fwd(x, wf, b, relu=True)
    if not stride2:
        return y
    N, H, W, C = y.shape
    ys = torch.empty(N, (H + 1) // 2, (W + 1) // 2, C, device=y.device, dtype=torch.float32)
    _lib.call('hk_subsample2', y, ys, N, H, W, C, _lib.stream_ptr())
    return ys


def _down_bwd(x, g, wd, stride2, need_dx):
    """g: gradient at the pre-activation of a down conv -> (dw, db, dx masked by x > 0, or None).  Stride 2 zero-inserts g
    to the input resolution first (the adjoint of the subsampling), as the trunk's 3x3s2 units do."""
    N, H, W, cin = x.shape
    cout = g.shape[-1]
    if stride2:
        gf = torch.empty(N, H, W, cout, device=g.device, dtype=torch.float32)
        _lib.call('hk_upsample2_zero', g, gf, N, H, W, cout, _lib.stream_ptr())
        g = gf
    dw = torch.empty(cout, cin, 3, 3, device=g.device, dtype=torch.float32)
    db = torch.empty(cout, device=g.device, dtype=torch.float32)
    conv3x3_wgrad(x, g, dw, db)
    return dw, db, (conv3x3_dgrad(g, wd, mask=x) if need_dx else None)


def nms(scores, anchors, topn):
    """hard_nms per image on the device: scores [B, A], anchors int32 [A, 4] -> (idx int64 [B, T], prob [B, T], boxes int32
    [B, T, 4]).  No gradient (``ProposalFn`` carries the gradient of prob)."""
    _check_cuda(scores, anchors)
    scores = _f32c(scores)
    B, A = scores.shape
    dev = scores.device
    idx = torch.empty(B, topn, device=dev, dtype=torch.int64)
    prob = torch.empty(B, topn, device=dev, dtype=torch.float32)
    boxes = torch.empty(B, topn, 4, device=dev, dtype=torch.int32)
    _lib.call('hk_nts_nms', scores, anchors.contiguous(), idx, prob, boxes, B, A, topn, _lib.stream_ptr())
    return idx, prob, boxes


class ProposalFn(Function):
    """ProposalNet on the detached layer4 map, the NMS and the gather (NTSNet.py:34-42) as one node.

    x NHWC [B, H, W, 2048] -> (rpn_score [B, A], top_n_prob [B, T], top_n_index int64 [B, T], boxes int32 [B, T, 4]).  Only
    top_n_prob is differentiable, as in the reference, where the gather is the one path by which a gradient reaches the
    proposal net: the backward reads the T kept scores per image (hk_nts_score_bwd), never a dense [B, A] gradient."""

    @staticmethod
    def forward(ctx, x, anchors, topn, save, w1, b1, w2, b2, w3, b3, t1w, t1b, t2w, t2b, t3w, t3b):
        _check_cuda(x, anchors, w1, w2, w3, t1w, t2w, t3w)
        x = _f32c(x)
        B, H1, W1, _ = x.shape
        s = _lib.stream_ptr()
        wf1, _ = conv3x3_pack(_f32c(w1), False)
        wf2, wd2 = conv3x3_pack(_f32c(w2), save)
        wf3, wd3 = conv3x3_pack(_f32c(w3), save)
        d1 = _down_fwd(x, wf1, b1, False)
        d2 = _down_fwd(d1, wf2, b2, True)
        d3 = _down_fwd(d2, wf3, b3, True)
        C = d1.shape[-1]
        tw = [_f32c(t).reshape(t.shape[0], C) for t in (t1w, t2w, t3w)]
        A = _lib.query('hk_nts_num_anchors', H1, W1)
        if anchors.shape[0] != A:
            raise _lib.HawkeyeLibError(f'NTSNet: a {H1}x{W1} layer4 map gives {A} scores, the model has {anchors.shape[0]} '
                                       'anchors (built for another image_size)')
        score = torch.empty(B, A, device=x.device, dtype=torch.float32)
        _lib.call('hk_nts_score_fwd', d1, d2, d3, tw[0], t1b, tw[1], t2b, tw[2], t3b, score, B, H1, W1, d2.shape[1],
                  d2.shape[2], d3.shape[1], d3.shape[2], C, s)
        idx, prob, boxes = nms(score, anchors, topn)
        ctx.mark_non_differentiable(score, idx, boxes)
        ctx.set_materialize_grads(False)
        ctx.rec = (x, d1, d2, d3, wd2, wd3, tw, idx) if save else None
        return score, prob, idx, boxes

    @staticmethod
    def backward(ctx, _dscore, dprob, _didx, _dboxes):
        if ctx.rec is None or dprob is None:
            return (None,) * 16
        x, d1, d2, d3, wd2, wd3, tw, idx = ctx.rec
        ctx.rec = None
        B, T = idx.shape
        dev, s = x.device, _lib.stream_ptr()
        g = [torch.empty_like(d) for d in (d1, d2, d3)]
        dt = [(torch.empty(a, C, 1, 1, device=dev, dtype=torch.float32), torch.empty(a, device=dev, dtype=torch.float32))
              for a, C in zip(TIDY, (d1.shape[-1],) * 3)]
        _lib.call('hk_nts_score_bwd', d1, d2, d3, tw[0], tw[1], tw[2], idx, _f32c(dprob), g[0], g[1], g[2], dt[0][0], dt[0][1],
                  dt[1][0], dt[1][1], dt[2][0], dt[2][1], B, T, d1.shape[1], d1.shape[2], d2.shape[1], d2.shape[2],
                  d3.shape[1], d3.shape[2], d1.shape[-1], s)
        dw3, db3, dx = _down_bwd(d2, g[2], wd3, True, True)
        add_(g[1], dx)
        dw2, db2, dx = _down_bwd(d1, g[1], wd2, True, True)
        add_(g[0], dx)
        dw1, db1, _ = _down_bwd(x, g[0], None, False, False)
        return (None, None, None, None, dw1, db1, dw2, db2, dw3, db3, dt[0][0], dt[0][1], dt[1][0], dt[1][1], dt[2][0],
                dt[2][1])


def proposal(x_nhwc, net, anchors, topn):
    """``net`` is a ProposalNet (down1..3, tidy1..3); -> (rpn_score, top_n_prob, top_n_index, boxes)."""
    params = [p for m in (net.down1, net.down2, net.down3, net.tidy1, net.tidy2, net.tidy3) for p in (m.weight, m.bias)]
    save = torch.is_grad_enabled() and any(p.requires_grad for p in params)
    return ProposalFn.apply(x_nhwc, anchors, topn, save, *params)


def crop(images, boxes, size=PART_SIZE, pad=PAD):
    """The part images of NTSNet.py:40-49 without a gradient (the reference detaches them, :50): images NCHW [B, C, H, W],
    boxes int32 [B, T, 4] in the padded image -> NCHW [B*T, C, size, size]."""
    return _crop(images, boxes, size, pad)


class DropoutFn(Function):
    """nn.Dropout(p) applied whatever the module's mode, as the reference's ``nn.Dropout(p=0.5)(x)`` (NTS_Net/resnet.py:148)
    is: a module built on every call, hence always in train mode.  The mask is a hash of the device seed and ``call``."""

    @staticmethod
    def forward(ctx, x, p, seed, call):
        x = _f32c(x)
        y = torch.empty_like(x)
        _lib.call('hk_dropout_fwd', x, y, x.numel(), float(p), seed, call, _lib.stream_ptr())
        ctx.p, ctx.seed, ctx.call = float(p), seed, call
        return y

    @staticmethod
    def backward(ctx, dy):
        dx = torch.empty_like(dy)
        _lib.call('hk_dropout_bwd', _f32c(dy), dx, dx.numel(), ctx.p, ctx.seed, ctx.call, _lib.stream_ptr())
        return dx, None, None, None


def dropout(x, p, seed, call):
    return x if p == 0 else DropoutFn.apply(x, p, seed, call)


class RankLossFn(Function):
    """part_logits [B*T, K], labels [B], top_n_prob [B, T] -> ranking_loss(top_n_prob, list_loss(part_logits)) (NTS_loss.py:
    32-47), differentiable in top_n_prob only."""

    @staticmethod
    def forward(ctx, part_logits, labels, prob):
        _check_cuda(part_logits, labels, prob)
        part_logits, prob = _f32c(part_logits), _f32c(prob)
        B, T = prob.shape
        K = part_logits.shape[-1]
        if part_logits.numel() != B * T * K:
            raise _lib.HawkeyeLibError(f'NTSLoss: {part_logits.numel() // K} part rows for {B} x {T} proposals')
        acc = torch.zeros(1, device=prob.device, dtype=torch.float64)
        dprob = torch.empty_like(prob)
        _lib.call('hk_nts_rank_loss', part_logits, labels.contiguous().to(torch.int64), prob, acc, dprob, B, T, K,
                  _lib.stream_ptr())
        ctx.save_for_backward(dprob)
        return acc[0].float()

    @staticmethod
    def backward(ctx, g):
        (dprob,) = ctx.saved_tensors
        return None, None, dprob * g
