"""CPU restatement of MGE-CNN's method-specific pieces (reference model/methods/MGE_CNN/MGE.py, grad_cam.py), in numpy:
the closed-form Grad-CAM weights, get_bbox's box (in float32 with ATen's upsample_bilinear2d arithmetic, so thresholds
fall where the reference's fall), the conv6* part head with its max position and gradient, the detached concatenation and
the gate (in float64)."""
import numpy as np

f32 = np.float32


def gradcam_weights(w_main, idx, hw):
    """GradCam's layer weights (grad_cam.py:65-90) in closed form: the gradient at the hooked layer4 output of
    logits[idx] = W[idx] . mean_p(x_p) + b is W[idx] / HW at every position -> relu(W[idx]) / HW, [N, C]."""
    return np.maximum(np.asarray(w_main, dtype=np.float64)[np.asarray(idx)], 0) / hw


def _taps(n_in, S):
    """upsample_bilinear2d (align_corners=True) taps of each output index with ATen's float32 arithmetic."""
    scale = f32(n_in - 1) / f32(S - 1) if S > 1 else f32(0)
    src = (scale * np.arange(S, dtype=f32)).astype(f32)
    i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
    lam = np.clip((src - i0.astype(f32)).astype(f32), f32(0), f32(1)).astype(f32)
    i1 = i0 + (i0 < n_in - 1)
    return i0, i1, (f32(1) - lam).astype(f32), lam


def upsample(cam, S):
    """cam float32 [h, w] -> [S, S]: (v00 w0 + v01 w1) h0 + (v10 w0 + v11 w1) h1, each step rounded to float32."""
    cam = np.asarray(cam, dtype=f32)
    y0, y1, h0, h1 = _taps(cam.shape[0], S)
    x0, x1, w0, w1 = _taps(cam.shape[1], S)
    top = (cam[y0][:, x0] * w0[None]).astype(f32) + (cam[y0][:, x1] * w1[None]).astype(f32)
    bot = (cam[y1][:, x0] * w0[None]).astype(f32) + (cam[y1][:, x1] * w1[None]).astype(f32)
    return ((top * h0[:, None]).astype(f32) + (bot * h1[:, None]).astype(f32)).astype(f32)


def cam_box(conv5, weights, rate, S):
    """get_bbox (MGE.py:48-72): conv5 [N, C, h, w], weights [N, C] -> boxes int [N, 4] (y0, x0, y1, x1), end exclusive, as
    the crop reads them: the extents of the kept pixels, or (0, 0, S, S) for a box of zero height or width.  The CAM is
    summed in float64 and rounded once (exact for integer maps with power-of-two weights)."""
    conv5, weights = np.asarray(conv5, dtype=np.float64), np.asarray(weights, dtype=np.float64)
    out = np.zeros((conv5.shape[0], 4), dtype=np.int64)
    for n in range(conv5.shape[0]):
        cam = (conv5[n] * weights[n][:, None, None]).sum(0).astype(f32)
        m = upsample(cam, S)
        lo, hi = m.min(), m.max()
        with np.errstate(invalid='ignore', divide='ignore'):
            nm = ((m - lo).astype(f32) / f32(hi - lo)).astype(f32)
        keep = ~(nm < f32(rate))                    # sign(sign(m - rate) + 1): NaN is kept
        rows, cols = np.nonzero(keep)
        if len(rows) == 0 or rows.min() == rows.max() or cols.min() == cols.max():
            out[n] = (0, 0, S, S)
        else:
            out[n] = (rows.min(), cols.min(), rows.max(), cols.max())
    return out


def part_head(x, w, b):
    """pool_max(relu(conv6(x))) with Conv2d(C, O, 1, 1, padding 1): x [N, H, W, C] (NHWC), w [O, C], b [O] ->
    (pooled [N, O], pos [N, O]: the first interior argmax in row-major order, or -1 when the border's relu(b) wins ties
    included)."""
    x, w, b = (np.asarray(t, dtype=np.float64) for t in (x, w, b))
    N, H, W, C = x.shape
    y = x.reshape(N, H * W, C) @ w.T + b                       # [N, HW, O]
    inner = np.maximum(y.max(1), 0)
    arg = y.argmax(1)
    border = np.maximum(b, 0)[None]
    pooled = np.where(border >= inner, border, inner)
    pos = np.where(border >= inner, -1, arg)
    return pooled, pos


def part_head_bwd(x, pos, pooled, g):
    """-> (dw [O, C], db [O]) of the part head: the gradient reaches the winning pixel only, nothing for the border."""
    x, g = np.asarray(x, dtype=np.float64), np.asarray(g, dtype=np.float64)
    N, H, W, C = x.shape
    xf = x.reshape(N, H * W, C)
    gm = g * (pooled > 0)
    dw = np.zeros((g.shape[1], C))
    for n in range(N):
        inner = pos[n] >= 0
        dw[inner] += gm[n, inner, None] * xf[n, pos[n, inner]]
    return dw, gm.sum(0)


def cat_l2n(a, b, scale=10.0):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.concatenate([scale * a / np.linalg.norm(a, axis=1, keepdims=True),
                           scale * b / np.linalg.norm(b, axis=1, keepdims=True)], 1)


def gate(h, w2, b2, cats):
    """cls_gate[1], softmax, gated sum -> (out [N, K], pr [N, 3])."""
    z = np.asarray(h, dtype=np.float64) @ np.asarray(w2, dtype=np.float64).T + np.asarray(b2, dtype=np.float64)
    e = np.exp(z - z.max(1, keepdims=True))
    pr = e / e.sum(1, keepdims=True)
    c = np.stack([np.asarray(t, dtype=np.float64) for t in cats], -1)
    return (c * pr[:, None]).sum(-1), pr


def gate_bwd(h, w2, pr, cats, dout):
    """-> (dz [N, 3], dh [N, F], dw2 [3, F], db2 [3])."""
    c = np.stack([np.asarray(t, dtype=np.float64) for t in cats], -1)
    d = (np.asarray(dout, dtype=np.float64)[..., None] * c).sum(1)
    dz = pr * (d - (pr * d).sum(1, keepdims=True))
    h = np.asarray(h, dtype=np.float64)
    return dz, dz @ np.asarray(w2, dtype=np.float64), dz.T @ h, dz.sum(0)
