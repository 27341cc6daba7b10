"""numpy restatements of AP-CNN's device-side pieces (reference model/methods/APCNN.py): the ROI selection with the tie rule
the kernel fixes, the ROI-guided refinement with explicit draws, the lateral add and the pooled form of the attended maps.
Test infrastructure only; nothing under hawkeye_b200/ imports it."""
import numpy as np

STRIDES, SIZES, TOPK, OFFSETS = (8, 16, 32), (64, 128, 256), (5, 3, 1), (0, 5, 8)


def nms_keep(size, stride, dy, dx, thresh=0.05):
    """True iff a box offset by (dy, dx) cells from a pick survives it: nms_pytorch's arithmetic in float32 (nms.py:67-90)."""
    f = np.float32
    w, h = max(f(0), f(size) - f(abs(dx) * stride)), max(f(0), f(size) - f(abs(dy) * stride))
    inter, area = f(w * h), f(size) * f(size)
    return bool(f(inter / f(f(area - inter) + area)) < f(thresh))


def roi_level(gate, level, num_classes, img_h, img_w):
    """gate [h, w] float32 -> (boxes [topk, 4] float32 with zeros past the count, count).  get_att_roi (:444-476) for one
    image; equal scores go to the highest flat index (a stable ascending argsort read from its end)."""
    h, w = gate.shape
    lo, hi = (0.2, 0.8) if num_classes == 200 else (0.1, 0.9)
    m = np.zeros_like(gate)
    m[int(lo * h):int(hi * h), int(lo * w):int(hi * w)] = gate[int(lo * h):int(hi * h), int(lo * w):int(hi * w)]
    s = m.reshape(-1)
    mean = np.float32(s.astype(np.float64).sum() / s.size)
    order = [int(i) for i in np.argsort(s, kind='stable') if s[i] > mean]
    stride, size = STRIDES[level], SIZES[level]
    boxes = np.zeros((TOPK[level], 4), dtype=np.float32)
    n = 0
    while order and n < TOPK[level]:
        p = order.pop()
        py, px = divmod(p, w)
        boxes[n] = (max(px * stride - size / 2, 0), max(py * stride - size / 2, 0), min(px * stride + size / 2, img_w - 1),
                    min(py * stride + size / 2, img_h - 1))
        n += 1
        order = [q for q in order if nms_keep(size, stride, q // w - py, q % w - px)]
    return boxes, n


def roi_select(gates, num_classes, img_h, img_w):
    """three [N, h, w] gates -> (boxes [N, 9, 4], counts [N, 3])."""
    N = gates[0].shape[0]
    boxes, counts = np.zeros((N, 9, 4), np.float32), np.zeros((N, 3), np.int32)
    for l in range(3):
        for n in range(N):
            b, c = roi_level(gates[l][n], l, num_classes, img_h, img_w)
            boxes[n, OFFSETS[l]:OFFSETS[l] + TOPK[l]], counts[n, l] = b, c
    return boxes, counts


def _axis(o, n_in, n_out):
    """ATen's align_corners=False source index in float32: (i0, i1, l0, l1)."""
    f = np.float32
    s = f(f(n_in) / f(n_out)) * f(f(o) + f(0.5)) - f(0.5)
    s = f(0) if s < 0 else s
    i0 = int(s)
    return i0, i0 + (1 if i0 < n_in - 1 else 0), f(1) - f(s - f(i0)), f(s - f(i0))


def refine(x, boxes, counts, draws):
    """x [N, C, H, W] float64, boxes [N, 9, 4], counts [N, 3], draws [N, 2] or None (eval) -> get_roi_crop_feat's output
    (:478-531).  draws[n] = (branch, fraction): branch < 0.3 drops level-3 ROI floor(fraction count), < 0.6 a level-4 ROI."""
    N, C, H, W = x.shape
    out = np.zeros_like(x)
    for n in range(N):
        rows = [boxes[n, OFFSETS[l] + t] / np.float32(8) for l in range(3) for t in range(counts[n, l])]
        r = np.array(rows, dtype=np.float32)
        xx1, yy1, xx2, yy2 = r[:, 0].min(), r[:, 1].min(), r[:, 2].max(), r[:, 3].max()
        X1, Y1, X2, Y2 = int(xx1), int(yy1), int(xx2), int(yy2)
        mask = np.ones((H, W))
        rate = 1.0
        if draws is not None:
            lv = 0 if draws[n, 0] < 0.3 else (1 if draws[n, 0] < 0.6 else -1)
            if lv >= 0 and counts[n, lv] > 0:
                t = min(int(np.float32(draws[n, 1]) * np.float32(counts[n, lv])), counts[n, lv] - 1)
                d = (boxes[n, OFFSETS[lv] + t] / np.float32(8)).astype(np.int64)
                mask[d[1]:d[3], d[0]:d[2]] = 0
            rate = float(np.float32(np.float32(yy2 - yy1) * np.float32(xx2 - xx1)) / np.float32(mask[Y1:Y2, X1:X2].sum()))
        crop = (x[n] * mask)[:, Y1:Y2, X1:X2] * rate
        ih, iw = crop.shape[1:]
        ys, xs = [_axis(o, ih, H) for o in range(H)], [_axis(o, iw, W) for o in range(W)]
        for oy, (h0, h1, a0, a1) in enumerate(ys):
            for ox, (w0, w1, b0, b1) in enumerate(xs):
                out[n, :, oy, ox] = (float(a0) * (float(b0) * crop[:, h0, w0] + float(b1) * crop[:, h0, w1]) +
                                     float(a1) * (float(b0) * crop[:, h1, w0] + float(b1) * crop[:, h1, w1]))
    return out


def lateral(top, lat):
    """nearest-2x(top) + lat on NCHW arrays (:221-230)."""
    return np.repeat(np.repeat(top, 2, axis=2), 2, axis=3) + lat


def attended_pool(F, gate, ch):
    """mean_hw((gate + ch) F) two ways, NCHW F [N, C, H, W], gate [N, 1, H, W], ch [N, C, 1, 1] -> (materialised, pooled form)."""
    return ((gate + ch) * F).mean((2, 3)), (gate * F).mean((2, 3)) + ch[:, :, 0, 0] * F.mean((2, 3))
