"""fp64 CPU restatement of NTS-Net's navigator and losses (reference model/methods/NTS_Net/NTSNet.py, anchors.py,
model/loss/NTS_loss.py) for the tests: the greedy NMS, the pad + slice + bilinear resize of the part crops, the proposal
head, and the list and ranking losses.  Written from the reference's definitions, not copied from it.  The anchors are
checked against the reference's own values, recorded in tests/golden/reference_nts.*.npz."""
import numpy as np
import torch
import torch.nn.functional as F

IOU = 0.25


def hard_nms(scores, anchors, topn):
    """Indices kept by greedy NMS: visit candidates by descending score (lower index first on equal scores), keep one
    unless an already kept box has IoU >= 0.25 with it (float64 IoU of the integer boxes, overlap 0 when an extent is
    negative), stop after topn."""
    s = np.asarray(scores, dtype=np.float64)
    a = np.asarray(anchors, dtype=np.float64)
    order = np.lexsort((np.arange(len(s)), -s))
    area = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    kept = []
    for c in order:
        ok = True
        for k in kept:
            dy = min(a[c, 2], a[k, 2]) - max(a[c, 0], a[k, 0])
            dx = min(a[c, 3], a[k, 3]) - max(a[c, 1], a[k, 1])
            inter = 0.0 if (dy < 0 or dx < 0) else dy * dx
            if inter / (area[c] + area[k] - inter) >= IOU:
                ok = False
                break
        if ok:
            kept.append(int(c))
            if len(kept) == topn:
                break
    return np.array(kept, dtype=np.int64)


def decisive_gap(scores, anchors, topn):
    """The smallest score difference that decides a pick of hard_nms: at every round, the picked score minus the best
    score still alive after it.  A score error below half of this cannot change the picks."""
    s = np.asarray(scores, dtype=np.float64)
    a = np.asarray(anchors, dtype=np.float64)
    area = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    alive = np.ones(len(s), bool)
    gap = np.inf
    for _ in range(topn):
        cand = np.nonzero(alive)[0]
        if len(cand) < 2:
            break
        o = cand[np.argsort(-s[cand], kind='stable')]
        gap = min(gap, s[o[0]] - s[o[1]])
        p = o[0]
        dy = np.minimum(a[:, 2], a[p, 2]) - np.maximum(a[:, 0], a[p, 0])
        dx = np.minimum(a[:, 3], a[p, 3]) - np.maximum(a[:, 1], a[p, 1])
        inter = np.where((dy < 0) | (dx < 0), 0.0, dy * dx)
        alive &= inter / (area + area[p] - inter) < IOU
    return gap


def crop(images, boxes, size=224, pad=224):
    """images [B, C, H, W], boxes [B, T, 4] (y0, x0, y1, x1) in the image zero-padded by ``pad`` -> [B*T, C, size, size]:
    each window resized with bilinear interpolation on the align_corners=True grid (src = dst (in - 1) / (size - 1))."""
    x = torch.as_tensor(images, dtype=torch.float64)
    B, C, H, W = x.shape
    xp = torch.zeros(B, C, H + 2 * pad, W + 2 * pad, dtype=torch.float64)
    xp[:, :, pad:pad + H, pad:pad + W] = x
    out = []
    for n in range(B):
        for y0, x0, y1, x1 in np.asarray(boxes[n]).tolist():
            win = xp[n, :, y0:y1, x0:x1]
            h, w = win.shape[1:]
            sy = torch.arange(size, dtype=torch.float64) * ((h - 1) / (size - 1))
            sx = torch.arange(size, dtype=torch.float64) * ((w - 1) / (size - 1))
            iy0, ix0 = sy.floor().long().clamp(max=h - 1), sx.floor().long().clamp(max=w - 1)
            iy1, ix1 = (iy0 + 1).clamp(max=h - 1), (ix0 + 1).clamp(max=w - 1)
            ly, lx = (sy - iy0)[:, None], (sx - ix0)[None, :]
            top = win[:, iy0][:, :, ix0] * (1 - lx) + win[:, iy0][:, :, ix1] * lx
            bot = win[:, iy1][:, :, ix0] * (1 - lx) + win[:, iy1][:, :, ix1] * lx
            out.append(top * (1 - ly) + bot * ly)
    return torch.stack(out)


def proposal_scores(x, p):
    """Layer4 map x [B, 2048, H, W] and p = {down1..3, tidy1..3: (weight, bias)} -> scores [B, A] in the reference's order:
    ReLU(conv) at strides 1, 2, 2 (padding 1), then each tidy 1x1 conv flattened channel-major and concatenated."""
    d, outs = torch.as_tensor(x, dtype=torch.float64), []
    for k, stride in ((1, 1), (2, 2), (3, 2)):
        w, b = p[f'down{k}']
        d = F.relu(F.conv2d(d, w.double(), b.double(), stride=stride, padding=1))
        tw, tb = p[f'tidy{k}']
        outs.append(F.conv2d(d, tw.double(), tb.double()).flatten(1))
    return torch.cat(outs, 1)


def list_loss(part_logits, labels_rows):
    """per-row NLL of log_softmax: [R, K], [R] -> [R]"""
    return -F.log_softmax(torch.as_tensor(part_logits, dtype=torch.float64), -1).gather(
        1, torch.as_tensor(labels_rows).view(-1, 1)).view(-1)


def ranking_loss(prob, L):
    """sum over images n and pairs (i, j) of relu(1 - prob[n, i] + prob[n, j]) [L[n, j] > L[n, i]], over B."""
    prob = torch.as_tensor(prob, dtype=torch.float64)
    L = torch.as_tensor(L, dtype=torch.float64)
    worse = (L[:, None, :] > L[:, :, None]).double()                  # [n, i, j]: L_j > L_i
    return (F.relu(1 - prob[:, :, None] + prob[:, None, :]) * worse).sum() / prob.shape[0]


def nts_loss(raw, concat, part, prob, labels, ls=0.1):
    """NTSLoss: three label-smoothed cross-entropies (part rows averaged over B*T) + the ranking loss."""
    B, T = prob.shape
    rows = torch.as_tensor(labels).repeat_interleave(T)
    part2 = torch.as_tensor(part, dtype=torch.float64).reshape(B * T, -1)
    ce = sum(F.cross_entropy(torch.as_tensor(z, dtype=torch.float64), y, label_smoothing=ls)
             for z, y in ((raw, torch.as_tensor(labels)), (concat, torch.as_tensor(labels)), (part2, rows)))
    return ce + ranking_loss(prob, list_loss(part2, rows).view(B, T))
