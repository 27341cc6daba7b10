"""Seeded NMS score vectors shared by tests/golden/make_golden_nts.py and the NTS-Net tests, so the fixture carries the
reference's picks and not the scores."""
import numpy as np

NMS_VECTORS = 200               # per image size
NMS_TOPN = {224: 8, 448: 26}    # the survivor bound at each size: the deepest NMS the model allows


def quarter_pairs(anchors):
    """Ordered pairs (i, j), i != j, of anchors whose IoU is exactly 0.25 (4 inter == union on the integer boxes)."""
    a = anchors.astype(np.int64)
    dy = np.minimum(a[:, None, 2], a[None, :, 2]) - np.maximum(a[:, None, 0], a[None, :, 0])
    dx = np.minimum(a[:, None, 3], a[None, :, 3]) - np.maximum(a[:, None, 1], a[None, :, 1])
    inter = np.where((dy < 0) | (dx < 0), 0, dy * dx)
    area = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    i, j = np.nonzero(4 * inter == area[:, None] + area[None, :] - inter)
    keep = i != j
    return np.stack([i[keep], j[keep]], 1)


def nms_scores(anchors, k):
    """Score vector k (float32 [A], no two equal): a random permutation of 0.01 * range(A); odd k put a random IoU-0.25 pair
    at the top two places, so the tie of the threshold decides the second pick."""
    A = len(anchors)
    rs = np.random.RandomState(9000 + 17 * k + A)
    s = rs.permutation(A).astype(np.float32) * np.float32(0.01)
    if k % 2:
        pairs = quarter_pairs(anchors)
        i, j = pairs[rs.randint(len(pairs))]
        top = np.argsort(-s)[:2]
        s[[top[0], i]] = s[[i, top[0]]]
        top2 = np.argsort(-s)[1]
        s[[top2, j]] = s[[j, top2]]
    return s
