"""Seeded inputs shared by tests/golden/make_golden_apcnn.py and the AP-CNN tests, so fixtures need not carry them."""
import numpy as np

ROI_IMAGE = 224                  # gate maps of 28x28, 14x14 and 7x7
ROI_BATCH = 6
E2E_IMAGE, E2E_BATCH, E2E_CLASSES = 160, 4, 12


def gates(num_classes, image=ROI_IMAGE, batch=ROI_BATCH):
    """Three float32 gate maps [batch, h, w] in (0, 1).  Images 0 and 1 are near zero with one and two far-apart peaks (fewer
    candidates than topk), the others are smooth random fields; no two cells of a map are equal."""
    out = []
    for l in range(3):
        h = image // (8 << l)
        rs = np.random.RandomState(4000 + 10 * l + (1 if num_classes == 200 else 0))
        z = rs.standard_normal((batch, h + 2, h + 2)).astype(np.float32)
        z = (z[:, :-2, :-2] + z[:, 1:-1, 1:-1] + z[:, 2:, 2:] + z[:, 1:-1, :-2] + z[:, :-2, 1:-1]) / np.float32(2.0)
        g = (1.0 / (1.0 + np.exp(-z.astype(np.float64)))).astype(np.float32)
        tiny = (np.float32(1e-4) * (np.float32(1) + g[:2])).astype(np.float32)      # distinct values, all below the mean
        g[:2] = tiny
        a, b = h * 2 // 7, h * 5 // 7
        g[0, a, a] = 0.75
        g[1, a, a] = 0.5
        g[1, b, b] = 0.625
        out.append(g)
    return out


def pad_rois(roi, batch, topk):
    """The reference's (image, x1, y1, x2, y2, score) rows -> (boxes [batch, topk, 4], counts [batch])."""
    roi = np.asarray(roi, dtype=np.float32)
    boxes = np.zeros((batch, topk, 4), dtype=np.float32)
    counts = np.zeros(batch, dtype=np.int32)
    for r in roi:
        n = int(r[0])
        boxes[n, counts[n]] = r[1:5]
        counts[n] += 1
    return boxes, counts


def e2e_state(net):
    """detgen.state_like weights with the spatial gates' weights scaled down, so that the gates of the end-to-end fixture are
    not saturated (saturated gates tie at 1.0 and the reference's picks then hang on its unstable argsort)."""
    import detgen
    sd = detgen.state_like(net)
    for k in sd:
        if k.startswith('apn.') and k.endswith('_1.conv.weight'):
            sd[k] = sd[k] * 0.01
    return sd
