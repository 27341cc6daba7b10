"""A CPU restatement of Mixup / CutMix from a mix row (hawkeye_b200.ops_mixup), in numpy float32 with every product and
sum rounded on its own: the arithmetic hk_mix_batch and hk_softmax_ce_ls_mix are specified to do.  The CPU tests pin
it to the reference's outputs bit for bit; the GPU tests then hold the kernels to it."""
import numpy as np

from hawkeye_b200 import ops_mixup as M


def mix_images(img, row):
    """img float32 [B, C, H, W] -> the mixed batch: image i against image i - 1 mod B."""
    img = np.asarray(img, np.float32)
    prev = np.roll(img, 1, axis=0)
    if int(row[M.KIND]) == M.MIXUP:
        lam = float(row[M.LAMBDA])
        return np.float32(img * np.float32(lam)) + np.float32(prev * np.float32(1.0 - lam))
    x1, y1, x2, y2 = (int(v) for v in row[M.BOX:M.BOX + 4])
    out = img.copy()
    out[:, :, y1:y2, x1:x2] = prev[:, :, y1:y2, x1:x2]
    return out


def dense_target(label, row, num_classes):
    """int64 labels [B] -> the reference's float32 target w onehot(label) + (1 - w) onehot(rolled label)."""
    w = float(row[M.WEIGHT])
    onehot = np.eye(num_classes, dtype=np.float32)[np.asarray(label)]
    return np.float32(onehot * np.float32(w)) + np.float32(np.roll(onehot, 1, axis=0) * np.float32(1.0 - w))


def row_of(draw):
    """A fixture's recorded draw [kind, lambda, x1, y1, x2, y2, weight] -> the port's mix row."""
    d = np.asarray(draw, np.float64)
    return M.mix_row(int(d[0]), float(d[1]), tuple(d[2:6]), float(d[6])).numpy()
