"""CPU restatement of Pairwise Confusion's loss (reference model/loss/pair_confusion.py) in float64 numpy, with its gradient.

loss = CE_ls(z, y) + lambda_a * sum_{i < B/2} [y_i != y_{B/2+i}] ||z_i - z_{B/2+i}|| / B, CE with mean reduction.  The
gradient of a pair term is +-(lambda_a / B) d / ||d|| on rows i and B/2 + i, and 0 where ||d|| = 0 (torch's norm backward)."""
import numpy as np


def ce_ls(z, target, smoothing=0.1):
    """CrossEntropyLoss(label_smoothing) with mean reduction -> (loss, dz)"""
    z = np.asarray(z, dtype=np.float64)
    B, K = z.shape
    m = z.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(z - m).sum(1))
    zy = z[np.arange(B), target]
    loss = ((1 - smoothing) * (lse - zy) + smoothing * (lse - z.mean(1))).mean()
    t = np.full((B, K), smoothing / K)
    t[np.arange(B), target] += 1 - smoothing
    return loss, (np.exp(z - lse[:, None]) - t) / B


def confusion(z, target):
    """-> (sum_i [y_i != y_{B/2+i}] ||d_i|| / B, its gradient dz, the number of pairs with differing labels)"""
    z = np.asarray(z, dtype=np.float64)
    target = np.asarray(target)
    B = z.shape[0]
    if B % 2:
        raise ValueError('Incorrect batch size provided')
    half = B // 2
    d = z[:half] - z[half:]
    n = np.sqrt((d * d).sum(1))
    m = (target[:half] != target[half:]) & (n > 0)
    g = np.where(m[:, None], d / np.where(n > 0, n, 1.0)[:, None], 0.0) / B
    return float(n[m].sum()) / B, np.concatenate([g, -g]), int((target[:half] != target[half:]).sum())


def pc_loss(z, target, lambda_a, smoothing=0.1):
    """-> (loss, dz) of PairwiseConfusionLoss"""
    target = np.asarray(target)
    ce, dce = ce_ls(z, target, smoothing)
    term, dterm, _ = confusion(z, target)
    return ce + lambda_a * term, dce + lambda_a * dterm
