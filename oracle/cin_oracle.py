"""CPU restatement of CIN's loss (reference model/loss/CIN_loss.py) in float64 numpy, with its gradients.

loss = CE_ls(Z, target) + alpha (L1 + L1^2), L1 = sum over the pairs i < B/2 with target[i] == target[B/2] of
||h(X_i) - h(X_{B/2+i}) + 1e-6||^2, h(x) = x W^T + b, X = Z_CCI viewed [B, F].  The reference's beta hinge is overwritten
by L1^2 and appears nowhere.  In float64 the bias cancels exactly, so the projection is taken of the difference."""
import numpy as np

PAIRWISE_EPS = 1e-6


def pair_mask(target):
    """target[:B/2] == target[B/2] (CIN_loss.py:39)"""
    target = np.asarray(target)
    return target[:len(target) // 2] == target[len(target) // 2]


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


def contrastive(z_cci, target, weight, alpha):
    """-> (term, L1, pairs, dz_cci, dweight, dbias): alpha (L1 + L1^2) and its gradients (dbias is zero)."""
    x = np.asarray(z_cci, dtype=np.float64).reshape(len(target), -1)
    w = np.asarray(weight, dtype=np.float64)
    half = len(target) // 2
    d = x[:half] - x[half:]
    v = d @ w.T + PAIRWISE_EPS
    m = pair_mask(target)
    l1 = float((v[m] ** 2).sum())
    dv = np.where(m[:, None], alpha * (1 + 2 * l1) * 2 * v, 0.0)
    dd = dv @ w
    dz = np.concatenate([dd, -dd]).reshape(np.shape(z_cci))
    return alpha * (l1 + l1 * l1), l1, int(m.sum()), dz, dv.T @ d, np.zeros(w.shape[0])


def cin_loss(z, z_cci, target, weight, alpha, smoothing=0.1):
    """-> (loss, dz, dz_cci, dweight, dbias) of CINLoss on the training output (Z, Z_CCI)"""
    target = np.asarray(target)
    ce, dz = ce_ls(z, target, smoothing)
    term, _, _, dz_cci, dw, db = contrastive(z_cci, target, weight, alpha)
    return ce + term, dz, dz_cci, dw, db
