"""fp64 restatement of DCL's head, stacked classifiers and loss (reference model/methods/DCL.py:31-45,
model/loss/DCL_loss.py:16-21) in plain torch, for the GPU tests and the fixture checks.  Inputs may be numpy arrays or
tensors; everything is promoted to float64, so autograd through these functions gives the fp64 gradients."""
import torch
import torch.nn.functional as F


def _d(t):
    return torch.as_tensor(t).double()


def head(x, w, b):
    """x [N, C, H, W], Convmask weight [1, C, 1, 1] (or [C]) and bias [1] -> (pooled [N, C], mask [N, (H/2)(W/2)])."""
    x = _d(x)
    z = torch.einsum('nchw,c->nhw', x, _d(w).reshape(-1)) + _d(b).reshape(())
    mask = torch.tanh(F.avg_pool2d(z[:, None], 2, stride=2)).flatten(1)
    return x.mean(dim=(2, 3)), mask


def classifiers(pooled, w, w2):
    """-> (logits [N, K], swap_logits [N, K2]), both bias-free."""
    p = _d(pooled)
    return p @ _d(w).T, p @ _d(w2).T


def _ce_ls(z, y, eps=0.1):
    logp = torch.log_softmax(z, dim=1)
    return ((1 - eps) * -logp.gather(1, y[:, None])[:, 0] + eps * -logp.mean(dim=1)).mean()


def loss(logits, swap_logits, mask, labels, labels_swap, law, alpha=1.0, beta=1.0, gamma=1.0):
    """alpha CE_ls(logits, labels) + beta CE_ls(swap_logits, labels_swap) + gamma mean |mask - law|, smoothing 0.1."""
    y, ys = torch.as_tensor(labels).long(), torch.as_tensor(labels_swap).long()
    return (alpha * _ce_ls(logits, y) + beta * _ce_ls(swap_logits, ys)
            + gamma * (_d(mask) - _d(law)).abs().mean())


def top1(logits, swap_logits, labels, cls_2xmul):
    """Top-1 hits, over logits + swap_logits[:, :K] + swap_logits[:, K:2K] under cls_2xmul (Examples/DCL.py:104-107)."""
    z = _d(logits)
    if cls_2xmul:
        K = z.shape[1]
        z = z + _d(swap_logits)[:, :K] + _d(swap_logits)[:, K:2 * K]
    return int((z.argmax(dim=1) == torch.as_tensor(labels).long()).sum())
