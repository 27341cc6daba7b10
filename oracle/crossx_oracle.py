"""CPU restatement of CrossX's new operations (reference model/methods/CrossX.py, model/loss/CrossX_loss.py) in float64
torch, gradients through autograd.  Maps are NHWC; part maps [N, HW, P, C].

* ``me``: out = relu(c + r), part p = relu(c sigmoid(m_p) + r) (Bottleneck.forward with meflag).
* ``fuse``: S = part + nearest-2x(R), the global max of the part and its first h-major position (AdaptiveMaxPool2d(1)).
* ``loss``: CrossXLoss in closed form: corr[i, j] = s_i . s_j / N^2 with s_i = sum_n xhat_i[n]; an all-zero feature row
  counts as 0 (the reference divides by its zero norm)."""
import torch


def _d(t):
    return torch.as_tensor(t).detach().double().clone().requires_grad_(True)


def me(c, r, m, dout, dparts):
    """c, r [N, HW, C], m [N, P, C], output gradients (dout may be None) -> (out, parts [N, HW, P, C], dc, dr, dm)"""
    c, r, m = _d(c), _d(r), _d(m)
    g = torch.sigmoid(m)[:, None]                                   # [N, 1, P, C]
    parts = torch.relu(c[:, :, None] * g + r[:, :, None])
    out = torch.relu(c + r)
    obj = (parts * torch.as_tensor(dparts).double()).sum()
    if dout is not None:
        obj = obj + (out * torch.as_tensor(dout).double()).sum()
    dc, dr, dm = torch.autograd.grad(obj, (c, r, m))
    return out.detach(), parts.detach(), dc, dr, dm


def fuse(parts, R, p, H, W):
    """parts [N, H*W, P, C], R [N, H/2 * W/2, C] -> (S [N, H*W, C], max [N, C], first argmax [N, C])"""
    x = torch.as_tensor(parts).double()[:, :, p]
    N, _, C = x.shape
    up = torch.as_tensor(R).double().view(N, H // 2, W // 2, C).repeat_interleave(2, 1).repeat_interleave(2, 2)
    mx, idx = x.max(1)
    first = (x == mx[:, None]).double().argmax(1)                   # first position of the maximum
    return x + up.reshape(N, H * W, C), mx, first


def fuse_bwd(dS, dmax, idx, H, W):
    """-> (dpart [N, HW, C], dR [N, HW/4, C])"""
    dS = torch.as_tensor(dS).double()
    N, HW, C = dS.shape
    dpart = dS.clone()
    dpart.scatter_add_(1, torch.as_tensor(idx).long()[:, None], torch.as_tensor(dmax).double()[:, None])
    dR = dS.view(N, H // 2, 2, W // 2, 2, C).sum((2, 4)).reshape(N, HW // 4, C)
    return dpart, dR


def _corr_reg(f, gamma, n_total=None, s_total=None):
    """gamma sum(triu(corr)) of features f [N, P, C] (autograd-able); s_total replaces the batch sums (another rank's
    share added), n_total the batch size behind them."""
    n = f.norm(dim=2, keepdim=True)
    xhat = torch.where(n > 0, f / torch.where(n > 0, n, torch.ones_like(n)), torch.zeros_like(f))
    s = xhat.sum(0)                                                   # [P, C]
    if s_total is not None:
        s = s + (s_total - s.detach())
    N2 = float(n_total or f.shape[0]) ** 2
    corr = s @ s.T / N2
    P = corr.shape[0]
    corr = torch.where(torch.eye(P, dtype=torch.bool), 1.0 - corr, corr)
    return gamma * torch.triu(corr).sum(), s.detach()


def loss(xf, xp, xc, fu, fp, fc, labels, gamma, smoothing=0.1):
    """-> (loss, (dxf, dxp, dxc, dfu, dfp, dfc)) of CrossXLoss with P > 1"""
    leaves = [_d(t) for t in (xf, xp, xc, fu, fp, fc)]
    xf, xp, xc, fu, fp, fc = leaves
    N = xf.shape[0]
    ce = torch.nn.functional.cross_entropy(xf + xp + xc, torch.as_tensor(labels), label_smoothing=smoothing)
    q = torch.softmax(xf, 1)
    kl = torch.nn.functional.kl_div(torch.log_softmax(xp, 1), q, reduction='sum') + \
        torch.nn.functional.kl_div(torch.log_softmax(xc, 1), q, reduction='sum')
    total = ce + kl / N
    for f, g in zip((fu, fp, fc), gamma):
        total = total + _corr_reg(f, g)[0]
    return total.item(), torch.autograd.grad(total, leaves)


def batch_sums(f):
    """[N, P, C] -> the batch sums of its L2-normalised rows [P, C]"""
    return _corr_reg(_d(f), 1.0)[1]
