"""fp64 CPU restatement of Interp-Parts' head (reference model/methods/Interp_Parts.py, model/loss/InterpParts_loss.py) for the
parity tests: the grouping unit, the part attention with the part sum, and the shaping loss, forward in torch so that
autograd gives the backward.  The distances are summed directly, sum_c (x - c)^2, as the package sums them."""
import torch
import torch.nn.functional as F


def grouping(x, w, smooth):
    """x [N, C, H, W], centres w [K, C, 1, 1] (or [K, C]), smooth [K] -> (out [N, K, C], assign [N, K, H, W]), :56-122."""
    N, C, H, W = x.shape
    c = w.reshape(w.shape[0], C)
    K = c.shape[0]
    xf = x.reshape(N, C, H * W).transpose(1, 2)                                 # [N, HW, C]
    d = ((xf[:, None, :, :] - c[None, :, None, :]) ** 2).sum(-1)                # [N, K, HW]
    beta = torch.sigmoid(smooth)
    assign = torch.softmax((-d).clamp(max=0.0) / beta[None, :, None], dim=1)
    qx = torch.bmm(assign, xf)                                                  # [N, K, C]
    s = assign.sum(2, keepdim=True).clamp(min=1e-5)
    sigma = (beta / 2).sqrt()
    out = (qx / s - c[None]) / sigma[None, :, None]
    return F.normalize(out, dim=2), assign.reshape(N, K, H, W)


def attention_pool(f, post, w, b, gamma, beta, running_mean, running_var, training, N, K, momentum=0.1, eps=1e-5):
    """f [N K, C], post [N K, D] -> (pooled [N, D], att [N, K], new running (mean, var)): Conv2d(C, 1) + BatchNorm(1) + ReLU,
    softmax over the parts, and the attention-weighted part sum (:289-291, :349-361)."""
    conv = f @ w.reshape(-1) + b.reshape(())
    if training:
        mean, var = conv.mean(), conv.var(unbiased=False)
        rm = (1 - momentum) * running_mean + momentum * mean.detach()
        rv = (1 - momentum) * running_var + momentum * conv.detach().var(unbiased=True)
    else:
        mean, var, rm, rv = running_mean, running_var, running_mean, running_var
    y = torch.relu((conv - mean) / torch.sqrt(var + eps) * gamma.reshape(()) + beta.reshape(()))
    att = torch.softmax(y.reshape(N, K), dim=1)
    pooled = (post.reshape(N, K, -1) * att[:, :, None]).sum(1)
    return pooled, att, (rm, rv)


def gaussian(radius, std):
    i = torch.arange(-radius, radius + 1, dtype=torch.float64)
    w = torch.exp(-(i[:, None] ** 2 + i[None, :] ** 2) / (2 * std * std))
    return w / w.sum()


def occupancy(assign, taps):
    """assign [N, K, H, W], taps [S, S] -> occ [N, K]: the max of the "valid" depthwise blur (:114-124)."""
    K, S = assign.shape[1], taps.shape[-1]
    blur = F.conv2d(assign, taps.reshape(1, 1, S, S).expand(K, 1, S, S).to(assign.dtype), groups=K)
    return blur.flatten(2).max(2).values


def shaping(occ, prior, eps=1e-5):
    """occ [R, K], prior [R] -> mean |log(sort(occ) + eps) - log(prior + eps)| (:125-138)."""
    emp, _ = occ.sort(dim=0)
    return ((emp + eps).log() - (prior.to(occ.dtype)[:, None] + eps).log()).abs().mean()
