"""fp64 restatement of S3N's sampler (reference model/methods/S3N.py:193-284: the class response maps' interpolation, top-5
and gate, the decision map, its peaks, the two sampling maps, create_grid and the warp) and of MultiSmoothLoss
(model/loss/S3N_loss.py), in plain torch, for the GPU tests and the fixture checks.  Inputs may be numpy arrays or tensors;
everything is promoted to float64, so autograd through these functions gives the fp64 gradients of radius, radius_inv and
the filter.  The peak search is a loop over images (a test size), as in the reference."""
import torch
import torch.nn.functional as F

GRID, PAD = 31, 30


def _d(t):
    return torch.as_tensor(t).double()


def interpolate_maps(crm):
    """crm [N, K, h, w] (the 1x1 conv's maps) -> [N, K, 31, 31], bilinear, align_corners=True (S3N.py:290-291)."""
    return F.interpolate(_d(crm), size=GRID, mode='bilinear', align_corners=True)


def decision_maps(maps31):
    """-> (normalised decision maps [N, 31, 31], top-5 class indices [N, 5], gate [N]) (S3N.py:197-212)."""
    maps31 = _d(maps31)
    prob = F.softmax(maps31.mean(dim=(2, 3)), dim=1)
    score, order = torch.sort(prob, dim=1, descending=True)
    gate = (score[:, :5] * torch.log(score[:, :5])).sum(1)
    out = []
    for n in range(maps31.shape[0]):
        m = maps31[n, order[n, 0]] if gate[n] > -0.2 else maps31[n, order[n, :5]].mean(0)
        out.append((m - m.min()) / (m.max() - m.min()))
    return torch.stack(out), order[:, :5], gate


def peaks(dm):
    """Peaks of one normalised map [31, 31]: the first maximum of the 3x3 window (-inf padding) that is >= the mean, in
    row-major order -> (positions [P] int64, scores [P])."""
    padded = F.pad(dm[None, None], (1, 1, 1, 1), value=float('-inf'))
    _, idx = F.max_pool2d(padded, 3, stride=1, return_indices=True)
    element = torch.arange(33 * 33).view(33, 33)[1:-1, 1:-1]
    is_peak = (idx[0, 0] == element) & (dm >= dm.mean())
    pos = torch.nonzero(is_peak.flatten())[:, 0]
    return pos, dm.flatten()[pos]


def gaussian(theta, pos):
    """kernel_generate(theta, 31, (x, y)) / its maximum: exp(-d^2 / (2 (31 theta)^2)), flattened [961]."""
    yy, xx = torch.meshgrid(torch.arange(GRID, dtype=torch.float64), torch.arange(GRID, dtype=torch.float64), indexing='ij')
    d2 = (xx - float(pos % GRID)) ** 2 + (yy - float(pos // GRID)) ** 2
    return torch.exp(-d2.flatten() / (2 * (theta * GRID) ** 2))


def assignment(pos, score, p, draws=None):
    """-> (to_zoom [P] bool, to_inv [P] bool) of S3N.py:226-258.  ``draws`` [961]: the uniform draw at each position (p=1)."""
    P = len(pos)
    if p == 0:
        return torch.ones(P, dtype=torch.bool), torch.ones(P, dtype=torch.bool)
    if p == 1:
        z = score > _d(draws)[pos]
        return z, ~z
    zoom, inv = torch.zeros(P, dtype=torch.bool), torch.zeros(P, dtype=torch.bool)
    s = score.tolist()
    zoom[s.index(max(s))] = True
    inv[s.index(min(s))] = True
    return zoom, inv


def sampling_maps(dms, p, radius, radius_inv, base_ratio, draws=None):
    """dms [N, 31, 31] normalised decision maps -> (xs [N, 961], xs_inv [N, 961], [(pos, score, zoom, inv)] per image);
    radius and radius_inv are 1-element tensors (pass ones that require grad for their gradients).  An image without peaks
    keeps base_ratio in both maps."""
    xs, xs_inv, recs = [], [], []
    for n in range(dms.shape[0]):
        dm = _d(dms[n])
        z = torch.full((GRID * GRID,), float(base_ratio), dtype=torch.float64) + 0 * radius.sum()
        c = torch.full((GRID * GRID,), float(base_ratio), dtype=torch.float64) + 0 * radius_inv.sum()
        if torch.isfinite(dm).all():
            pos, score = peaks(dm)
        else:
            pos, score = torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.float64)
        zoom, inv = assignment(pos, score, p, None if draws is None else draws[n]) if len(pos) else ([], [])
        for i in range(len(pos)):
            s, q = score[i], int(pos[i])
            if zoom[i]:
                z = z + s * gaussian(radius.reshape(()) * torch.sqrt(s), q)
            if inv[i]:
                c = c + (1 / s) * gaussian(radius_inv.reshape(()) * torch.sqrt(s), q)
        xs.append(z)
        xs_inv.append(c)
        recs.append((pos, score, zoom, inv))
    return torch.stack(xs), torch.stack(xs_inv), recs


def coarse_grid(maps, filt):
    """create_grid (S3N.py:156-183) before its F.interpolate: maps [B, 31, 31] (or [B, 961]), filter [61, 61] -> the
    31x31 grid [B, 31, 31, 2] (x, y)."""
    m = F.pad(_d(maps).reshape(-1, 1, GRID, GRID), (PAD,) * 4, mode='replicate')
    g = torch.arange(GRID + 2 * PAD, dtype=torch.float64)
    basis = (g - PAD) / (GRID - 1.0)
    px, py = basis.expand(GRID + 2 * PAD, -1), basis[:, None].expand(-1, GRID + 2 * PAD)
    w = _d(filt).reshape(1, 1, 2 * PAD + 1, 2 * PAD + 1)
    s0 = F.conv2d(m, w)
    sx = F.conv2d(m * px, w)
    sy = F.conv2d(m * py, w)
    gx = torch.clamp(sx / s0 * 2 - 1, min=-1, max=1)
    gy = torch.clamp(sy / s0 * 2 - 1, min=-1, max=1)
    return torch.cat([gx, gy], 1).permute(0, 2, 3, 1)


def fine_grid(coarse, size):
    """[B, 31, 31, 2] -> [B, size, size, 2], bilinear, align_corners=True (S3N.py:186)."""
    return F.interpolate(_d(coarse).permute(0, 3, 1, 2), size=(size, size), mode='bilinear',
                         align_corners=True).permute(0, 2, 3, 1)


def warp(x, coarse):
    """x [N, C, H, W], coarse grid [B, 31, 31, 2] -> image b % N sampled at the upsampled grid [B, C, H, W]."""
    x = _d(x)
    N, H = x.shape[0], x.shape[2]
    B = coarse.shape[0]
    xb = x[torch.arange(B) % N]
    return F.grid_sample(xb, fine_grid(coarse, H), mode='bilinear', padding_mode='zeros', align_corners=True)


def multi_smooth_loss(outputs, target, smooth_ratio, loss_weight=None):
    """MultiSmoothLoss (S3N_loss.py:15-37) in fp64."""
    target = torch.as_tensor(target).long()
    w = [1.0] * len(outputs)
    for k, v in (loss_weight or {}).items():
        w[int(k)] = v
    loss = 0
    for i, o in enumerate(outputs):
        o = _d(o)
        if i in (1, len(outputs) - 1):
            logp = F.log_softmax(o, dim=1)
            y = torch.zeros_like(logp).scatter_(1, target[:, None], 1)
            y = smooth_ratio * y + (1 - smooth_ratio) * (1 - y) / (o.shape[1] - 1)
            loss = loss - w[i] * (logp * y).sum(1).mean()
        else:
            loss = loss + w[i] * F.cross_entropy(o, target)
    return loss
