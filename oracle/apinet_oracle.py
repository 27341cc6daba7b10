"""fp64 restatements of APINet (reference model/methods/APINet.py, model/loss/APINet_loss.py) for the tests: pair mining with
numpy's argmin semantics, the pair head with given dropout masks, the loss, and the library's dropout hash bit for bit."""
import numpy as np
import torch
import torch.nn.functional as F

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def dropout_keep(seed, call, shape, p):
    """The keep mask of hk_dropout_* / hk_apinet_gate_*: splitmix64 output number (call << 40 | i) + 1 of the stream seeded
    with ``seed``; kept when its top 24 bits, as a fraction of 2^24, are >= p (compared in fp32, as on the device)."""
    n = int(np.prod(shape))
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over='ignore'):
        c = (np.uint64(call) << np.uint64(40)) | i
        z = np.uint64(np.int64(seed).astype(np.uint64)) + (c + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    u = (z >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
    return (u >= np.float32(p)).reshape(shape)


def pair_distances(pool):
    """pdist (APINet.py:116-119) in fp64: -2 <x_i, x_j> + |x_j|^2 + |x_i|^2."""
    x = torch.as_tensor(pool).double()
    sq = (x * x).sum(1)
    return -2 * x @ x.T + sq.view(1, -1) + sq.view(-1, 1)


def apinet_pairs(pool, labels, dist=None):
    """get_pairs (APINet.py:76-113) with numpy's argmin: -> (intra [n], inter [n], dist [n, n]) — ties to the lowest index,
    a row without candidates gets 0."""
    d = (pair_distances(pool) if dist is None else torch.as_tensor(dist).double()).numpy()
    lab = np.asarray(labels).reshape(-1, 1)
    same = lab == lab.T
    np.fill_diagonal(same, False)
    ds = np.where(same, d, np.inf)
    diff = lab != lab.T
    dd = np.where(diff, d, np.inf)
    return np.argmin(ds, axis=1), np.argmin(dd, axis=1), d


def apinet_head(pool, intra, inter, st, masks=None, p=0.5):
    """pool [n, D] -> (feats [8n, D] = [f1_self; f2_self; f1_other; f2_other], logits [8n, K]) in fp64 (APINet.py:36-69).
    ``st`` holds map1 / map2 / fc weights under the state_dict names; ``masks`` (optional) = the five keep masks in call order
    (map1 output, f1_self, f1_other, f2_self, f2_other), applied with scale 1 / (1 - p)."""
    x = torch.as_tensor(pool).double()
    n = x.shape[0]
    w = {k: torch.as_tensor(v).double() for k, v in st.items()}
    idx1 = torch.cat([torch.arange(n), torch.arange(n)])
    idx2 = torch.cat([torch.as_tensor(intra), torch.as_tensor(inter)]).long()
    f1, f2 = x[idx1], x[idx2]
    scale = 1.0 / (1.0 - p)

    def drop(t, k):
        return t if masks is None else t * torch.as_tensor(masks[k]).double() * scale

    h = drop(torch.cat([f1, f2], 1) @ w['map1.weight'].T + w['map1.bias'], 0)
    m = h @ w['map2.weight'].T + w['map2.bias']
    g1, g2 = torch.sigmoid(m * f1), torch.sigmoid(m * f2)
    f1s, f1o = drop(g1 * f1 + f1, 1), drop(g2 * f1 + f1, 2)
    f2s, f2o = drop(g2 * f2 + f2, 3), drop(g1 * f2 + f2, 4)
    feats = torch.cat([f1s, f2s, f1o, f2o], 0)
    return feats, feats @ w['fc.weight'].T + w['fc.bias']


def apinet_loss(logits, targets, margin=0.05, smoothing=0.1):
    """APINet_loss.py:26-39 in fp64: CE(label_smoothing) over all 8n rows + MarginRankingLoss between the target's softmax
    score under the self rows (first half) and the other rows (second half)."""
    z = torch.as_tensor(logits).double()
    t = torch.as_tensor(targets).long()
    ce = F.cross_entropy(z, t, label_smoothing=smoothing)
    R = z.shape[0] // 2
    sc = torch.softmax(z, 1).gather(1, t.view(-1, 1)).view(-1)
    rank = torch.clamp_min(sc[R:] - sc[:R] + margin, 0).mean()
    return ce + rank
