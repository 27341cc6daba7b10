"""fp64 restatement of ProtoTree (reference model/methods/ProtoTree/, Examples/ProtoTreeNet.py) for the tests: distances
summed directly, the tree walked node by node in pre-order, the NLL, and the derivative-free leaf update.  Differentiable
with torch autograd, so the tests take gradients from it.  Prototype row k belongs to the k-th branch in pre-order."""
import torch


def layout(height):
    """-> list of (node index, depth, kind, left, right) in pre-order; kind 'b' (branch) or 'l' (leaf)."""
    nodes = []

    def walk(i, d):
        if d == height:
            nodes.append((i, d, 'l', None, None))
            return 1
        slot = len(nodes)
        nodes.append(None)
        left = walk(i + 1, d + 1)
        right = walk(i + 1 + left, d + 1)
        nodes[slot] = (i, d, 'b', i + 1, i + 1 + left)
        return 1 + left + right

    walk(0, 0)
    return nodes


def distances(z, protos):
    """z [N, HW, D], protos [P, D] -> (mind [N, P], argmin [N, P]): min over positions of sqrt(sum (z - p)^2 + 1e-14), the
    first minimising position on ties."""
    d = torch.sqrt(((z[:, :, None, :] - protos[None, None]) ** 2).sum(-1) + 1e-14)      # [N, HW, P]
    mind = d.min(dim=1).values
    hit = d == mind[:, None, :]
    HW = z.shape[1]
    first = torch.where(hit, torch.arange(HW)[None, :, None], torch.full_like(hit, HW, dtype=torch.long)).min(dim=1).values
    return mind, first


def route(mind, theta, height):
    """mind [N, P], theta [L, K] -> (pred [N, K], ps [N, P] by branch rank, pa [N, nodes] by node index)."""
    nodes = layout(height)
    N = mind.shape[0]
    ps = torch.exp(-mind)
    sm = torch.softmax(theta - theta.max(dim=1, keepdim=True).values, dim=1)
    pa = [None] * len(nodes)
    pa[0] = torch.ones(N, dtype=mind.dtype)
    rank = {}
    leaf = {}
    for i, _, kind, _, _ in nodes:
        (rank if kind == 'b' else leaf)[i] = len(rank if kind == 'b' else leaf)
    pred = 0
    for i, _, kind, left, right in nodes:
        if kind == 'b':
            p = ps[:, rank[i]]
            pa[left] = (1 - p) * pa[i]
            pa[right] = p * pa[i]
        else:
            pred = pred + pa[i][:, None] * sm[leaf[i]][None]
    return pred, ps, torch.stack(pa, 1)


def leaf_indices(height):
    return [i for i, _, kind, _, _ in layout(height) if kind == 'l']


def nll(pred, labels):
    """F.nll_loss(torch.log(pred), labels)."""
    return -torch.log(pred[torch.arange(pred.shape[0]), torch.as_tensor(labels).long()]).mean()


def leaf_update(theta, theta0, pa_leaves, pred, labels, num_batches):
    """Examples/ProtoTreeNet.py:116-132 on every leaf: theta [L, K], pa_leaves [N, L] -> the updated theta."""
    K = theta.shape[1]
    sm = torch.softmax(theta - theta.max(dim=1, keepdim=True).values, dim=1)
    target = torch.nn.functional.one_hot(torch.as_tensor(labels).long(), K).to(theta.dtype)
    update = torch.einsum('nl,lk,nk->lk', pa_leaves, sm, target / pred)
    return torch.relu(theta - theta0 / num_batches) + update
