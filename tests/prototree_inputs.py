"""Inputs of the tree-only ProtoTree fixtures (tests/golden/make_golden_prototree.py), rebuilt from their detgen seeds, in
the package's order: prototype row k is the k-th branch in pre-order."""
import torch

import detgen


def tree_inputs(G, tag, N=4, S=7, K=200, D=256):
    seed = int(G[f'{tag}_seed'])
    perm = torch.as_tensor(G[f'{tag}_perm'])
    P = perm.numel()
    protos = (0.5 + 0.1 * detgen.det((P, D, 1, 1), seed))[perm]
    theta = torch.stack([detgen.det((K,), seed + 1 + j) for j in range(P + 1)])
    feat = torch.sigmoid(detgen.det((N, D, S, S), seed + 2000))
    labels = torch.as_tensor(G[f'{tag}_labels'])
    return feat, protos, theta, labels


def theta0(L, K=200):
    return torch.stack([(0.3 * detgen.det((K,), 3000 + j)).abs() for j in range(L)])
