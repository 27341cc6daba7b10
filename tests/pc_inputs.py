"""Deterministic inputs of the Pairwise Confusion fixtures (tests/golden/make_golden_pc.py) and tests: logits at the shipped
shape (batch 24, 200 classes) under four label patterns, and the batch-4 ResNet-50 step."""
import numpy as np
import torch

import detgen

B, K = 24, 200
LAMBDAS = (0.1, 10.0)
SCALE = 3.0
NET_B, NET_K, NET_IMAGE, NET_LAMBDA = 4, 200, 224, 10.0


def labels(name, B=B, K=K):
    """'differ': every pair (i, B/2 + i) has different labels; 'same': one label for the whole batch (the term is 0);
    'mix': pairs alternately equal and different; 'identical': as 'differ', with rows 0 and B/2 made identical by logits()."""
    half = B // 2
    if name in ('differ', 'identical'):
        y = np.arange(B) % K
    elif name == 'same':
        y = np.full(B, 3 % K)
    elif name == 'mix':
        first = np.arange(half) % K
        second = np.where(np.arange(half) % 2 == 0, first, (first + 1) % K)
        y = np.concatenate([first, second])
    else:
        raise KeyError(name)
    return torch.from_numpy(y.astype(np.int64))


NAMES = ('differ', 'same', 'mix', 'identical')


def logits(name, B=B, K=K, seed=7000):
    z = detgen.det((B, K), seed, SCALE)
    if name == 'identical':
        z[B // 2] = z[0]
    return z


def net_labels():
    """pair (0, 2) shares a label, pair (1, 3) does not"""
    return torch.tensor([5, 17, 5, 101], dtype=torch.int64)


def net_image():
    return detgen.det((NET_B, 3, NET_IMAGE, NET_IMAGE), 7100)
