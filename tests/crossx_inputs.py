"""Deterministic inputs of the CrossX fixtures (tests/golden/make_golden_crossx.py) and tests: logits and pooled part
features for the loss, and the batch-4 448x448 model step."""
import torch

import detgen

K = 200
GAMMA = (0.5, 0.25, 0.5)
LOSS_CASES = ((2, 2), (2, 8), (3, 2), (3, 8))       # (P, N)
CU, CP = 2048, 1024
NET_B, NET_P, NET_IMAGE = 4, 2, 448
NET_BN_MOMENTUM = 1.0     # the eval step normalises with the train step's batch statistics


def loss_inputs(P, N, seed=8000):
    """-> (xf, xp, xc [N, K], fu [N, P, 2048], fp [N, P, 1024], fc [N, P, 1024], labels).  Features are positive (they
    are pooled ReLU maps in the model), the cmbn ones signed (no ReLU after bn3_i)."""
    xs = [detgen.det((N, K), seed + i, 2.0) for i in range(3)]
    fu = detgen.det((N, P, CU), seed + 3, positive=True)
    fp = detgen.det((N, P, CP), seed + 4, positive=True)
    fc = detgen.det((N, P, CP), seed + 5)
    labels = detgen.det_labels(N, K, seed + 6)
    return (*xs, fu, fp, fc, labels)


def net_labels():
    return torch.tensor([5, 17, 5, 101], dtype=torch.int64)


def net_image():
    return detgen.det((NET_B, 3, NET_IMAGE, NET_IMAGE), 8100)
