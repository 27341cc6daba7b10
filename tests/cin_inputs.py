"""Inputs of CIN's loss fixtures (tests/golden/make_golden_cin_loss.py) at the shape the shipped config trains: batch 20
(4 classes x 5 images), Z_CCI [20, 2048, 49] (a 224x224 input), h: 100352 -> 512, 200 classes."""
import numpy as np
import torch

import detgen

B, C, WH, R, K = 20, 2048, 49, 512, 200
F = C * WH
ALPHA = 2.0
# Z_CCI's scale keeps L1 of order 1-10 with detgen's h, so that both L1 and L1^2 weigh in the loss
SCALE = 0.02
LABELS = {
    'balanced': np.repeat(np.arange(4), 5),                  # BalancedBatchSampler's 4 x 5 order: target[10] = 2, no pair
    'some': np.array([1, 0, 1, 2, 1, 3, 0, 1, 2, 3, 1, 0, 2, 3, 0, 1, 2, 3, 0, 2]),   # target[10] = 1: pairs 0, 2, 4, 7
    'allsame': np.zeros(B, dtype=np.int64),                  # every pair
}


def labels(name):
    return torch.from_numpy(LABELS[name].astype(np.int64))


def logits():
    return detgen.det((B, K), 6000)


def z_cci():
    return detgen.det((B, C, WH), 6001, SCALE)


def h_state():
    """detgen.state_like of a module holding h (the keys of CINLoss's state_dict: h.weight, h.bias)."""
    m = torch.nn.Module()
    m.h = torch.nn.Linear(F, R, device='meta')
    return detgen.state_like(m)
