"""The oracle's restatement of the MAMC / N-pairs loss (model/loss/MAMC_loss.py) against reference-generated fixtures, and the
closed form the CUDA kernel uses (sum_k exp(n_k - p_j) = exp(-p_j) sum_k exp(n_k)) against the oracle — CPU only."""
import os

import numpy as np
import pytest
import torch

from oracle import hop_oracle as O

from conftest import load_golden  # noqa: E402

G = load_golden('reference_cin')
TAGS = ['npair_b8_p2', 'npair_b12_p3', 'npair_b6_p2_allsame', 'npair_b4_p2_alldiff']


@pytest.mark.parametrize('tag', TAGS)
def test_oracle_npairs_matches_reference(tag):
    f = torch.from_numpy(G[f'{tag}_feats']).double().requires_grad_(True)
    lab = torch.from_numpy(G[f'{tag}_labels'])
    loss = O.npairs_loss(f, lab)
    loss.backward()
    assert abs(loss.item() - float(G[f'{tag}_loss'])) < 1e-5 * max(1.0, abs(float(G[f'{tag}_loss'])))
    ref = torch.from_numpy(G[f'{tag}_dfeats']).double()
    assert (f.grad - ref).norm() <= 1e-4 * ref.norm() + 1e-9


def test_oracle_mamc_matches_reference():
    pred = torch.from_numpy(G['mamc_pred']).double().requires_grad_(True)
    parts = torch.from_numpy(G['mamc_parts']).double().requires_grad_(True)
    loss = O.mamc_loss(pred, parts, torch.from_numpy(G['mamc_labels']))
    loss.backward()
    assert abs(loss.item() - float(G['mamc_loss'])) < 1e-5
    for g, k in ((pred.grad, 'mamc_dpred'), (parts.grad, 'mamc_dparts')):
        ref = torch.from_numpy(G[k]).double()
        assert (g - ref).norm() <= 1e-4 * ref.norm()


@pytest.mark.parametrize('tag', TAGS)
def test_closed_form_equals_loop(tag):
    """what npair_fwd_bwd_kernel evaluates: per anchor E_A = sum over non-(same attention, same class) of exp(prod),
    E_B = sum over (different attention, different class); loss = sum_pos log1p(E exp(-p))."""
    f = torch.from_numpy(G[f'{tag}_feats']).double()
    lab = torch.from_numpy(G[f'{tag}_labels'])
    b, p, _ = f.shape
    n = b * p
    x = torch.nn.functional.normalize(f.reshape(n, -1), dim=1)
    prod = x @ x.t()
    cls, part = lab.repeat_interleave(p), torch.arange(p).repeat(b)
    sc, sa = cls[:, None] == cls[None, :], part[:, None] == part[None, :]
    typ = (~sa).long() * 2 + (~sc).long()
    e = torch.exp(prod)
    EA = (e * (typ != 0)).sum(1, keepdim=True)
    EB = (e * (typ == 3)).sum(1, keepdim=True)
    E = torch.where(typ == 0, EA, EB)
    loss = (torch.log1p(E * torch.exp(-prod)) * (typ != 3)).sum() / n
    assert abs(loss.item() - O.npairs_loss(f, lab).item()) < 1e-10
