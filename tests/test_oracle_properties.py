"""Size-independent properties of the CPU oracle (oracle/hop_oracle.py) — the same invariants the GPU tests check at the
benchmark sizes — plus cross-checks of its hand-written backward formulas against autograd in fp64."""
import numpy as np
import pytest
import torch

import detgen
from oracle import hop_oracle as O


@pytest.mark.parametrize('shape', [(2, 8, 3, 4), (1, 32, 5, 5), (3, 16, 2, 2)])
def test_bilinear_pool_invariants_and_backward(shape):
    x = detgen.det_uniform(shape, 3).double()
    y = O.bilinear_pool_fwd(x)
    B, C = shape[0], shape[1]
    Y = y.view(B, C, C)
    assert torch.allclose(y.norm(dim=1), torch.ones(B, dtype=torch.float64), atol=1e-12)      # F.normalize, BCNN.py:26
    assert torch.allclose(Y, Y.transpose(1, 2), atol=1e-14) and (y > 0).all()                  # Gram symmetry, sqrt(+eps)
    # hand-derived backward == autograd of the forward
    xg = x.clone().requires_grad_(True)
    dy = detgen.det(y.shape, 4).double()
    (dx_auto,) = torch.autograd.grad(O.bilinear_pool_fwd(xg), xg, dy)
    assert torch.allclose(O.bilinear_pool_bwd(x, dy), dx_auto, rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize('d', [16, 97, 256])
def test_cbp_fft_path_equals_gram_scatter(d):
    """CBCNN.py:114-133 (sketch, FFT, product, inverse FFT, spatial sum) == signed scatter of the Gram (DESIGN §4 CBP)."""
    x = detgen.det_uniform((2, 24, 3, 3), 9).double()
    hashes = O.cbp_hashes(24, d)
    pre = O.cbp_presqrt_gram_scatter(x, d, hashes)
    y = O.cbp_fwd(x, d, hashes)
    ref = torch.sign(pre) * torch.sqrt(pre.abs() + 1e-10)
    ref = ref / ref.norm(dim=1, keepdim=True).clamp_min(1e-12)
    # empty bins: the FFT path leaves ~1e-14 of round-off where the scatter has an exact 0, and sign(v) sqrt(|v| + 1e-10)
    # turns that into +-1e-5 before normalisation (the ill-conditioning of the signed sqrt) — hence the absolute tolerance
    assert torch.allclose(y.double(), ref, rtol=1e-6, atol=5e-6)
    h1, s1, h2, s2 = hashes
    assert (np.abs(s1) == 1).all() and (np.abs(s2) == 1).all() and h1.min() >= 0 and h1.max() < d and h2.max() < d


def test_cbp_hashes_are_the_numpy_legacy_streams():
    """CBCNN.py:76-91: np.random.seed(1/3/5/7) + randint — the bit-exact contract of the count sketch."""
    for d in (8192, 6000):
        h1, s1, h2, s2 = O.cbp_hashes(512, d)
        np.random.seed(1); e1 = np.random.randint(d, size=512)
        np.random.seed(3); t1 = 2 * np.random.randint(2, size=512) - 1
        np.random.seed(5); e2 = np.random.randint(d, size=512)
        np.random.seed(7); t2 = 2 * np.random.randint(2, size=512) - 1
        assert np.array_equal(h1, e1) and np.array_equal(s1, t1) and np.array_equal(h2, e2) and np.array_equal(s2, t2)


def test_covpool_is_the_centred_covariance_and_backward_matches_autograd():
    x = detgen.det((2, 12, 4, 5), 5).double()
    c = O.covpool_fwd(x)
    X = x.view(2, 12, 20)
    Xc = X - X.mean(dim=2, keepdim=True)
    assert torch.allclose(c, Xc @ Xc.transpose(1, 2) / 20, rtol=1e-10, atol=1e-12)             # X (I/M - 11^T/M^2) X^T
    g = detgen.det(c.shape, 6).double()
    xg = x.clone().requires_grad_(True)
    (dx,) = torch.autograd.grad(O.covpool_fwd(xg), xg, g)
    # Covpool.backward (MPNCOV.py:121-134) symmetrises the incoming gradient: equals autograd for the symmetrised g
    (dx_sym,) = torch.autograd.grad(O.covpool_fwd(xg), xg, 0.5 * (g + g.transpose(1, 2)))
    ours = O.covpool_bwd(x, g)
    assert torch.allclose(ours, 2 * dx_sym, rtol=1e-9, atol=1e-12) or torch.allclose(ours, dx_sym, rtol=1e-9, atol=1e-12) \
        or torch.allclose(ours, dx, rtol=1e-9, atol=1e-12)


def test_newton_schulz_converges_on_well_conditioned_input():
    """The recurrence of MPNCOV.py:144-161 is a Newton-Schulz square root: with enough iterations on an SPD matrix whose
    spectrum is well inside the convergence region it reproduces the true square root (the reference uses 5, unconverged)."""
    torch.manual_seed(0)
    a = torch.randn(2, 10, 10, dtype=torch.float64)
    spd = a @ a.transpose(1, 2) / 10 + torch.eye(10, dtype=torch.float64)
    y, _ = O.sqrtm_fwd(spd, 25)
    assert torch.allclose(y @ y, spd, rtol=1e-8, atol=1e-8)


def test_triuvec_roundtrip_and_order():
    x = detgen.det((2, 7, 7), 8).double()
    v = O.triuvec_fwd(x)
    assert v.shape == (2, 28, 1)
    r, c = np.triu_indices(7)                                  # row-major upper triangle = ones.triu().nonzero(), MPNCOV.py:213
    assert torch.equal(v[:, :, 0], x[:, r, c])
    back = O.triuvec_bwd(v, 7)
    assert torch.equal(back[:, r, c], v[:, :, 0]) and back.tril(-1).abs().sum() == 0


def test_cross_entropy_label_smoothing_matches_torch():
    logits = detgen.det((6, 11), 2)
    labels = detgen.det_labels(6, 11, 3)
    ref = torch.nn.CrossEntropyLoss(label_smoothing=0.1)(logits, labels)
    assert torch.allclose(O.cross_entropy_ls(logits, labels, 0.1), ref, rtol=1e-6, atol=1e-7)


def test_sgd_momentum_step_matches_torch_optim():
    p = detgen.det((37,), 1).clone()
    ref_p = torch.nn.Parameter(p.clone())
    opt = torch.optim.SGD([ref_p], lr=0.05, momentum=0.9, weight_decay=1e-3)
    buf = None
    for it in range(3):
        g = detgen.det((37,), 10 + it)
        ref_p.grad = g.clone()
        opt.step()
        p, buf = O.sgd_momentum_step(p, g, buf, 0.05, 0.9, 1e-3, it == 0)
    assert torch.allclose(p, ref_p.detach(), rtol=1e-6, atol=1e-7)
