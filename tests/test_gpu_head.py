"""Classifier GEMMs, label-smoothing CE and the fused optimizers vs torch-CPU fp64."""
import pytest
import torch
import torch.nn.functional as F

import detgen
from conftest import rel_l2

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('B,Fdim,N', [(2, 16384, 200), (32, 262144, 200), (5, 8192, 200), (8, 1024, 200)])
def test_linear(B, Fdim, N):
    """with and without bias; F < 2048 runs the forward as one K slice, which without bias the GEMM writes directly"""
    from hawkeye_b200 import ops
    x = detgen.det((B, Fdim), 1, Fdim ** -0.5)
    w = detgen.det((N, Fdim), 2, (2.0 / Fdim) ** 0.5)
    b = detgen.det((N,), 3, 0.01)
    dy = detgen.det((B, N), 4, 0.01)
    xg, wg, bg = (t.cuda().requires_grad_(True) for t in (x, w, b))
    y = ops.linear(xg, wg, bg)
    dx, dw, db = torch.autograd.grad(y, (xg, wg, bg), dy.cuda())
    xd, wd_, bd = (t.double().requires_grad_(True) for t in (x, w, b))
    y_ref = F.linear(xd, wd_, bd)
    rx, rw, rb = torch.autograd.grad(y_ref, (xd, wd_, bd), dy.double())
    errs = [rel_l2(y.detach().cpu(), y_ref.detach()), rel_l2(dx.cpu(), rx), rel_l2(dw.cpu(), rw), rel_l2(db.cpu(), rb)]
    print(f'linear B={B} F={Fdim}: y {errs[0]:.2e} dx {errs[1]:.2e} dw {errs[2]:.2e} db {errs[3]:.2e}')
    assert max(errs[:3]) < 2e-3 and errs[3] < 1e-5
    # bias-free: the input and weight gradients do not depend on the bias
    y0 = ops.linear(xg, wg, None)
    dx0, dw0 = torch.autograd.grad(y0, (xg, wg), dy.cuda())
    errs0 = [rel_l2(y0.detach().cpu(), F.linear(xd, wd_).detach()), rel_l2(dx0.cpu(), rx), rel_l2(dw0.cpu(), rw)]
    print(f'linear B={B} F={Fdim} no bias: y {errs0[0]:.2e} dx {errs0[1]:.2e} dw {errs0[2]:.2e}')
    assert max(errs0) < 2e-3


@pytest.mark.parametrize('precise', [0, 1])
def test_cross_entropy_ls(precise):
    """default mode: dlogits are rounded to tf32 on store (operand of the classifier MMAs) -> 2^-12 rms; precise: fp32.
    The top-1 count is checked against the fp64 arg-max.  A second batch labels row 0 with K and row 5 with -1: such a row
    adds eps (lse - mean(z)) to the loss, gets softmax - eps/K and never counts (the rule of include/hawkeye_b200.h)."""
    from hawkeye_b200 import ops, _lib
    B, K, eps = 32, 200, 0.1
    logits = detgen.det((B, K), 1)
    labels = detgen.det_labels(B, K, 2)
    out_of_range = labels.clone()
    out_of_range[0], out_of_range[5] = K, -1     # z[y] of these rows would still lie inside the logits tensor
    for y in (labels, out_of_range):
        lg = logits.cuda().requires_grad_(True)
        ce = ops.CrossEntropyLS(eps)
        _lib.set_precise(precise)
        try:
            loss = ce(lg, y.cuda())
            (g,) = torch.autograd.grad(loss, lg)
        finally:
            _lib.set_precise(0)
        ld = logits.double().requires_grad_(True)
        valid = (y >= 0) & (y < K)
        if valid.all():
            ref = F.cross_entropy(ld, y, label_smoothing=eps)
            (rg,) = torch.autograd.grad(ref, ld)
        else:
            z, yc = ld.detach(), y.clamp(0, K - 1)
            lse = torch.logsumexp(z, 1)
            nll_y = torch.where(valid, lse - z.gather(1, yc[:, None])[:, 0], 0.0)
            ref = ((1 - eps) * nll_y + eps * (lse - z.mean(1))).mean()
            rg = (torch.softmax(z, 1) - (1 - eps) * F.one_hot(yc, K) * valid[:, None] - eps / K) / B
        assert abs(loss.item() - ref.item()) < 1e-5 and rel_l2(g.cpu(), rg) < (1e-5 if precise else 3e-4)
        assert ce.last_correct.item() == ((logits.double().argmax(1) == y) & valid).sum().item()


def test_sgd_and_adam():
    from hawkeye_b200 import _lib
    from oracle import hop_oracle as O
    n = 100003
    p, g = detgen.det((n + 1,), 1)[:n].clone(), detgen.det((n + 1,), 2)[:n].clone()
    pg, gg, buf = p.cuda(), g.cuda(), torch.zeros(n, device='cuda')
    s = _lib.stream_ptr()
    pr, br = p.double(), None
    for step in range(3):
        _lib.call('hk_sgd_momentum', pg, gg, buf, n, 0.01, 0.9, 1e-4, 0.5, int(step == 0), s)
        pr, br = O.sgd_momentum_step(pr, g.double() * 0.5, br, 0.01, 0.9, 1e-4, step == 0)
    assert rel_l2(pg.cpu(), pr) < 1e-6
    pa = torch.nn.Parameter(p.clone().double())
    opt = torch.optim.Adam([pa], lr=1e-3, weight_decay=2e-5)
    pg, m, v = p.cuda(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    for step in range(1, 4):
        pa.grad = g.double().clone()
        opt.step()
        _lib.call('hk_adam', pg, gg, m, v, n, 1e-3, 0.9, 0.999, 1e-8, 2e-5, 1.0, step, s)
    assert rel_l2(pg.cpu(), pa.detach()) < 1e-5
