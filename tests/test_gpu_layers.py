"""The layers the methods share (hawkeye_b200/ops.py) as autograd nodes against fp64 torch: the 1x1 convolution with and
without bias and with either input frozen, the 3x3 convolution with bias, the NCHW <-> NHWC transposes and ReLU / ELU."""
import pytest
import torch
import torch.nn.functional as F

import detgen
from conftest import rel_l2
from kernel_check import nchw, nhwc, precise  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu
TOL = {0: 2e-3, 1: 1e-4}     # single-pass TF32 operands / 3xTF32, fp32 accumulate


def _check_conv(fn, k, N, H, W, cin, cout, bias, grad_x, grad_w, tol):
    x = detgen.det((N, cin, H, W), 1)
    w = detgen.det((cout, cin, k, k), 2, (2.0 / (cin * k * k)) ** 0.5)
    b = detgen.det((cout,), 3, 0.1) if bias else None
    g = detgen.det((N, cout, H, W), 4)
    xd, wd = x.double().requires_grad_(grad_x), w.double().requires_grad_(grad_w)
    bd = b.double().requires_grad_(True) if bias else None
    ref = F.conv2d(xd, wd, bd, padding=k // 2)
    ref.backward(g.double())

    xg = nhwc(x).cuda().requires_grad_(grad_x)
    wg = w.cuda().requires_grad_(grad_w)
    bg = b.cuda().requires_grad_(True) if bias else None
    y = fn(xg, wg, bg)
    y.backward(nhwc(g).cuda())
    assert y.shape == (N, H, W, cout)
    assert rel_l2(nchw(y.detach()).cpu(), ref.detach()) < tol
    assert (xg.grad is not None) == grad_x and (wg.grad is not None) == grad_w
    if grad_x:
        assert rel_l2(nchw(xg.grad).cpu(), xd.grad) < tol
    if grad_w:
        assert rel_l2(wg.grad.cpu(), wd.grad) < tol
    if bias:
        assert rel_l2(bg.grad.cpu(), bd.grad) < tol


@pytest.mark.parametrize('bias', [True, False], ids=['bias', 'nobias'])
@pytest.mark.parametrize('grad_x,grad_w', [(True, True), (False, True), (True, False)], ids=['both', 'w_only', 'x_only'])
def test_conv1x1(precise, bias, grad_x, grad_w):
    from hawkeye_b200 import ops
    _check_conv(ops.Conv1x1Fn.apply, 1, 2, 5, 7, 128, 256, bias, grad_x, grad_w, TOL[precise])


@pytest.mark.parametrize('N,H,W,cin,cout', [(2, 7, 7, 128, 128), (2, 16, 32, 64, 128)])
@pytest.mark.parametrize('bias', [True, False], ids=['bias', 'nobias'])
def test_conv3x3(precise, N, H, W, cin, cout, bias):
    from hawkeye_b200 import ops
    _check_conv(ops.Conv3x3Fn.apply, 3, N, H, W, cin, cout, bias, True, True, TOL[precise])


def test_layout_transposes():
    from hawkeye_b200 import ops
    x = detgen.det((2, 6, 5, 3), 5).cuda()
    a = x.clone().requires_grad_(True)
    y = ops.ToNHWCFn.apply(a)
    assert torch.equal(y, x.permute(0, 2, 3, 1))
    g = detgen.det(y.shape, 6).cuda()
    y.backward(g)
    assert torch.equal(a.grad, g.permute(0, 3, 1, 2))

    b = x.clone().requires_grad_(True)                   # read as NHWC [2, 6, 5, 3]
    z = ops.ToNCHWFn.apply(b)
    assert torch.equal(z, x.permute(0, 3, 1, 2))
    g = detgen.det(z.shape, 7).cuda()
    z.backward(g)
    assert torch.equal(b.grad, g.permute(0, 2, 3, 1))

    # a strided view goes through the same transpose
    c = detgen.det((2, 6, 5, 8), 8).cuda()[..., ::2]
    assert torch.equal(ops.ToNHWCFn.apply(c), c.permute(0, 2, 3, 1))


@pytest.mark.parametrize('elu', [False, True], ids=['relu', 'elu'])
def test_act(elu):
    from hawkeye_b200 import ops
    x = detgen.det((3, 5, 7, 11), 9).cuda().requires_grad_(True)
    y = ops.ActFn.apply(x, elu)
    g = detgen.det(y.shape, 10).cuda()
    y.backward(g)
    x64 = x.detach().double().requires_grad_(True)
    r = F.elu(x64) if elu else F.relu(x64)
    r.backward(g.double())
    assert (y.double() - r).abs().max() < 1e-6 and (x.grad.double() - x64.grad).abs().max() < 1e-6
