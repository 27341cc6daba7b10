"""Matched-activation parity helper (tests only).

A ReLU / max-pool network is piecewise smooth: two correct implementations whose forward values differ by rounding
take different branches on a small fraction of elements, and each such flip changes that element's gradient by O(1)
— so parameter gradients of a TF32 forward cannot be compared with an fp32 reference at 1e-3, bug or no bug.
Here the GPU forward records the branch it took (``hawkeye_b200.ops.CAPTURE``) and the CPU oracle is evaluated in fp64
ON THAT BRANCH (``oracle.hop_oracle.MaskTape``).  What remains between the two gradients is arithmetic error only, so a
plumbing bug (wrong tap, wrong stride adjoint, missing term) shows up as O(1) while TF32 rounding stays at ~1e-3.
"""
import torch
import torch.nn.functional as F

from conftest import rel_l2
from kernel_check import nchw

# rel-L2 tolerance of the gradients by precision mode: single-pass TF32 and 3xTF32 (test_gpu_matched.py)
TOL = {0: 3e-3, 1: 2e-4}


def tape_items(capture):
    """hawkeye_b200.ops.CAPTURE records (device tensors, NHWC) -> oracle.hop_oracle.MaskTape items (CPU, NCHW)."""
    items = []
    for rec in capture:
        kind = rec[0]
        if kind == 'relu':
            items.append(('relu', (nchw(rec[1]) > 0).cpu()))
        elif kind == 'pool2':
            # same routing rule as hk_maxpool2x2_bwd and torch: first maximum in scan order
            _, idx = F.max_pool2d(nchw(rec[1]).cpu().contiguous(), 2, 2, return_indices=True)
            items.append(('pool', idx))
        elif kind == 'pool3':
            am, (N, H, W, C) = nchw(rec[1]).cpu().long(), rec[2]
            Ho, Wo = am.shape[2:]
            hh = 2 * torch.arange(Ho).view(1, 1, Ho, 1) + am // 3 - 1
            ww = 2 * torch.arange(Wo).view(1, 1, 1, Wo) + am % 3 - 1
            items.append(('pool', hh * W + ww))
        elif kind == 'ssqrt':
            items.append(('ssqrt', rec[1].detach().cpu()))
        else:
            raise ValueError(kind)
    return items


def gpu_step(net, x, labels, smoothing=0.1):
    """forward + CE(label smoothing) + backward of a hawkeye_b200 model with the decision capture on.
    -> (logits cpu, loss float, {name: grad cpu}, tape items)"""
    from hawkeye_b200 import ops
    ops.CAPTURE = []
    try:
        logits = net(x.cuda())
        cap = ops.CAPTURE
    finally:
        ops.CAPTURE = None
    loss = ops.CrossEntropyLS(smoothing)(logits, labels.cuda())
    net.zero_grad(set_to_none=True)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu() for k, p in net.named_parameters() if p.grad is not None}
    return logits.detach().cpu(), float(loss.item()), grads, tape_items(cap)


def oracle_step(forward_fn, x, labels, state, items, train_keys):
    """fp64 oracle loss/gradients on the recorded branch.  forward_fn(x, state, nl)."""
    from oracle import hop_oracle as O
    tape = O.MaskTape(items)
    st = {k: (v.double() if v.is_floating_point() else v) for k, v in state.items()}
    logits, loss, grads = O.loss_and_grads(lambda xx, s: forward_fn(xx, s, tape), x.double(), labels, st, set(train_keys))
    assert tape.done(), 'oracle consumed fewer decisions than the GPU forward recorded'
    return logits, float(loss), grads


def compare_grads(gpu_grads, ref_grads, tol, what=''):
    errs = {k: rel_l2(g, ref_grads[k]) for k, g in gpu_grads.items()}
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print(f'{what}: {len(errs)} parameter gradients, worst rel-L2: ' + ', '.join(f'{k} {v:.2e}' for k, v in worst))
    bad = {k: v for k, v in errs.items() if not v < tol}
    assert not bad, f'{what}: gradients beyond {tol}: {bad}'
    return errs


class Recorder:
    """CPU stand-in for the GPU capture (tests of the tape machinery itself): runs the plain non-linearities and records
    them in the SAME format hawkeye_b200.ops.CAPTURE uses (NHWC tensors, u8 window positions for the 3x3 pool)."""

    def __init__(self):
        self.cap = []

    def relu(self, x):
        y = F.relu(x)
        self.cap.append(('relu', y.detach().permute(0, 2, 3, 1)))
        return y

    def maxpool(self, x, k, s, p=0):
        if k == 2:
            self.cap.append(('pool2', x.detach().permute(0, 2, 3, 1)))
            return F.max_pool2d(x, 2, 2)
        y, idx = F.max_pool2d(x, 3, 2, 1, return_indices=True)
        N, C, H, W = x.shape
        Ho, Wo = y.shape[2:]
        kh = idx // W - 2 * torch.arange(Ho).view(1, 1, Ho, 1) + 1
        kw = idx % W - 2 * torch.arange(Wo).view(1, 1, 1, Wo) + 1
        self.cap.append(('pool3', (kh * 3 + kw).to(torch.uint8).permute(0, 2, 3, 1), (N, H, W, C)))
        return y

    def signed_sqrt(self, v):
        self.cap.append(('ssqrt', v.detach()))
        return torch.sign(v) * torch.sqrt(torch.abs(v) + 1e-10)
