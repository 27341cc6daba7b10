"""The train steps bench.py times, end to end at 448x448 batch 32: the fused VGG-16 path against fp64 on the branch it
took, and the mpn workload's CUDA-graph replay against its eager step.

Every kernel of these steps has its own element-wise test.  What those cannot see is the wiring between them on the
timed path: which buffers the Trainer hands the backward (views of one flat gradient buffer, filled with accumulate=1),
which forward VGGFeaturesFn takes when no activation capture is on (conv + pool in one kernel, the direct conv1_1, conv1_1's
weight gradient inside conv1_2's data gradient), which inputs a graph replay reads, and which learning rate and step
count each optimizer group gets.

A. bcnn_s2, bcnn_s1, cbcnn8192 (trainers built as bench.py builds them, deterministic weights, two steps).  Per step:
   1. the capture forward (ops.CAPTURE, the unfused path) and the production step give the same features and logits bit
      for bit, and for bcnn_s2 the same input of every layer and the same pool codes (the fused hk_conv3x3_fwd_pool code
      against hk_maxpool2x2_fwd_idx): the capture tape describes the branch the timed step took;
   2. the fp64 oracle on that branch, on the device in chunks of CHUNK images weighted n_c / N (BCNN couples no images
      before the mean cross-entropy), against logits, loss and the trained parameters' gradients in the Trainer's flat
      buffer, and per output channel for bcnn_s2;
   3. the SGD update element by element against fp64 on the device's own p, g and momentum buffer.
B. mpn: step 5, the second replay, against two eager runs of the same step on the graph stream, and its FusedAdam update
   against fp64 Adam with the three group learning rates.
C. Planted defects on tensors the tests already hold must fail the check each targets; a CPU test pins the chunked,
   weighted oracle to the unchunked one.
"""
import gc
import os
import re
import time

import numpy as np
import pytest
import torch

import detgen
import matched
from kernel_check import c_bound, check
from matched import TOL, rel_l2, tape_items
from step_check import make_trainer

BATCH, SIZE, CLASSES = 32, 448, 200
CHUNK = 4                   # images per fp64 oracle evaluation (VGG-16 at 448x448 in fp64: ~2 GB of activations each)
U = 2.0 ** -24              # fp32 unit roundoff

# The oracle runs on the branch the device took, so what separates it from the device is arithmetic alone: ~17 chained
# single-pass TF32 products (operands rounded to 10 mantissa bits, ~5e-4 each).  These are test_gpu_matched.py's bounds,
# which a plumbing defect (wrong buffer, missing or doubled term) exceeds by orders of magnitude.
LOGIT_REL = 1e-3            # per image: |logits - ref| / |ref|
# CBCNN's head takes sign(v) sqrt(|v|) of 8192 sketch bins, each a signed sum of ~32 Gram entries: on a bin that cancels
# to near zero a relative error e of the features becomes ~sqrt(e) of that bin.  That raises the per-image logit error of
# the TF32 step to 1.3e-3 (H100 SXM, 700 W); CBCNN_LOGIT_REL leaves 4.8x over it.  The bins are also summed with atomics,
# so the capture forward and the production forward (bit-identical features) give logits that differ by the order of
# those sums alone (1.5e-5 per image), bounded at a tenth of the fp64 bound.
CBCNN_LOGIT_REL = 6e-3
CBCNN_ORDER_REL = CBCNN_LOGIT_REL / 10
LOSS_ABS = 1e-4
# GRAD_REL bounds the relative L2 of every trained parameter's gradient.  On the timed step conv1_1's weight and bias
# gradients take 0.86 and 0.74 of it (H100 SXM, 700 W), as at batch 1 (2.35e-3 in smoke()): the error is in dY itself,
# after 12 TF32 data gradients (the bias gradient is a plain sum of dY), not in the split-K sums of the weight gradient,
# whose growth with the pixels per CTA a larger batch would show.
GRAD_REL = TOL[0]           # 3e-3
# Per output channel of a weight gradient: |dw[co] - ref[co]| / max(|ref[co]|, PER_CO_FLOOR * RMS over co of |ref[co]|).
# The floor keeps near-dead channels, whose tiny gradients carry the same absolute rounding as the others, from setting
# the figure.  The timed step's worst channel errs by 2e-2 (conv4_1 and conv5_x, H100 SXM, 700 W): the bound leaves 5x over
# it.  A channel whose gradient is lost or doubled errs by 1.0 relative to its own norm, 10x beyond the bound.
PER_CO_FLOOR = 0.25
PER_CO_REL = 0.1
# Optimizer updates, element by element against fp64 on the same fp32 inputs and the same fp32 hyper-parameters.
# SGD (sgd_momentum_kernel): g' = fma(wd, p, g) and buf = fma(m, buf, g') round once each, lr * buf and p - lr * buf once
# each: at most ~3 units of |p| + lr * (|g'| + m |buf|) (2 of |g'| + m |buf| for buf).  16 units: 5x that worst case.
SGD_ULPS = 16
# Adam (adam_kernel): m and v take 3 and 5 roundings of b1 |m| + (1 - b1) |g'| and of v; the step adds two square roots,
# two divisions, eps and the subtraction: ~12 units of |p| + lr / bc1 * M / denom at most.  48 units: 4x that worst case.
# hk_adam forms the bias corrections 1 - b^t in fp32 from powf (as torch's fused Adam does in fp32): one unit of b^t is
# b^t / (1 - b^t) units of the correction, ~200 units of bc2 at t = 5, of which the step takes half through the square
# root.  adam_bias_units() adds that term, for powf within one unit, to the bound of the update.
ADAM_ULPS = 48
# Graph replay against eager, for the tensors that two eager runs of the same step already give differently (sums whose
# order the atomics pick): the replay is one more such run, so it may differ from eager by the eager-to-eager spread,
# times REPLAY_SPREAD; the spread is measured in the test and printed beside the result.  On the mpn step these are the
# 3x3 convolutions' weight gradients, 3.0e-7 apart between eager runs and from the replay (H100 SXM, 700 W).
REPLAY_SPREAD = 8.0

WORKLOADS = {'bcnn_s2': ('BCNN_S2.yaml', 'BCNN', 2, None),
             'bcnn_s1': ('BCNN_S1.yaml', 'BCNN', 1, None),
             'cbcnn8192': ('CBCNN_S1.yaml', 'CBCNN', 1, 8192)}
MID_LAYER = 'backbone.17.weight'    # conv4_1, 256 -> 512 at 56x56: the planted one-block defect
MID_CO0 = 256


def _f32(v):
    """the value a float hyper-parameter has once it is passed to the kernel as a C float"""
    return float(np.float32(v))


def oracle_forward(stage, d=None):
    from oracle import hop_oracle as O
    if d is None:
        return lambda xx, st, nl: O.bcnn_forward(xx, st, stage, nl=nl)
    return lambda xx, st, nl: O.cbcnn_forward(xx, st, d, stage, nl=nl)


def slice_capture(cap, n0, n1):
    """ops.CAPTURE records of images n0..n1 (every record is batch-first; the 3x3 pool's also carries its input shape)"""
    out = []
    for rec in cap:
        r = (rec[0], rec[1][n0:n1])
        if rec[0] == 'pool3':
            r += ((n1 - n0,) + tuple(rec[2][1:]),)
        out.append(r)
    return out


def chunked_oracle(forward_fn, x, labels, state, cap, train_keys, chunk=CHUNK, device=None):
    """fp64 logits, mean cross-entropy and gradients of the batch on the recorded branch, `chunk` images at a time: each
    chunk's tape is built from the capture sliced to it (host memory stays at one chunk's masks), each chunk's mean loss
    and gradients are weighted n_c / N.  `state` is already fp64 on the device the oracle runs on."""
    N = x.shape[0]
    logits, loss, grads = [], 0.0, {}
    for n0 in range(0, N, chunk):
        n1 = min(N, n0 + chunk)
        items = [(k, v.to(device)) if device is not None else (k, v)
                 for k, v in tape_items(slice_capture(cap, n0, n1))]
        lg, ls, gr = matched.oracle_step(forward_fn, x[n0:n1], labels[n0:n1], state, items, train_keys)
        w = (n1 - n0) / N
        logits.append(lg)
        loss += w * ls
        for k, g in gr.items():
            grads[k] = grads[k] + w * g if k in grads else w * g
        del items, gr
    return torch.cat(logits), loss, grads


# ------------------------------------------------------------------------------------------------------------------
# C. the chunked, weighted oracle is the unchunked one (CPU)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [None, 256])
def test_chunked_oracle_matches_unchunked(d):
    """4 images of 64x64 on a quarter-width VGG-16, recorded by the CPU stand-in of the capture; chunks of 3 + 1 images,
    so that the weights n_c / N differ.  d: the compact bilinear head, whose signed-square-root bins are sliced too."""
    from oracle import hop_oracle as O
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg = O.vgg_cfg_scaled(4)
    state = detgen.vgg_bcnn_state(cfg, CLASSES, seed=100, head_in=d)
    x, labels = detgen.det((4, 3, 64, 64), 41), detgen.det_labels(4, CLASSES, 42)

    def fwd(xx, st, nl):
        return O.bcnn_forward(xx, st, 2, cfg=cfg, nl=nl) if d is None else O.cbcnn_forward(xx, st, d, 2, cfg=cfg, nl=nl)

    rec = matched.Recorder()
    with torch.no_grad():
        fwd(x.double(), {k: v.double() for k, v in state.items()}, rec)
    keys = list(state)
    ref_logits, ref_loss, ref = matched.oracle_step(fwd, x, labels, state, tape_items(rec.cap), keys)
    st64 = {k: v.double() for k, v in state.items()}
    logits, loss, grads = chunked_oracle(fwd, x, labels, st64, rec.cap, keys, chunk=3)
    assert rel_l2(logits, ref_logits) < 1e-12 and abs(loss - ref_loss) < 1e-12
    errs = {k: rel_l2(grads[k], ref[k]) for k in keys}
    assert max(errs.values()) < 1e-12, errs


# ------------------------------------------------------------------------------------------------------------------
# shared pieces of the GPU tests
# ------------------------------------------------------------------------------------------------------------------
class Checks:
    """worst share of its bound per named check (printed at the end), and the failures, asserted once all are printed"""

    def __init__(self, tag):
        self.tag, self.worst, self.failed = tag, {}, []

    def add(self, name, share, what=''):
        self.worst[name] = max(self.worst.get(name, 0.0), float(share))
        if not share <= 1.0:
            self.failed.append(f'{name}: {share:.3g} of its bound {what}')

    def bound(self, name, out, ref, absref, c, tag, names):
        """kernel_check.check of one tensor against c * absref"""
        try:
            self.add(name, check(out, ref, c_bound(absref, c), tag, names=names))
        except AssertionError as e:
            self.failed.append(f'{name}: {e}')
            self.worst[name] = max(self.worst.get(name, 0.0), _ratio_of(e))

    def equal(self, name, a, b):
        n = _ndiff(a, b)
        if n:
            self.failed.append(f'{name}: {n} of {a.numel()} elements differ')

    def report(self):
        print(f'{self.tag}: worst share of bound ' + ', '.join(f'{k} {v:.3g} (margin {1 / max(v, 1e-30):.3g}x)'
                                                                for k, v in self.worst.items()), flush=True)
        assert not self.failed, f'{self.tag}: ' + '; '.join(self.failed[:12])


def _ratio_of(err):
    m = re.search(r'ratio ([0-9.eE+-]+|inf|nan)', str(err))
    return float(m.group(1)) if m else float('inf')


def _ndiff(a, b):
    """elements whose bits differ (a shape mismatch counts every element)"""
    if a.shape != b.shape or a.dtype != b.dtype:
        return max(a.numel(), 1)
    if a.is_floating_point():
        a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    return int((a != b).sum())


def rejects(name, share):
    """a planted defect: its check must fail; prints how far beyond the bound it lands"""
    print(f'planted defect {name}: {share:.3g} of its bound', flush=True)
    assert not share <= 1.0, f'planted defect {name} passes its check ({share:.3g} of the bound)'   # NaN fails a check


def _bound_share(out, ref, absref, c):
    """the worst |out - ref| / (c * absref) that kernel_check.check would report (a check expected to fail)"""
    try:
        check(out, ref, c_bound(absref, c), 'planted', names=('i',))
    except AssertionError as e:
        return _ratio_of(e)
    return 0.0


def flat_layout(tr):
    """[(name, offset, numel)] of the trained parameters in the flat buffers, and the mask of the alignment padding"""
    from hawkeye_b200 import engine
    names = {id(p): n for n, p in tr.model.named_parameters()}
    out, off = [], 0
    for p in tr.flat.params:
        out.append((names[id(p)], off, p.numel()))
        off += engine._align(p.numel())
    pad = torch.ones(tr.flat.numel, dtype=torch.bool, device=tr.flat.flat.device)
    for _, a, n in out:
        pad[a:a + n] = False
    return out, pad


def check_views(tr, layout, checks):
    """every trained parameter and its .grad are the views of the flat buffers the Trainer laid out"""
    params = dict(tr.model.named_parameters())
    for name, a, n in layout:
        p = params[name]
        ok = (p.data_ptr() == tr.flat.flat.data_ptr() + 4 * a and p.grad is not None
              and p.grad.data_ptr() == tr.flat.grad.data_ptr() + 4 * a and p.grad.numel() == n)
        if not ok:
            checks.failed.append(f'{name}: parameter or gradient is not its view of the flat buffer')


def check_padding(checks, pad, **bufs):
    for k, t in bufs.items():
        n = int((t[pad].view(torch.int32) != 0).sum())
        if n:
            checks.failed.append(f'{k}: {n} alignment padding elements are not +0.0')


def per_co_share(dev, ref, where=None):
    """worst per-output-channel share of PER_CO_REL; `where` collects (channel, its norm over the RMS norm)"""
    d, r = dev.double().flatten(1), ref.double().flatten(1)
    rn = r.norm(dim=1)
    rms = rn.pow(2).mean().sqrt()
    e = (d - r).norm(dim=1) / rn.clamp_min(PER_CO_FLOOR * rms).clamp_min(1e-30)
    co = int(torch.nan_to_num(e, nan=float('inf')).argmax())
    if where is not None:
        where.append((co, float(rn[co] / rms)))
    return float(e[co]) / PER_CO_REL


def grad_shares(dev, ref, per_co, where=None):
    """{check: share} of the gradient checks: whole-tensor relative L2 of every trained parameter and, with per_co, the
    per-output-channel figure of every weight (`where` collects its worst channel)"""
    out = {}
    for k, r in ref.items():
        out[f'grad {k}'] = rel_l2(dev[k], r) / GRAD_REL
        if per_co and k.endswith('weight'):
            w = []
            out[f'per-co {k}'] = per_co_share(dev[k], r, w)
            if where is not None:
                where[f'per-co {k}'] = w[0]
    return out


def logit_errs(dev, ref):
    """per-image relative error of the logits"""
    d, r = dev.double(), ref.double()
    return (d - r).norm(dim=1) / r.norm(dim=1)


def _trainer(cfg_name, trainer, monkeypatch, graph):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    torch.manual_seed(0)
    tr = make_trainer(monkeypatch, trainer, cfg_name, graph=graph)
    return tr, tr.config


def _batches(n, dev):
    """bench.py's seeded batch, then the next ones from the same generator"""
    g = torch.Generator().manual_seed(1234)
    out = []
    for _ in range(n):
        x = torch.randn(BATCH, 3, SIZE, SIZE, generator=g)
        y = torch.randint(0, CLASSES, (BATCH,), generator=g)
        out.append((x.to(dev), y.to(dev)))
    return out


def _free():
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# A. the VGG-16 steps against fp64
# ------------------------------------------------------------------------------------------------------------------
def _sgd_refs(tr, layout, p0, g0, b0, first, lr_scale=None):
    """fp64 torch.optim.SGD step per group on the device's own fp32 p, g and buf: -> [(a, b, p_ref, buf_ref, |p| bound
    scale, |buf| bound scale)]; lr_scale {group index: factor} plants a wrong group learning rate"""
    from oracle import hop_oracle as O
    out = []
    for gi, (pg, (a, b)) in enumerate(zip(tr.optimizer.param_groups, tr.flat.group_slices)):
        lr = _f32(pg['lr'] * (lr_scale or {}).get(gi, 1.0))
        mom, wd, gs = _f32(pg['momentum']), _f32(pg['weight_decay']), _f32(tr.optimizer.grad_scale)
        p, g, buf = p0[a:b].double(), g0[a:b].double() * gs, b0[a:b].double()
        p_ref, buf_ref = O.sgd_momentum_step(p, g, buf, lr, mom, wd, first)
        babs = (g + wd * p).abs() + (0.0 if first else mom * buf.abs())
        out.append((a, b, p_ref, buf_ref, p.abs() + lr * babs, babs))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('workload', list(WORKLOADS))
def test_vgg_train_step_vs_fp64(workload, monkeypatch):
    from oracle import hop_oracle as O
    from hawkeye_b200 import ops
    t0 = time.time()
    _free()
    torch.cuda.reset_peak_memory_stats()
    cfg_name, trainer, stage, d = WORKLOADS[workload]
    tr, cfg = _trainer(cfg_name, trainer, monkeypatch, graph=False)
    model, dev = tr.model, tr.device
    model.load_state_dict(detgen.vgg_bcnn_state(O.VGG16_D, CLASSES, seed=100, head_in=d))
    layout, pad = flat_layout(tr)
    train_keys = [n for n, _, _ in layout]
    assert len(train_keys) == (28 if stage == 2 else 2)
    mults = [m for _, m in tr.trained_groups()]
    assert [pg['initial_lr'] for pg in tr.optimizer.param_groups] == [cfg.train.optimizer.lr * m for m in mults]
    frozen = {n: p.detach().clone() for n, p in model.named_parameters() if not p.requires_grad}
    assert len(frozen) == (0 if stage == 2 else 26)
    if d is not None:       # the oracle's count-sketch matrices, built on the host, go where the features are
        orig_sketch = O.sketch_matrix
        monkeypatch.setattr(O, 'sketch_matrix', lambda h, s, dim, dtype=torch.float32: orig_sketch(h, s, dim, dtype).to(dev))
    kept = []          # (ctx.records, features) of every VGGFeaturesFn forward
    orig_fwd = ops.VGGFeaturesFn.forward

    def fwd(ctx, x, cfg_, save, *params):
        out = orig_fwd(ctx, x, cfg_, save, *params)
        kept.append((ctx.records, out.detach()))
        return out
    monkeypatch.setattr(ops.VGGFeaturesFn, 'forward', staticmethod(fwd))
    fwd_fn = oracle_forward(stage, d)
    batches = _batches(2, dev)
    checks = Checks(workload)
    first_tape0 = None
    for step, (x, y) in enumerate(batches, 1):
        ts = time.time()
        # 1. the capture forward (the branch record), then the production step exactly as bench.py's step_resident
        kept.clear()
        ops.CAPTURE = []
        try:
            logits_cap = model(x).detach()
            cap = ops.CAPTURE
        finally:
            ops.CAPTURE = None
        out = model(x)
        loss = tr.criterion(out, y)
        tr.optimizer.zero_grad()
        loss.backward()
        tr.allreduce.finish()
        torch.cuda.synchronize()
        assert len(kept) == 2
        (rec_cap, feat_cap), (rec_prod, feat_prod) = kept
        checks.equal(f'step {step} features', feat_prod, feat_cap)
        if d is None:
            checks.equal(f'step {step} logits', out.detach(), logits_cap)
        else:
            e = logit_errs(out.detach(), logits_cap)
            checks.add('capture vs production logits', float(e.max()) / CBCNN_ORDER_REL, f'(step {step})')
            print(f'{workload} step {step}: capture vs production logits (sketch bins summed in another order): '
                  f'{int((out.detach() != logits_cap).sum())} of {out.numel()} differ, per image up to {float(e.max()):.3g}',
                  flush=True)
        if stage == 2:
            assert rec_cap is not None and rec_prod is not None and len(rec_cap) == len(rec_prod) == 13
            ncodes = 0
            for li, (rc, rp) in enumerate(zip(rec_cap, rec_prod)):
                checks.equal(f'step {step} layer {li} input', rp['inp'], rc['inp'])
                if rc.get('code') is not None or rp.get('code') is not None:
                    checks.equal(f'step {step} layer {li} pool code', rp['code'], rc['code'])
                    ncodes += 1
            assert ncodes == 5
        kept.clear()
        del rec_cap, rec_prod, feat_cap, feat_prod
        dev_logits, dev_loss = out.detach().clone(), float(loss.item())
        del out, loss
        check_views(tr, layout, checks)
        g0 = tr.flat.grad.clone()
        p0, b0, first = tr.flat.flat.clone(), tr.optimizer.buf.clone(), tr.optimizer.first
        assert first == (step == 1)
        grads = {n: g0[a:a + k].view_as(p) for (n, a, k), p in zip(layout, tr.flat.params)}

        # 2. fp64 on the recorded branch, on the device
        state = {k: v.detach().double() for k, v in model.state_dict().items()}
        ref_logits, ref_loss, ref = chunked_oracle(fwd_fn, x, y, state, cap, train_keys, device=dev)
        logit_rel = LOGIT_REL if d is None else CBCNN_LOGIT_REL
        e = logit_errs(dev_logits, ref_logits)
        checks.add('logits', float(e.max()) / logit_rel, f'(step {step})')
        checks.add('loss', abs(dev_loss - ref_loss) / LOSS_ABS, f'(step {step}: {dev_loss:.7f} vs {ref_loss:.7f})')
        where = {}
        shares = grad_shares(grads, ref, stage == 2, where)
        for k, v in shares.items():
            checks.add(k.split(' ')[0], v, f'({k}, step {step})')
        top = sorted(shares.items(), key=lambda kv: -kv[1])[:6]
        print(f'{workload} step {step}: loss {dev_loss:.6f} (fp64 {ref_loss:.6f}); logits per image: median '
              f'{float(e.median()):.3g}, max {float(e.max()):.3g}; worst gradient shares ' +
              ', '.join(f'{k} {v:.3g}' + (' (co {}, norm {:.2f} x RMS)'.format(*where[k]) if k in where else '')
                        for k, v in top), flush=True)

        # C. planted defects on what this step holds
        if step == 1:
            k = BATCH - 1
            items = [(kk, v.to(dev)) for kk, v in tape_items(slice_capture(cap, k, k + 1))]
            _, _, gk = matched.oracle_step(fwd_fn, x[k:k + 1], y[k:k + 1], state, items, train_keys)
            loo = {n: (BATCH * r - gk[n]) / (BATCH - 1) for n, r in ref.items()}
            rejects(f'{workload}: fp64 gradients without image {k}',
                    max(v for kk, v in grad_shares(grads, loo, False).items()))
            del items, gk, loo
            first_tape0 = tape_items(slice_capture(cap, 0, CHUNK))
            if stage == 2:
                bad = dict(grads, **{'backbone.0.weight': 2 * grads['backbone.0.weight']})
                rejects('conv1_1 dw accumulated twice', grad_shares(bad, ref, False)['grad backbone.0.weight'])
                dw = grads[MID_LAYER].clone()
                dw[MID_CO0:MID_CO0 + 32] = 0
                bad = dict(grads, **{MID_LAYER: dw})
                s = grad_shares(bad, ref, True)
                print(f'planted defect: co {MID_CO0}..{MID_CO0 + 31} of {MID_LAYER} zeroed: whole-tensor check at '
                      f'{s["grad " + MID_LAYER]:.3g} of its bound', flush=True)
                rejects(f'co block {MID_CO0}..{MID_CO0 + 31} of {MID_LAYER} zeroed (per-channel check)',
                        s['per-co ' + MID_LAYER])
        else:
            tape = O.MaskTape([(kk, v.to(dev)) for kk, v in first_tape0])
            with torch.no_grad():
                lg = fwd_fn(x[:CHUNK].double(), state, tape)
            # BCNN: the wrong masks pass negative maps, whose Gram's square root is NaN
            rejects(f'{workload}: tape of step 1 on the images of step 2',
                    float(logit_errs(dev_logits[:CHUNK], lg).max()) / logit_rel)
            del tape, lg
        del cap, state, ref, ref_logits
        _free()

        # 3. the SGD update
        tr.optimizer.step()
        torch.cuda.synchronize()
        c = SGD_ULPS * U
        for gi, (a, b, p_ref, buf_ref, pabs, babs) in enumerate(_sgd_refs(tr, layout, p0, g0, b0, first)):
            checks.bound('sgd p', tr.flat.flat[a:b], p_ref, pabs, c, f'{workload} step {step} sgd p group {gi}',
                         names=('i',))
            checks.bound('sgd buf', tr.optimizer.buf[a:b], buf_ref, babs, c, f'{workload} step {step} sgd buf group {gi}',
                         names=('i',))
        check_padding(checks, pad, params=tr.flat.flat, grad=g0, momentum=tr.optimizer.buf)
        gi = len(tr.optimizer.param_groups) - 1
        a, b, p_ref, _, pabs, _ = _sgd_refs(tr, layout, p0, g0, b0, first, lr_scale={gi: 0.1})[gi]
        rejects(f'{workload} step {step}: SGD group {gi} at a tenth of its lr',
                _bound_share(tr.flat.flat[a:b], p_ref, pabs, c))
        if step == 2:        # at step 1 the momentum buffer is zero, so `first` changes nothing there
            for a, b, p_ref, buf_ref, pabs, babs in _sgd_refs(tr, layout, p0, g0, b0, not first)[:1]:
                rejects(f'{workload} step {step}: SGD with first flipped', _bound_share(tr.optimizer.buf[a:b], buf_ref,
                                                                                       babs, c))
        for n, p in model.named_parameters():
            if n in frozen and (p.grad is not None or _ndiff(p.detach(), frozen[n])):
                checks.failed.append(f'step {step}: frozen {n} changed or has a gradient')
        del g0, p0, b0, grads
        _free()
        print(f'{workload} step {step}: {time.time() - ts:.1f} s', flush=True)
    print(f'{workload}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)
    checks.report()
    del tr, model
    _free()


# ------------------------------------------------------------------------------------------------------------------
# B. the mpn step: graph replay against eager, FusedAdam against fp64
# ------------------------------------------------------------------------------------------------------------------
def adam_bias_units(b1, b2, t):
    """units of the update that fp32 bias corrections from a powf within one unit may cost (ADAM_ULPS)"""
    return 2 * (b1 ** t / (1 - b1 ** t) + 0.5 * b2 ** t / (1 - b2 ** t))


def _adam_refs(tr, p0, m0, v0, g, t, lrs=None):
    """fp64 torch.optim.Adam step per group from the snapshot on the replayed gradients: -> [(a, b, (p, m, v) refs,
    (p, m, v) bounds in units of U)]"""
    b1, b2, eps = _f32(tr.optimizer.betas[0]), _f32(tr.optimizer.betas[1]), _f32(tr.optimizer.eps)
    bias = adam_bias_units(b1, b2, t)
    gs = _f32(tr.optimizer.grad_scale)
    out = []
    for gi, (pg, (a, b)) in enumerate(zip(tr.optimizer.param_groups, tr.flat.group_slices)):
        lr, wd = _f32(lrs[gi] if lrs else pg['lr']), _f32(pg['weight_decay'])
        p, m, v = p0[a:b].double(), m0[a:b].double(), v0[a:b].double()
        gg = g[a:b].double() * gs + wd * p
        m1 = b1 * m + (1 - b1) * gg
        v1 = b2 * v + (1 - b2) * gg * gg
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        denom = v1.sqrt() / bc2 ** 0.5 + eps
        p1 = p - lr / bc1 * m1 / denom
        mabs = b1 * m.abs() + (1 - b1) * gg.abs()
        upd = lr / bc1 * mabs / denom
        out.append((a, b, (p1, m1, v1), (ADAM_ULPS * (p.abs() + upd) + bias * upd, ADAM_ULPS * mabs, ADAM_ULPS * v1)))
    return out


@pytest.mark.gpu
def test_mpn_graph_replay_and_adam(monkeypatch):
    t0 = time.time()
    _free()
    torch.cuda.reset_peak_memory_stats()
    tr, cfg = _trainer('MPN.yaml', 'MPN', monkeypatch, graph=True)
    model = tr.model
    assert tr._graph_wanted()
    layout, pad = flat_layout(tr)
    base = cfg.train.optimizer.lr
    pgs = tr.optimizer.param_groups
    assert len(pgs) == 3 and [pg['initial_lr'] for pg in pgs] == [0.2 * base, base, base]
    assert pgs[0]['lr'] == pytest.approx(0.2 * pgs[1]['lr'], rel=1e-12) and pgs[1]['lr'] == pgs[2]['lr']
    assert all(pg['weight_decay'] == 2e-5 for pg in pgs) and tr.optimizer.eps == 1e-8
    batches = _batches(5, tr.device)
    for s, (x, y) in enumerate(batches[:4], 1):       # eager 1-3, captured on 3, replayed at 4
        tr._graph_step(x, y)
        tr.optimizer.step()
        assert (tr._graph is not None) == (s >= 3)
    torch.cuda.synchronize()
    x, y = batches[4]
    bufs = dict(model.named_buffers())
    snap = dict(p=tr.flat.flat.clone(), m=tr.optimizer.m.clone(), v=tr.optimizer.v.clone(), t=tr.optimizer.t,
                bn={k: b.clone() for k, b in bufs.items()})
    assert snap['t'] == 4 and any(k.endswith('running_var') for k in bufs)

    def collect(out, loss):
        torch.cuda.synchronize()
        res = dict(logits=out.detach().clone(), loss=loss.detach().clone(), correct=tr.criterion.last_correct.clone())
        g = tr.flat.grad.clone()
        res.update({f'grad {n}': g[a:a + k] for n, a, k in layout})
        res.update({f'buffer {k}': b.clone() for k, b in bufs.items()})
        return res, g

    def restore():
        tr.flat.flat.copy_(snap['p'])
        tr.optimizer.m.copy_(snap['m'])
        tr.optimizer.v.copy_(snap['v'])
        tr.optimizer.t = snap['t']
        for k, b in bufs.items():
            b.copy_(snap['bn'][k])

    replay, g_replay = collect(*tr._graph_step(x, y))        # step 5: the second replay, on a batch it was not captured on
    checks = Checks('mpn')

    # FusedAdam on the replayed gradients
    tr.optimizer.step()
    torch.cuda.synchronize()
    t = snap['t'] + 1
    assert tr.optimizer.t == t
    c = U
    print(f'mpn: Adam at t = {t}: bias corrections add {adam_bias_units(_f32(0.9), _f32(0.999), t):.0f} units to the '
          f'bound of the update', flush=True)
    dev_state = (tr.flat.flat, tr.optimizer.m, tr.optimizer.v)
    for gi, (a, b, refs, scales) in enumerate(_adam_refs(tr, snap['p'], snap['m'], snap['v'], g_replay, t)):
        for nm, got, ref, sc in zip(('p', 'm', 'v'), dev_state, refs, scales):
            checks.bound(f'adam {nm}', got[a:b], ref, sc, c, f'mpn adam {nm} group {gi}', names=('i',))
    check_padding(checks, pad, params=tr.flat.flat, grad=g_replay, m=tr.optimizer.m, v=tr.optimizer.v)
    a, b, refs, scales = _adam_refs(tr, snap['p'], snap['m'], snap['v'], g_replay, t - 1)[0]
    rejects('Adam step count off by one', _bound_share(tr.flat.flat[a:b], refs[0], scales[0], c))
    lrs = [pg['lr'] for pg in pgs]
    a, b, refs, scales = _adam_refs(tr, snap['p'], snap['m'], snap['v'], g_replay, t, lrs=[lrs[1]] + lrs[1:])[0]
    rejects('Adam backbone group at the head groups\' lr', _bound_share(tr.flat.flat[a:b], refs[0], scales[0], c))

    # the same step eagerly, twice, on the graph stream (autograd bound the AccumulateGrad nodes to it)
    eager = []
    gs = tr._graph_stream
    for _ in range(2):
        restore()
        cur = torch.cuda.current_stream()
        gs.wait_stream(cur)
        with torch.cuda.stream(gs):
            out, loss = tr.eager_step(x, y)
        cur.wait_stream(gs)
        eager.append(collect(out, loss)[0])
        del out, loss
    e1, e2 = eager
    same = {k for k in e1 if _ndiff(e1[k], e2[k]) == 0}
    for k in ['logits', 'loss', 'correct'] + [k for k in e1 if k.startswith('buffer ')]:
        assert k in same, f'{k}: two eager runs of the same forward differ'
    spread = {k: rel_l2(e2[k], e1[k]) for k in e1 if k not in same}
    assert all(k.startswith('grad ') for k in spread), sorted(spread)
    for k in sorted(same):
        checks.equal(f'replay {k}', replay[k], e1[k])
    if spread:
        bound = REPLAY_SPREAD * max(spread.values())
        worst = max(spread, key=lambda k: rel_l2(replay[k], e1[k]))
        for k in spread:
            checks.add('replay vs eager (order-dependent sums)', rel_l2(replay[k], e1[k]) / bound, k)
        print(f'mpn: {len(same)} tensors bit-identical across the eager runs and under replay; {len(spread)} gradients '
              f'summed in a run-dependent order, eager-to-eager relative L2 up to {max(spread.values()):.3g}, bound '
              f'{bound:.3g}; worst replay {worst} {rel_l2(replay[worst], e1[worst]):.3g}: ' +
              ', '.join(sorted(k[5:] for k in spread)[:8]), flush=True)
    print(f'mpn: loss {float(replay["loss"]):.6f}, top-1 {int(replay["correct"])}; {time.time() - t0:.1f} s, peak '
          f'{torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)
    checks.report()
    del tr, model, eager, replay
    _free()
