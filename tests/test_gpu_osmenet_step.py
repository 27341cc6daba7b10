"""The osmenet train step bench.py times, end to end at 448x448 batch 32: ResNet-101, OSME and MAMC against fp64 on the
branch the device took, the SGD update element by element, and the step under CUDA-graph replay.

Every kernel of this step has its own element-wise test (test_gpu_resnet50_units.py, test_gpu_osme_head.py).  What those
cannot see is the wiring between them: the NCHW trunk output flattened into the two 401408-wide attention FCs, the trunk
gradient as the sum of both SE-gate backwards, the classifier on the sum of the attention features, MAMC's two terms, the
flat gradient buffer and its two groups (backbone at 0.1x lr), the warm-up lr, weight decay, and the running statistics
of the 104 train-mode BatchNorms.

A. The step under test is OSMENetTrainer.batch_training, built as bench.py builds it, on deterministic weights, two steps
   on different class-balanced batches (class-major, then interleaved).  The trunk's decisions are recorded with
   ops.CAPTURE and the OSME bottleneck ReLU's output through ActFn, so the fp64 oracle (oracle.hop_oracle.osmenet_forward,
   restated segment by segment) runs on the branch the device took.
B. The oracle runs the whole batch on the device without a full autograd tape: the stem and each of the 33 bottlenecks are
   checkpointed (torch.utils.checkpoint, non-reentrant), each segment replaying its own slice of the tape, and the BN
   batch statistics are recorded in the first forward only.  The two 1024 x 401408 attention FC weights are never held in
   fp64: their forward runs ROWS output features at a time, and their weight gradient is formed block by block from the
   kept dy and input, compared and dropped.
C. Two precision legs.  3xTF32 (_lib.set_precise(1)) checks the wiring against fp64 with tight bounds.  TF32 (the mode
   bench.py times) is compared with fp64 and with a stock PyTorch fp32 + TF32 run of the same restatement on the same
   tape: the worst of each kind must be within STOCK_RATIO of the stock run's, and every tensor under a ceiling.
D. SGD (momentum 0, weight decay, warm-up lr) element by element against fp64 on the device's own p and g, with the group
   lrs computed from configs/OSMENet.yaml.
E. Planted defects on tensors the test holds fail the check each targets; CPU self-tests pin the block-recomputed runner
   to a plain full-tape run, osme_forward to the reference fixtures and the row-blocked FC to the unblocked one.
"""
import math
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import detgen
import matched
from conftest import load_golden, rel_l2
from matched import tape_items
from step_check import assert_trainer_replays, eager_and_graph_losses, make_trainer, no_host_sync
from test_gpu_train_step import Checks, _f32, _free, check_padding, check_views, flat_layout

BATCH, SIZE, CLASSES = 32, 448, 200
N_CLASSES, N_SAMPLES = 8, 4            # configs/OSMENet.yaml: BalancedBatchSampler's n_classes x n_samples
BLOCKS = (3, 4, 23, 3)                 # ResNet-101
N_BN = 1 + 3 * sum(BLOCKS) + 4         # stem, three per bottleneck, one per downsample
ROWS = 128                             # output features per block of the attention FCs' oracle
SGD_CHUNK = 1 << 25                    # parameters per fp64 chunk of the SGD check
U = 2.0 ** -24
F64 = torch.float64
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FC_WEIGHTS = ('osme.fcs.0.weight', 'osme.fcs.1.weight')
PER_ROW_FLOOR = 0.25                   # a row's error is taken over max(its norm, PER_ROW_FLOOR x the RMS row norm)

# Bounds, each a distance from fp64 (see distances()): logits and x_part per image (worst relative L2 of an image's row),
# the loss (absolute; it is ~80 on these weights), every gradient as a whole tensor (relative L2), the rows of the
# attention FCs' and the classifier's weight gradients (worst row, PER_ROW_FLOOR), the batch mean per BN that entered the
# running mean (worst channel, in units of the batch's standard deviation) and the unbiased batch variance that entered
# the running variance (relative L2 over the channels).  The device's batch statistics are read back from its running
# averages: (running after - 0.9 running before) / 0.1.
#
# 3xTF32 leg: what separates the device from fp64 on the recorded branch is arithmetic alone.  Worst measured over two
# runs of both steps (H100 80GB HBM3, 700 W), and each bound's margin over it:
#   logits  5.9e-4  -> 2.5e-3 (4.2x)     x_part  5.7e-4 -> 2.5e-3 (4.4x)    loss  4.6e-4 -> 2e-3 (4.3x)
#   grad    8.9e-4 (backbone.7.2.bn2.weight) -> 4e-3 (4.5x)                 row   2.0e-3 (osme.fcs.0.weight) -> 8e-3 (4.1x)
#   bn mean 2.8e-5  -> 1.2e-4 (4.3x)     bn var  2.5e-5 -> 1.05e-4 (4.2x)
# A wiring defect moves these by O(1): a missing image, swapped FC gradients, an NHWC flatten (see the planted defects).
# The running variance's bound sits below the 1 / (n - 1) = 1.6e-4 that the biased variance differs by on the 14x14 maps.
PRECISE = {'logits': 2.5e-3, 'x_part': 2.5e-3, 'loss': 2e-3, 'grad': 4e-3, 'row': 8e-3, 'bn mean': 1.2e-4,
           'bn var': 1.05e-4}
# TF32 leg (the mode bench.py times).  A random-weight train-mode ResNet-101 at 448x448 amplifies single-pass TF32
# rounding to O(1) at the head: the stock fp32 + TF32 run of the same restatement on the same tape is itself up to 0.52
# (logits per image), 0.62 (a gradient) and 1.7 (a row of the FC gradients) from fp64.  So the TF32 leg holds the library
# to the stock run: its worst distance of each kind at most STOCK_RATIO times the stock run's worst of that kind (measured
# up to 1.3x, the rows of step 2), the rule of test_gpu_resnet_backward.test_resnet101_features_vs_stock_tf32.  The
# loss, one number, is held to its ceiling only.  So are the BN batch statistics: the library's TF32 GEMMs truncate their
# fp32 operands (kernel_check.TRUNC) where cuDNN rounds them, and on the 1x1 convolutions of layer1 and layer2 (bn1 and
# the downsample) the library's batch variance is measured up to 15x, its batch mean up to 4.6x, further from fp64 than
# the stock run's.  Ceilings: the worst measured, over two runs of both steps (H100 80GB HBM3, 700 W), times 4 or more:
#   logits 0.51 -> 2.1    x_part 0.47 -> 2.0    loss 2.2 -> 9.0    grad 0.66 -> 2.7    row 1.28 -> 5.2
#   bn mean 0.34 -> 1.4   bn var 0.114 -> 0.46
TF32_CEIL = {'logits': 2.1, 'x_part': 2.0, 'loss': 9.0, 'grad': 2.7, 'row': 5.2, 'bn mean': 1.4, 'bn var': 0.46}
STOCK_RATIO = 2.0
STOCK_KINDS = ('logits', 'x_part', 'grad', 'row')
# SGD (sgd_momentum_kernel): g' = fma(wd, p, g), buf = fma(m, buf, g'), lr * buf and p - lr * buf round once each: at most
# ~3 units of |p| + lr |g'| (2 of |g'| for buf).  16 units: 5x that worst case (test_gpu_train_step.SGD_ULPS).
SGD_ULPS = 16


# ------------------------------------------------------------------------------------------------------------------
# the block-recomputed oracle
# ------------------------------------------------------------------------------------------------------------------
class BlockLinear(torch.autograd.Function):
    """y = s w^T in s's dtype, w cast `rows` output features at a time (never whole in that dtype).  The backward
    returns ds only and keeps (s, dy): the weight gradient dy^T s is formed block by block by whoever checks it."""

    @staticmethod
    def forward(ctx, s, w, keep, rows):
        ctx.save_for_backward(s)
        ctx.w, ctx.keep, ctx.rows = w, keep, rows
        return torch.cat([s @ w[r:r + rows].to(s.dtype).T for r in range(0, w.shape[0], rows)], 1)

    @staticmethod
    def backward(ctx, dy):
        (s,) = ctx.saved_tensors
        w, rows = ctx.w, ctx.rows
        ctx.keep.update(s=s.detach(), dy=dy.detach())
        ds = None
        for r in range(0, w.shape[0], rows):
            t = dy[:, r:r + rows] @ w[r:r + rows].to(dy.dtype)
            ds = t if ds is None else ds + t
        return ds, None, None, None


def blocked_linear(keeps, rows=ROWS, nhwc=None):
    """a `linear` for osme_forward: BlockLinear plus the bias, one keep dict appended per call.  nhwc = (C, H, W) plants
    a defect: the gated map flattened in NHWC order"""
    def linear(s, w, b):
        if nhwc is not None:
            s = s.view(s.shape[0], *nhwc).permute(0, 2, 3, 1).reshape(s.shape[0], -1)
        keeps.append({})
        return BlockLinear.apply(s, w, keeps[-1], rows) + b
    return linear


def wgrad_block(keep, r0, r1, images=None):
    """rows r0:r1 of the weight gradient dy^T s of a BlockLinear (images: the batch rows that enter it)"""
    dy, s = keep['dy'], keep['s']
    if images is not None:
        dy, s = dy[images], s[images]
    return dy[:, r0:r1].T @ s


def run_oracle(x, labels, state, items, dtype, layers=None, rows=ROWS):
    """OSMENet's forward, MAMC loss and backward on the recorded tape, in `dtype` on x's device, with the stem and every
    bottleneck checkpointed.  state: the fp32 parameters the device step used (the attention FC weights stay these fp32
    tensors).  -> dict(logits, x_part, loss, feat (the trunk output), grads {name: gradient} of every parameter but the
    attention FC weights, keeps [per attention FC: its input s and dy], stats {BN: bn_batch_stats})"""
    from torch.utils.checkpoint import checkpoint
    from oracle import hop_oracle as O
    layers = O.RESNET101_LAYERS if layers is None else layers
    dev = x.device
    sd = {}
    for k, v in state.items():
        if k in FC_WEIGHTS:
            sd[k] = v
        elif v.is_floating_point() and 'running' not in k:
            sd[k] = v.detach().to(dev, dtype).requires_grad_(True)
        else:
            sd[k] = v
    stats = {}

    def bn(z, s, pre):
        if pre not in stats:            # the first forward; a recompute finds its statistics recorded
            stats[pre] = tuple(t.detach() for t in O.bn_batch_stats(z.detach()))
        return O._bn_train(z, s, pre)
    pos = [0]

    def segment(fn, n):
        """fn(input, tape) checkpointed with its own MaskTape, built inside the segment from its n items"""
        its = items[pos[0]:pos[0] + n]
        pos[0] += n

        def run(inp):
            tape = O.MaskTape([(k, v.to(dev)) for k, v in its])
            out = fn(inp, tape)
            assert tape.done(), 'a segment consumed fewer decisions than the device recorded'
            return out
        return run
    f = checkpoint(segment(lambda inp, t: O.resnet_stem(inp, sd, 'backbone.', t, bn), 2), x.to(dtype),
                   use_reentrant=False)
    for pre, stride, ds in O.resnet_block_plan(layers):
        f = checkpoint(segment(lambda inp, t, pre=pre, stride=stride, ds=ds: O._bottleneck(inp, sd, pre, stride, ds, t, bn),
                               3), f, use_reentrant=False)
    keeps = []
    head = O.MaskTape([(k, v.to(dev)) for k, v in items[pos[0]:]])
    x1, x_part = O.osme_forward(f, sd, 'osme.', head, blocked_linear(keeps, rows))
    assert head.done(), 'the oracle consumed fewer decisions than the device recorded'
    logits = F.linear(x1, sd['classifier.weight'], sd['classifier.bias'])
    loss = O.mamc_loss(logits, x_part, labels)
    keys = [k for k, v in sd.items() if v.requires_grad]
    grads = dict(zip(keys, torch.autograd.grad(loss, [sd[k] for k in keys])))
    return dict(logits=logits.detach(), x_part=x_part.detach(), loss=float(loss.detach()), feat=f.detach(), grads=grads,
                keeps=keeps, stats=stats)


def head_items(hs):
    """MaskTape items of the OSME bottleneck ReLU outputs [N, C / 16]"""
    return [('relu', (h > 0).cpu()) for h in hs]


# ------------------------------------------------------------------------------------------------------------------
# distances from fp64
# ------------------------------------------------------------------------------------------------------------------
def image_dist(out, ref):
    """worst relative L2 of one image's row"""
    d, r = out.double().flatten(1), ref.double().flatten(1)
    return float(((d - r).norm(dim=1) / r.norm(dim=1)).max())


def row_dist(err2, ref2):
    """worst per-row error from the squared row norms of the error and of the reference"""
    rms = ref2.mean().sqrt()
    e = err2.sqrt() / ref2.sqrt().clamp_min(PER_ROW_FLOOR * rms).clamp_min(1e-300)
    return float(torch.nan_to_num(e, nan=math.inf).max())


def fc_dists(got, keep, rows=ROWS, images=None):
    """(relative L2, worst row) of an attention FC's weight gradient: got(r0, r1) -> its rows r0:r1 in fp64, against
    the fp64 oracle's dy^T s, one row block at a time"""
    D = keep['dy'].shape[1]
    err2 = torch.zeros(D, dtype=F64, device=keep['dy'].device)
    ref2 = torch.zeros_like(err2)
    for r in range(0, D, rows):
        ref = wgrad_block(keep, r, min(D, r + rows), images)
        err2[r:r + rows] = (got(r, min(D, r + rows)) - ref).pow(2).sum(1)
        ref2[r:r + rows] = ref.pow(2).sum(1)
        del ref
    whole = float((err2.sum() / ref2.sum()).sqrt())
    return (whole if math.isfinite(whole) else math.inf), row_dist(err2, ref2)


def bn_dists(mean, unb, ref_stats, biased=False):
    """(worst channel of |mean - fp64 mean| / fp64 sigma, relative L2 of unb against fp64's unbiased variance) of the batch
    mean and unbiased variance a BN put into its running averages.  biased=True plants a defect: fp64's biased variance
    where the running average takes the unbiased one"""
    m64, v64, u64 = ref_stats
    em = float(torch.nan_to_num((mean.double() - m64).abs() / v64.sqrt().clamp_min(1e-30), nan=math.inf).max())
    return em, rel_l2(unb, v64 if biased else u64)


def distances(dev, ref, fc_got, bn_got):
    """{(kind, name): distance from the fp64 run `ref`} of a run's outputs.  dev: dict(logits, x_part, loss, grads);
    fc_got[i](r0, r1): rows of attention FC i's weight gradient; bn_got: {BN: (batch mean, unbiased variance)} that
    entered the running statistics"""
    out = {('logits', 'logits'): image_dist(dev['logits'], ref['logits']),
           ('x_part', 'x_part'): image_dist(dev['x_part'], ref['x_part']),
           ('loss', 'loss'): abs(dev['loss'] - ref['loss'])}
    for k, r in ref['grads'].items():
        out[('grad', k)] = rel_l2(dev['grads'][k], r)
    out[('row', 'classifier.weight')] = per_row(dev['grads']['classifier.weight'], ref['grads']['classifier.weight'])
    for i, k in enumerate(FC_WEIGHTS):
        out[('grad', k)], out[('row', k)] = fc_dists(fc_got[i], ref['keeps'][i])
    for k, (m, u) in bn_got.items():
        out[('bn mean', k)], out[('bn var', k)] = bn_dists(m, u, ref['stats'][k])
    return out


def per_row(got, ref):
    d, r = got.double(), ref.double()
    return row_dist((d - r).pow(2).sum(1), r.pow(2).sum(1))


# ------------------------------------------------------------------------------------------------------------------
# C. the step against fp64, in both precision legs
# ------------------------------------------------------------------------------------------------------------------
def balanced_batch(seed, interleaved):
    """n_classes x n_samples images of distinct classes: the sampler's order (same-class samples adjacent) or interleaved;
    pinned host tensors, as the loader hands them over"""
    classes = np.random.RandomState(seed).choice(CLASSES, N_CLASSES, replace=False)
    lab = np.tile(classes, N_SAMPLES) if interleaved else np.repeat(classes, N_SAMPLES)
    return {'img': detgen.det((BATCH, 3, SIZE, SIZE), seed).pin_memory(),
            'label': torch.from_numpy(lab.astype(np.int64)).pin_memory()}


class _Stock:
    """cuDNN and cuBLAS with TF32 allowed, as a stock PyTorch training run has them"""

    def __enter__(self):
        self.saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.saved


def _sgd_check(checks, tr, p0, b0, lrs, wd, first, tag, planted=None):
    """every element of p and buf after FusedSGD against fp64 SGD on the device's own p0, b0 and g, SGD_CHUNK at a time.
    planted {group: lr}: the worst share of the p check under those lrs instead (expected to fail) -> that share"""
    from oracle.hop_oracle import sgd_momentum_step
    c = SGD_ULPS * U
    gs = _f32(tr.optimizer.grad_scale)
    worst = 0.0
    for gi, (a, b) in enumerate(tr.flat.group_slices):
        if planted is not None and gi not in planted:
            continue
        lr = _f32((planted or {}).get(gi, lrs[gi]))
        for c0 in range(a, b, SGD_CHUNK):
            c1 = min(b, c0 + SGD_CHUNK)
            p, g, buf = p0[c0:c1].double(), tr.flat.grad[c0:c1].double() * gs, b0[c0:c1].double()
            p_ref, b_ref = sgd_momentum_step(p, g, buf, lr, 0.0, wd, first)
            babs = (g + wd * p).abs()
            for what, out, ref, absref in (('p', tr.flat.flat[c0:c1], p_ref, p.abs() + lr * babs),
                                           ('buf', tr.optimizer.buf[c0:c1], b_ref, babs)):
                if planted is not None and what == 'buf':
                    continue
                err = (out.double() - ref).abs()
                r = torch.where(err == 0, torch.zeros_like(err), err / (c * absref))
                share = float(torch.nan_to_num(r, nan=math.inf).max())
                worst = max(worst, share)
                if planted is None:
                    checks.add(f'sgd {what}', share, f'({tag} group {gi} elements {c0}:{c1})')
            del p, g, buf, p_ref, b_ref
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize('precise', [1, 0], ids=['3xtf32', 'tf32'])
def test_osmenet_train_step_vs_fp64(precise, monkeypatch):
    from hawkeye_b200 import _lib, ops
    from hawkeye_b200.config import load_config
    t0 = time.time()
    _free()
    torch.cuda.reset_peak_memory_stats()
    leg = '3xtf32' if precise else 'tf32'
    _lib.set_precise(0)
    torch.manual_seed(0)
    tr = make_trainer(monkeypatch, 'OSMENet', 'OSMENet.yaml', graph=False)
    model, dev = tr.model, tr.device
    model.load_state_dict(detgen.state_like(model))
    layout, pad = flat_layout(tr)
    names = [n for n, _, _ in layout]
    assert len(tr.flat.group_slices) == 2
    # the group lrs from the yaml: lr x the warm-up factor at epoch 0 (lr_warmup_decay) x {backbone 0.1, the rest 1.0}
    oc = load_config(os.path.join(REPO, 'configs', 'OSMENet.yaml')).train
    assert 'momentum' not in oc.optimizer and oc.scheduler.warmup_epochs > 0
    lrs = [oc.optimizer.lr * oc.scheduler.lr_warmup_decay * m for m in (0.1, 1.0)]
    wd = _f32(oc.optimizer.weight_decay)
    for pg, lr in zip(tr.optimizer.param_groups, lrs):
        assert pg['lr'] == pytest.approx(lr, rel=1e-12) and pg['momentum'] == 0.0 and _f32(pg['weight_decay']) == wd
    n_backbone = sum(1 for n in names if n.startswith('backbone.'))
    a0, b0_ = tr.flat.group_slices[0]
    assert names[:n_backbone] == [n for n in names if n.startswith('backbone.')] and \
        layout[n_backbone][1] == b0_ and a0 == 0
    bufs = dict(model.named_buffers())
    bns = sorted({k.rsplit('.', 1)[0] for k in bufs if k.endswith('running_mean')})
    assert len(bns) == N_BN
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)

    osme_h, outs = [], []
    orig_act = ops.ActFn.apply

    def act(x, *args):
        y = orig_act(x, *args)
        if ops.CAPTURE is not None:
            osme_h.append(y.detach().clone())
        return y
    monkeypatch.setattr(ops.ActFn, 'apply', act)
    orig_fm = tr.forward_model

    def forward_model(images, labels):
        out = orig_fm(images, labels)
        outs.append(tuple(t.detach().clone() for t in out))
        return out
    monkeypatch.setattr(tr, 'forward_model', forward_model)

    checks = Checks(f'osmenet {leg}')
    raw, planted = {}, []
    _lib.set_precise(precise)
    try:
        for step, batch in enumerate((balanced_batch(11, False), balanced_batch(12, True)), 1):
            ts = time.time()
            # 1. the step exactly as bench.py runs it, with the decisions recorded
            p0, b0 = tr.flat.flat.clone(), tr.optimizer.buf.clone()
            bn0 = {k: b.clone() for k, b in bufs.items()}
            first = tr.optimizer.first
            assert first == (step == 1)
            osme_h.clear()
            outs.clear()
            ops.CAPTURE = []
            try:
                loss = tr.batch_training(batch)
                cap = ops.CAPTURE
            finally:
                ops.CAPTURE = None
            torch.cuda.synchronize()
            assert len(outs) == 1 and len(osme_h) == 2 and all(h.shape == (BATCH, 128) for h in osme_h)
            dev_out = dict(logits=outs[0][0], x_part=outs[0][1], loss=float(loss))
            del loss
            items = tape_items(cap) + head_items(osme_h)
            assert len(items) == 2 + 3 * sum(BLOCKS) + 2
            del cap
            osme_h.clear()
            _free()
            check_views(tr, layout, checks)
            g = tr.flat.grad
            dev_out['grads'] = {n: g[a:a + k].view_as(p) for (n, a, k), p in zip(layout, tr.flat.params)}
            state = {n: p0[a:a + k].view_as(p) for (n, a, k), p in zip(layout, tr.flat.params)}
            for k, b in bn0.items():
                state[k] = b
            bn_dev = {}
            for k in bns:
                if int(bufs[k + '.num_batches_tracked']) != int(bn0[k + '.num_batches_tracked']) + 1:
                    checks.failed.append(f'step {step}: {k}.num_batches_tracked did not advance by one')
                # the batch statistics the device put into its running averages (momentum 0.1)
                bn_dev[k] = ((bufs[k + '.running_mean'].double() - 0.9 * bn0[k + '.running_mean'].double()) / 0.1,
                             (bufs[k + '.running_var'].double() - 0.9 * bn0[k + '.running_var'].double()) / 0.1)
            x, y = batch['img'].to(dev), batch['label'].to(dev)

            # 2. fp64 on the recorded branch; in the TF32 leg also the stock fp32 + TF32 run on it
            tr_ = time.time()
            ref = run_oracle(x, y, state, items, F64)
            t_ref = time.time() - tr_
            assert set(ref['grads']) | set(FC_WEIGHTS) == set(names) and set(ref['stats']) == set(bns)
            fc_dev = [lambda r0, r1, k=k: dev_out['grads'][k][r0:r1].double() for k in FC_WEIGHTS]
            d_dev = distances(dev_out, ref, fc_dev, bn_dev)
            d_stock = None
            if not precise:
                with _Stock():
                    stock = run_oracle(x, y, state, items, torch.float32)
                    fc_st = [lambda r0, r1, i=i: wgrad_block(stock['keeps'][i], r0, r1).double() for i in range(2)]
                    d_stock = distances(stock, ref, fc_st, {k: (v[0], v[2]) for k, v in stock['stats'].items()})
                del stock
            for (kind, name), v in d_dev.items():
                tag = f'(step {step} {name})'
                checks.add(kind if precise else f'{kind} ceiling', v / (PRECISE if precise else TF32_CEIL)[kind], tag)
                raw[kind] = max(raw.get(kind, 0.0), v)
            if d_stock is not None:
                for kind in STOCK_KINDS:
                    wd_, ws_ = (max(v for (kk, _), v in d.items() if kk == kind) for d in (d_dev, d_stock))
                    checks.add(f'{kind} vs stock', wd_ / max(STOCK_RATIO * ws_, 1e-300),
                               f'(step {step}: library {wd_:.3g}, stock {ws_:.3g})')
            top = sorted(((v, kn) for kn, v in d_dev.items()), reverse=True)
            print(f'osmenet {leg} step {step}: loss {dev_out["loss"]:.7f} (fp64 {ref["loss"]:.7f}); fp64 oracle {t_ref:.1f} s; '
                  f'worst distances per kind: ' + ', '.join(
                      f'{k} {max(v for (kk, _), v in d_dev.items() if kk == k):.3g}' for k in PRECISE), flush=True)
            if d_stock is not None:
                ratios = {kn: d_dev[kn] / max(d_stock[kn], 1e-300) for kn in d_dev}
                print(f'osmenet {leg} step {step}: stock TF32 worst per kind: ' + ', '.join(
                    f'{k} {max(v for (kk, _), v in d_stock.items() if kk == k):.3g}' for k in PRECISE) +
                    '; library / stock, worst: ' + ', '.join(f'{kn[0]} {kn[1]} {v:.3g}' for kn, v in
                                                             sorted(ratios.items(), key=lambda kv: -kv[1])[:6]), flush=True)
            print(f'osmenet {leg} step {step}: largest distances: ' + ', '.join(f'{kn[1]} {v:.3g}' for v, kn in top[:6]),
                  flush=True)

            # E. planted defects, on the 3xTF32 leg's tight bounds
            if precise and step == 1:
                bnd = PRECISE
                k = BATCH - 1
                others = torch.arange(BATCH, device=dev) != k
                s = [fc_dists(fc_dev[i], ref['keeps'][i], images=others)[0] / bnd['grad'] for i in range(2)]
                planted.append(('attention FC weight gradients of the oracle without image 31', min(s)))
                swapped = [fc_dists(fc_dev[1 - i], ref['keeps'][i])[0] / bnd['grad'] for i in range(2)]
                planted.append(('the two attention FCs\' weight gradients swapped', min(swapped)))
                from oracle import hop_oracle as O
                st64 = {kk: (v if kk in FC_WEIGHTS else v.double()) for kk, v in state.items() if v.is_floating_point()}
                with torch.no_grad():
                    _, xp = O.osme_forward(ref['feat'], st64, 'osme.', O.MaskTape([(kk, v.to(dev)) for kk, v in items[-2:]]),
                                           blocked_linear([], nhwc=tuple(ref['feat'].shape[1:])))
                planted.append(('the gated map flattened NHWC in the oracle', image_dist(dev_out['x_part'], xp) /
                                bnd['x_part']))
                del xp, st64
                planted.append(('the biased variance in the running-variance oracle', max(
                    bn_dists(bn_dev[kk][0], bn_dev[kk][1], ref['stats'][kk], biased=True)[1] for kk in bns) / bnd['bn var']))
            del ref, state, items, x, y
            _free()

            # D. the SGD update
            _sgd_check(checks, tr, p0, b0, lrs, wd, first, f'{leg} step {step}')
            check_padding(checks, pad, params=tr.flat.flat, grad=tr.flat.grad, momentum=tr.optimizer.buf)
            if step == 1:
                planted.append((f'{leg}: the backbone group at lr multiplier 1.0 in the SGD oracle',
                                _sgd_check(checks, tr, p0, b0, lrs, wd, first, '', planted={0: lrs[1]})))
            del p0, b0, bn0, dev_out
            _free()
            print(f'osmenet {leg} step {step}: {time.time() - ts:.1f} s', flush=True)
    finally:
        _lib.set_precise(0)
    print(f'osmenet {leg}: raw worst distances ' + ', '.join(f'{k} {v:.3g}' for k, v in raw.items()), flush=True)
    print(f'osmenet {leg}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)
    for name, share in planted:
        print(f'planted defect {name}: {share:.3g} of its bound', flush=True)
    checks.report()
    bad = [n for n, s in planted if s <= 1.0]
    assert not bad, f'planted defects that pass their check: {bad}'
    del tr, model
    _free()


# ------------------------------------------------------------------------------------------------------------------
# graph replay and the no-sync step
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_osmenet_graph_replay_and_no_sync(monkeypatch):
    """4 steps eager and with graph replay (steps 1-3 eager, captured on 3, replayed at 4) from one state, both groups at
    lr 0: at this size a random-weight step changes the loss by a quarter, and two eager runs whose atomics sum in another
    order drift apart step by step, so each step is compared on the weights the eager run had.  Then the trainer replays
    its own step with library kernels in it, and an eager step makes no host synchronisation."""
    batches = [balanced_batch(20 + i, i % 2 == 1) for i in range(4)]

    def build(graph):
        return make_trainer(monkeypatch, 'OSMENet', 'OSMENet.yaml', graph=graph)
    (eager, _), (replayed, _) = eager_and_graph_losses(build, batches, frozen_groups=(0, 1))
    print('osmenet eager', eager, 'graph', replayed, flush=True)
    for a, b in zip(eager, replayed):
        assert abs(a - b) < 2e-3 * max(1.0, abs(a)), (eager, replayed)
    _free()
    torch.manual_seed(0)
    assert_trainer_replays(build(True), batches)
    _free()
    torch.manual_seed(0)
    tr = build(False)
    tr.batch_training(batches[0])
    torch.cuda.synchronize()
    with no_host_sync():
        tr.batch_training(batches[1])
    torch.cuda.synchronize()
    del tr
    _free()


# ------------------------------------------------------------------------------------------------------------------
# CPU self-tests
# ------------------------------------------------------------------------------------------------------------------
def _small_state(layers, D, shape, classes=CLASSES, P=2, seed=300):
    """OSMENet-shaped state: a trunk of `layers` (planes, blocks, stride), OSME with P attentions of D features on a
    shape x shape map, and the classifier"""
    st, n = {}, [seed]

    def w(shp, fan):
        n[0] += 1
        return detgen.det(shp, n[0], (2.0 / fan) ** 0.5)

    def bn(pre, c):
        n[0] += 2
        st.update({pre + '.weight': 1 + detgen.det((c,), n[0] - 1, 0.1), pre + '.bias': detgen.det((c,), n[0], 0.1),
                   pre + '.running_mean': torch.zeros(c), pre + '.running_var': torch.ones(c),
                   pre + '.num_batches_tracked': torch.zeros((), dtype=torch.int64)})
    cin = layers[0][0]
    st['backbone.0.weight'] = w((cin, 3, 7, 7), 3 * 49)
    bn('backbone.1', cin)
    for li, (planes, blocks, _) in enumerate(layers):
        for b in range(blocks):
            pre = f'backbone.{4 + li}.{b}'
            st[pre + '.conv1.weight'] = w((planes, cin, 1, 1), cin)
            bn(pre + '.bn1', planes)
            st[pre + '.conv2.weight'] = w((planes, planes, 3, 3), planes * 9)
            bn(pre + '.bn2', planes)
            st[pre + '.conv3.weight'] = w((4 * planes, planes, 1, 1), planes)
            bn(pre + '.bn3', 4 * planes)
            if b == 0:
                st[pre + '.downsample.0.weight'] = w((4 * planes, cin, 1, 1), cin)
                bn(pre + '.downsample.1', 4 * planes)
            cin = 4 * planes
    for i in range(P):
        pre = f'osme.blocks.{i}.block.'
        st[pre + '0.weight'], st[pre + '0.bias'] = w((cin // 16, cin), cin), detgen.det((cin // 16,), n[0] + 1, 0.1)
        st[pre + '2.weight'], st[pre + '2.bias'] = w((cin, cin // 16), cin // 16), detgen.det((cin,), n[0] + 2, 0.1)
        fi = cin * shape * shape
        st[f'osme.fcs.{i}.weight'], st[f'osme.fcs.{i}.bias'] = w((D, fi), fi), detgen.det((D,), n[0] + 3, 0.1)
    st['classifier.weight'], st['classifier.bias'] = w((classes, D), D), detgen.det((classes,), n[0] + 4, 0.1)
    return st


class _HeadRecorder(matched.Recorder):
    """matched.Recorder for the trunk; the OSME bottleneck ReLU ([N, C / 16]) recorded as head_items does"""

    def __init__(self):
        super().__init__()
        self.head = []

    def relu(self, x):
        if x.dim() == 2:
            y = F.relu(x)
            self.head += head_items([y])
            return y
        return super().relu(x)


def test_block_recomputed_runner_matches_full_tape():
    """quarter-width trunk with blocks (1, 1, 2, 1), 64x64 inputs, batch 4, feature_shape 2, FC row blocks of 24 (64
    features: a partial last block): run_oracle against osmenet_forward on one full autograd tape"""
    from oracle import hop_oracle as O
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    layers = tuple(zip((16, 32, 64, 128), (1, 1, 2, 1), (1, 2, 2, 2)))
    st = _small_state(layers, 64, 2)
    x, labels = detgen.det((4, 3, 64, 64), 310), torch.tensor([3, 3, 7, 7])
    rec = _HeadRecorder()
    with torch.no_grad():
        O.osmenet_forward(x.double(), {k: (v.double() if v.is_floating_point() else v) for k, v in st.items()}, rec,
                          layers)
    items = tape_items(rec.cap) + rec.head
    # the full tape: every parameter in fp64, the attention FCs unblocked
    sd = {k: (v.double().requires_grad_('running' not in k) if v.is_floating_point() else v) for k, v in st.items()}
    stats = {}

    def bn(z, s, pre):
        stats[pre] = O.bn_batch_stats(z.detach())
        return O._bn_train(z, s, pre)
    tape = O.MaskTape(items)
    logits, x_part = O.osmenet_forward(x.double(), sd, tape, layers, bn=bn)
    assert tape.done()
    loss = O.mamc_loss(logits, x_part, labels)
    keys = [k for k, v in sd.items() if v.requires_grad]
    full = dict(zip(keys, torch.autograd.grad(loss, [sd[k] for k in keys])))
    got = run_oracle(x, labels, st, items, F64, layers=layers, rows=24)
    assert abs(got['loss'] - float(loss)) < 1e-12
    assert rel_l2(got['logits'], logits.detach()) < 1e-12 and rel_l2(got['x_part'], x_part.detach()) < 1e-12
    errs = {k: rel_l2(got['grads'][k], full[k]) for k in keys if k not in FC_WEIGHTS}
    for i, k in enumerate(FC_WEIGHTS):
        errs[k] = rel_l2(torch.cat([wgrad_block(got['keeps'][i], r, min(64, r + 24)) for r in range(0, 64, 24)]), full[k])
    assert len(errs) == len(keys) and max(errs.values()) < 1e-12, sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    assert set(got['stats']) == set(stats) and len(stats) == 1 + 3 * 5 + 4
    for k, v in stats.items():
        assert all(rel_l2(a, b) < 1e-12 for a, b in zip(got['stats'][k], v)), k


@pytest.mark.parametrize('tag, C, shape, B', [('osme_c256_7', 256, 7, 4), ('osme_c128_14', 128, (14, 14), 2)])
def test_osme_forward_matches_reference_fixtures(tag, C, shape, B):
    """osme_forward in fp64 against the reference OSME's fp32 outputs, input gradient and parameter gradients
    (tests/golden/make_golden_cin.py: weights from detgen.state_like, x = det(95, positive), loss (f det(96)).sum() +
    (parts det(97)).sum(); weight gradients of more than 65536 elements stored as [:, ::29] column slices)"""
    from hawkeye_b200.methods.osme import OSME
    from oracle import hop_oracle as O
    gold = load_golden('reference_cin')
    st = detgen.state_like(OSME(C, 64, feature_shape=shape, num_attention=2))
    hw = shape if isinstance(shape, tuple) else (shape, shape)
    sd = {k: v.double().requires_grad_(True) for k, v in st.items()}
    x = detgen.det((B, C) + hw, 95, positive=True).double().requires_grad_(True)
    f, parts = O.osme_forward(x, sd, prefix='')
    ((f * detgen.det(f.shape, 96).double()).sum() + (parts * detgen.det(parts.shape, 97).double()).sum()).backward()
    errs = {'f': rel_l2(f.detach(), gold[f'{tag}_f']), 'parts': rel_l2(parts.detach(), gold[f'{tag}_parts']),
            'dx': rel_l2(x.grad, gold[f'{tag}_dx'])}
    for k, v in sd.items():
        g = v.grad
        ref = gold[f'{tag}_g_{k}']
        errs[k] = rel_l2(g if g.numel() <= 65536 else g.reshape(g.shape[0], -1)[:, ::29], ref)
    print(tag, ', '.join(f'{k} {v:.2e}' for k, v in errs.items()))
    assert len(errs) == 3 + 12 and max(errs.values()) < 1e-5, errs


def test_blocked_linear_matches_unblocked():
    """BlockLinear's forward, ds and the block-wise weight gradient against F.linear's autograd, rows that do not divide
    the output features"""
    s = detgen.det((5, 300), 320).double().requires_grad_(True)
    w, b = detgen.det((70, 300), 321), detgen.det((70,), 322).double().requires_grad_(True)
    dy = detgen.det((5, 70), 323).double()
    keeps = []
    y = blocked_linear(keeps, rows=16)(s, w, b)
    ds, db = torch.autograd.grad(y, [s, b], dy)
    w64 = w.double().requires_grad_(True)
    y_ref = F.linear(s, w64, b)
    ds_ref, dw_ref, db_ref = torch.autograd.grad(y_ref, [s, w64, b], dy)
    dw = torch.cat([wgrad_block(keeps[0], r, min(70, r + 16)) for r in range(0, 70, 16)])
    assert len(keeps) == 1 and y.dtype == F64
    for a, r in ((y, y_ref), (ds, ds_ref), (dw, dw_ref), (db, db_ref)):
        assert rel_l2(a.detach(), r.detach()) < 1e-14
