"""CPU restatement of Hawkeye's high-order-pooling hot path (TEST INFRASTRUCTURE ONLY).

This is the parity ORACLE, not product code.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it; nothing under ``hawkeye_b200/`` does, and the product fails
loudly when its CUDA library is missing rather than routing here.

Pinning: the reference ships no tests or golden vectors, so the
oracle is pinned by (a) ``tests/golden/*.npz`` — outputs of the UNMODIFIED
reference modules imported through oracle/ref_harness by ``tests/golden/make_golden.py``
— and (b) the numpy-RNG known answers for the count-sketch hashes
(``tests/test_oracle.py``).  Every function cites the reference lines it restates.
All arithmetic is numpy / torch-CPU; ``dtype`` selects fp32 (the reference's
precision) or fp64 (to separate our error from the reference's own rounding).
"""
import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# Non-smooth points of the path (ReLU, max-pool arg-max, CBCNN's signed sqrt).  `Plain` is what the reference does.
# `MaskTape` replays decisions recorded from ANOTHER forward pass of the same network (the GPU's): ReLU becomes a
# multiplication by the recorded 0/1 mask, max-pool a gather at the recorded arg-max, the signed square root takes its
# derivative at the recorded bin values.  The function is then identical to the reference's wherever both forwards made
# the same decisions, and smooth in between — so its gradients are what the other implementation must reproduce up to
# its arithmetic error alone ("matched-activation" parity, tests/test_gpu_matched.py).
# --------------------------------------------------------------------------------------


class Plain:
    @staticmethod
    def relu(x):
        return F.relu(x)

    @staticmethod
    def maxpool(x, k, s, p=0):
        return F.max_pool2d(x, k, s, p)

    @staticmethod
    def signed_sqrt(v):
        return torch.sign(v) * torch.sqrt(torch.abs(v) + 1e-10)                 # CBCNN.py:132


class _SignedSqrtAt(torch.autograd.Function):
    """forward: sign(v) sqrt(|v|+1e-10) of v itself; backward: the derivative evaluated at the recorded values."""

    @staticmethod
    def forward(ctx, v, rec):
        ctx.save_for_backward(rec)
        return torch.sign(v) * torch.sqrt(torch.abs(v) + 1e-10)

    @staticmethod
    def backward(ctx, g):
        (rec,) = ctx.saved_tensors
        return g * (rec != 0).to(g.dtype) / (2 * torch.sqrt(torch.abs(rec) + 1e-10)), None


class MaskTape:
    """items, in execution order: ('relu', bool mask NCHW) | ('pool', int64 flat H*W indices [N,C,Ho,Wo]) |
    ('ssqrt', recorded pre-sqrt values [B,d])."""

    def __init__(self, items):
        self.items, self.i = list(items), 0

    def _next(self, kind):
        k, v = self.items[self.i]
        assert k == kind, f'tape out of step: wanted {kind}, recorded {k} at {self.i}'
        self.i += 1
        return v

    def relu(self, x):
        m = self._next('relu')
        assert m.shape == x.shape, (m.shape, x.shape)
        return x * m.to(x.dtype)

    def maxpool(self, x, k, s, p=0):
        idx = self._next('pool')
        return x.flatten(2).gather(2, idx.flatten(2)).view(idx.shape)

    def signed_sqrt(self, v):
        return _SignedSqrtAt.apply(v, self._next('ssqrt').to(v.dtype))

    def done(self):
        return self.i == len(self.items)


# --------------------------------------------------------------------------------------
# BCNN bilinear pooling  (model/methods/BCNN.py:13-27)
# --------------------------------------------------------------------------------------


def bilinear_pool_fwd(x):
    """x: [B,C,H,W] -> [B,C*C].  bmm(x,xT)/HW (:17-18); sqrt(.+1e-5) (:21); F.normalize (:26)."""
    B, C = x.shape[0], x.shape[1]
    hw = x.shape[2] * x.shape[3]
    xf = x.reshape(B, C, hw)
    g = torch.bmm(xf, xf.transpose(1, 2)) / hw
    z = torch.sqrt(g.reshape(B, -1) + 1e-5)
    n = z.norm(dim=1, keepdim=True).clamp_min(1e-12)  # F.normalize: x / max(||x||_2, eps)
    return z / n


def bilinear_pool_bwd(x, dy):
    """Closed-form input gradient of BCNN.py:13-27 (what autograd derives).

    dz=(dy - y<y,dy>)/||z||; dG=dz/(2z); dX=(dG+dG^T) X / HW.
    """
    B, C = x.shape[0], x.shape[1]
    hw = x.shape[2] * x.shape[3]
    xf = x.reshape(B, C, hw)
    g = torch.bmm(xf, xf.transpose(1, 2)) / hw
    z = torch.sqrt(g.reshape(B, -1) + 1e-5)
    n = z.norm(dim=1, keepdim=True).clamp_min(1e-12)
    y = z / n
    dz = (dy - y * (y * dy).sum(1, keepdim=True)) / n
    dg = (dz / (2 * z)).reshape(B, C, C)
    dx = torch.bmm(dg + dg.transpose(1, 2), xf) / hw
    return dx.reshape_as(x)


# --------------------------------------------------------------------------------------
# CBCNN compact bilinear pooling  (model/methods/CBCNN.py:38-164)
# --------------------------------------------------------------------------------------


def cbp_hashes(input_dim, output_dim):
    """Count-sketch hash/sign vectors, bit-exact contract (CBCNN.py:76-91).

    numpy legacy global MT19937 stream: seed(1)->h1, seed(3)->s1, seed(5)->h2, seed(7)->s2.
    Returns int64 arrays (h1, s1, h2, s2).
    """
    np.random.seed(1)
    h1 = np.random.randint(output_dim, size=input_dim)
    np.random.seed(3)
    s1 = 2 * np.random.randint(2, size=input_dim) - 1
    np.random.seed(5)
    h2 = np.random.randint(output_dim, size=input_dim)
    np.random.seed(7)
    s2 = 2 * np.random.randint(2, size=input_dim) - 1
    return (h1.astype(np.int64), s1.astype(np.int64), h2.astype(np.int64), s2.astype(np.int64))


def sketch_matrix(h, s, output_dim, dtype=torch.float32):
    """Dense [input_dim, output_dim] one-hot*sign matrix (CBCNN.py:137-164)."""
    m = torch.zeros(len(h), output_dim, dtype=dtype)
    m[torch.arange(len(h)), torch.from_numpy(np.asarray(h))] = torch.from_numpy(np.asarray(s)).to(dtype)
    return m


def cbp_fwd(x, output_dim, hashes=None, nl=Plain):
    """x: [B,C,H,W] -> [B,d].  The reference's FFT route (CBCNN.py:96-135)."""
    B, C, H, W = x.shape
    h1, s1, h2, s2 = hashes if hashes is not None else cbp_hashes(C, output_dim)
    S1 = sketch_matrix(h1, s1, output_dim, x.dtype)
    S2 = sketch_matrix(h2, s2, output_dim, x.dtype)
    flat = x.permute(0, 2, 3, 1).contiguous().view(-1, C)          # :114
    sk1, sk2 = flat.mm(S1), flat.mm(S2)                             # :117-118
    prod = torch.fft.fft(sk1) * torch.fft.fft(sk2)                  # :120-123
    cbp = torch.fft.ifft(prod).real.view(B, H, W, output_dim)       # :125-127
    cbp = cbp.sum(dim=1).sum(dim=1)                                 # :130
    cbp = nl.signed_sqrt(cbp)                                       # :132
    return F.normalize(cbp)                                         # :133


def cbp_presqrt_gram_scatter(x, output_dim, hashes=None):
    """Identity cross-check: sum_p ifft(fft(xS1)*fft(xS2)) ==
    signed scatter of the un-normalised Gram  X X^T  into bins (h1[i]+h2[j]) mod d."""
    B, C, H, W = x.shape
    h1, s1, h2, s2 = hashes if hashes is not None else cbp_hashes(C, output_dim)
    xf = x.reshape(B, C, H * W)
    g = torch.bmm(xf, xf.transpose(1, 2))
    idx = torch.from_numpy((h1[:, None] + h2[None, :]) % output_dim).reshape(-1)
    sgn = torch.from_numpy((s1[:, None] * s2[None, :])).to(x.dtype).reshape(-1)
    out = torch.zeros(B, output_dim, dtype=x.dtype)
    out.index_add_(1, idx, g.reshape(B, -1) * sgn)
    return out


# --------------------------------------------------------------------------------------
# Fast MPN-COV  (model/methods/MPNCOV.py:105-230)
# --------------------------------------------------------------------------------------


def covpool_fwd(x):
    """Covpool.forward (MPNCOV.py:107-119): X I_hat X^T, I_hat = I/M - 11^T/M^2."""
    B, C = x.shape[0], x.shape[1]
    M = x.shape[2] * x.shape[3]
    xf = x.reshape(B, C, M)
    I_hat = (-1.0 / M / M) * torch.ones(M, M, dtype=x.dtype) + (1.0 / M) * torch.eye(M, dtype=x.dtype)
    return xf.matmul(I_hat).bmm(xf.transpose(1, 2))


def covpool_bwd(x, g):
    """Covpool.backward (MPNCOV.py:121-134): (g+g^T) X I_hat."""
    B, C = x.shape[0], x.shape[1]
    M = x.shape[2] * x.shape[3]
    xf = x.reshape(B, C, M)
    I_hat = (-1.0 / M / M) * torch.ones(M, M, dtype=x.dtype) + (1.0 / M) * torch.eye(M, dtype=x.dtype)
    return (g + g.transpose(1, 2)).bmm(xf).matmul(I_hat).reshape_as(x)


def sqrtm_fwd(x, iterN):
    """Sqrtm.forward (MPNCOV.py:139-164).  Returns (y, saved) with saved=(A, YZY, normA, Y, Z)."""
    B, dim = x.shape[0], x.shape[1]
    I3 = 3.0 * torch.eye(dim, dtype=x.dtype).expand(B, dim, dim)
    normA = (1.0 / 3.0) * (x * I3).sum(dim=1).sum(dim=1)
    A = x / normA.view(B, 1, 1)
    Y = torch.zeros(B, iterN, dim, dim, dtype=x.dtype)
    Z = torch.eye(dim, dtype=x.dtype).view(1, 1, dim, dim).repeat(B, iterN, 1, 1)
    if iterN < 2:
        ZY = 0.5 * (I3 - A)
        YZY = A.bmm(ZY)
    else:
        ZY = 0.5 * (I3 - A)
        Y[:, 0] = A.bmm(ZY)
        Z[:, 0] = ZY
        for i in range(1, iterN - 1):
            ZY = 0.5 * (I3 - Z[:, i - 1].bmm(Y[:, i - 1]))
            Y[:, i] = Y[:, i - 1].bmm(ZY)
            Z[:, i] = ZY.bmm(Z[:, i - 1])
        YZY = 0.5 * Y[:, iterN - 2].bmm(I3 - Z[:, iterN - 2].bmm(Y[:, iterN - 2]))
    y = YZY * torch.sqrt(normA).view(B, 1, 1)
    return y, (A, YZY, normA, Y, Z)


def sqrtm_bwd(x, saved, g, iterN):
    """Sqrtm.backward (MPNCOV.py:166-202), the reference's hand-derived formulae verbatim in order."""
    A, ZYs, normA, Y, Z = saved
    B, dim = x.shape[0], x.shape[1]
    P = g * torch.sqrt(normA).view(B, 1, 1)
    aux = (g * ZYs).sum(dim=1).sum(dim=1) / (2 * torch.sqrt(normA))
    I3 = 3.0 * torch.eye(dim, dtype=x.dtype).expand(B, dim, dim)
    if iterN < 2:
        D = 0.5 * (P.bmm(I3 - A) - A.bmm(P))
    else:
        Yl, Zl = Y[:, iterN - 2], Z[:, iterN - 2]
        dldY = 0.5 * (P.bmm(I3 - Yl.bmm(Zl)) - Zl.bmm(Yl).bmm(P))
        dldZ = -0.5 * Yl.bmm(P).bmm(Yl)
        for i in range(iterN - 3, -1, -1):
            YZ = I3 - Y[:, i].bmm(Z[:, i])
            ZY = Z[:, i].bmm(Y[:, i])
            dldY_ = 0.5 * (dldY.bmm(YZ) - Z[:, i].bmm(dldZ).bmm(Z[:, i]) - ZY.bmm(dldY))
            dldZ_ = 0.5 * (YZ.bmm(dldZ) - Y[:, i].bmm(dldY).bmm(Y[:, i]) - dldZ.bmm(ZY))
            dldY, dldZ = dldY_, dldZ_
        D = 0.5 * (dldY.bmm(I3 - A) - dldZ - A.bmm(dldY))
    D = D.transpose(1, 2)                                            # :195
    gx = D / normA.view(B, 1, 1)                                     # :196
    gaux = (D * x).sum(dim=1).sum(dim=1)                             # :197
    coef = aux - gaux / (normA * normA)                              # :198-201
    gx = gx + coef.view(B, 1, 1) * torch.eye(dim, dtype=x.dtype)
    return gx


def triuvec_index(dim):
    """Row-major positions of ones(dim,dim).triu() (MPNCOV.py:213-214)."""
    return torch.ones(dim, dim).triu().reshape(-1).nonzero().reshape(-1)


def triuvec_fwd(x):
    """Triuvec.forward (MPNCOV.py:207-218) -> [B, dim(dim+1)/2, 1]."""
    B, dim = x.shape[0], x.shape[1]
    return x.reshape(B, dim * dim)[:, triuvec_index(dim)].unsqueeze(-1)


def triuvec_bwd(g, dim):
    """Triuvec.backward (MPNCOV.py:220-230)."""
    B = g.shape[0]
    out = torch.zeros(B, dim * dim, dtype=g.dtype)
    out[:, triuvec_index(dim)] = g.reshape(B, -1)
    return out.reshape(B, dim, dim)


class _CovpoolFn(torch.autograd.Function):
    """Covpool as the reference defines it: its OWN backward formula (MPNCOV.py:121-134), not autograd's."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return covpool_fwd(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return covpool_bwd(x, g)


class _SqrtmFn(torch.autograd.Function):
    """Sqrtm with the reference's hand-derived backward (MPNCOV.py:166-202)."""

    @staticmethod
    def forward(ctx, x, iterN):
        y, saved = sqrtm_fwd(x, iterN)
        ctx.x, ctx.saved, ctx.iterN = x, saved, iterN
        return y

    @staticmethod
    def backward(ctx, g):
        return sqrtm_bwd(ctx.x, ctx.saved, g, ctx.iterN), None


class _TriuvecFn(torch.autograd.Function):
    """Triuvec with the reference's scatter backward (MPNCOV.py:220-230)."""

    @staticmethod
    def forward(ctx, x):
        ctx.dim = x.shape[1]
        return triuvec_fwd(x)

    @staticmethod
    def backward(ctx, g):
        return triuvec_bwd(g, ctx.dim)


def mpncov_pool_fwd(x, iterN=5):
    """cov -> sqrtm -> triuvec on a [B,C,H,W] (already dimension-reduced) feature (MPNCOV.py:97-101)."""
    c = covpool_fwd(x)
    y, saved = sqrtm_fwd(c, iterN)
    return triuvec_fwd(y), (c, saved)


def mpncov_pool_bwd(x, g, iterN=5):
    c = covpool_fwd(x)
    _, saved = sqrtm_fwd(c, iterN)
    gs = triuvec_bwd(g, c.shape[1])
    gc = sqrtm_bwd(c, saved, gs, iterN)
    return covpool_bwd(x, gc)


# --------------------------------------------------------------------------------------
# VGG-16 "D" features  (model/backbone/vgg.py:56-70,76) and the BCNN / CBCNN heads
# --------------------------------------------------------------------------------------

VGG16_D = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M']


def vgg_cfg_scaled(width_div=1):
    """VGG16_D with channel widths divided (for small parity cases); width_div=1 is the reference."""
    return [v if v == 'M' else max(v // width_div, 8) for v in VGG16_D]


def vgg_state_keys(cfg=VGG16_D):
    """Sequential indices of the conv layers: backbone.{0,2,5,...}.{weight,bias}."""
    keys, idx = [], 0
    for v in cfg:
        if v == 'M':
            idx += 1
        else:
            keys.append(idx)
            idx += 2
    return keys


def vgg_features_fwd(x, state, cfg=VGG16_D, prefix='backbone.', nl=Plain):
    """conv3x3(s1,p1)+bias -> ReLU, 'M' = MaxPool2d(2,2) (vgg.py:56-70)."""
    idx = 0
    for v in cfg:
        if v == 'M':
            x = nl.maxpool(x, 2, 2)
            idx += 1
        else:
            x = nl.relu(F.conv2d(x, state[f'{prefix}{idx}.weight'], state[f'{prefix}{idx}.bias'], padding=1))
            idx += 2
    return x


def cross_entropy_ls(logits, labels, smoothing=0.1):
    """nn.CrossEntropyLoss(label_smoothing=0.1) (train.py:211-212), mean reduction."""
    return F.cross_entropy(logits, labels, label_smoothing=smoothing)


def bcnn_forward(x, state, stage=2, cfg=VGG16_D, nl=Plain):
    """BCNN.forward (BCNN.py:49-55)."""
    f = vgg_features_fwd(x, state, cfg, nl=nl)
    if stage == 1:
        f = f.detach()
    y = bilinear_pool_fwd(f)
    return F.linear(y, state['classifier.weight'], state['classifier.bias'])


def cbcnn_forward(x, state, output_dim, stage=2, cfg=VGG16_D, nl=Plain):
    """CBCNN.forward (CBCNN.py:29-35)."""
    f = vgg_features_fwd(x, state, cfg, nl=nl)
    if stage == 1:
        f = f.detach()
    y = cbp_fwd(f, output_dim, nl=nl)
    return F.linear(y, state['classifier.weight'], state['classifier.bias'])


def loss_and_grads(forward_fn, x, labels, state, train_keys=None):
    """loss = CE_ls(forward(x)); returns (logits, loss, {param: grad}) via torch-CPU autograd over the
    restated forward — the same thing the reference's loss.backward() (train.py:315-319) computes."""
    st = {k: v.detach().clone().requires_grad_(train_keys is None or k in train_keys) for k, v in state.items()}
    logits = forward_fn(x, st)
    loss = cross_entropy_ls(logits, labels)
    params = [v for v in st.values() if v.requires_grad]
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    names = [k for k, v in st.items() if v.requires_grad]
    return logits.detach(), loss.detach(), dict(zip(names, grads))


def sgd_momentum_step(p, g, buf, lr, momentum, weight_decay, first):
    """torch.optim.SGD (Examples/BCNN.py:40): g+=wd*p; buf = g (first) | m*buf+g; p-=lr*buf."""
    g = g + weight_decay * p
    buf = g.clone() if first else momentum * buf + g
    return p - lr * buf, buf


# --------------------------------------------------------------------------------------
# ResNet-50 v1.5 trunk (model/backbone/resnet.py:89-252) + MPN (MPNCOV.py:23-102), functional restatement
# --------------------------------------------------------------------------------------
RESNET50_LAYERS = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))   # (planes, blocks, stride)


def resnet_layers(blocks):
    """(planes, blocks, stride) of layer1..4 for a trunk with the given block counts, e.g. (3, 4, 23, 3) for ResNet-101."""
    return tuple(zip((64, 128, 256, 512), blocks, (1, 2, 2, 2)))


def _bn_train(x, st, pre, eps=1e-5):
    """nn.BatchNorm2d in train mode: batch statistics (biased var), affine (resnet.py:114-140 via norm_layer)."""
    return F.batch_norm(x, None, None, st[pre + '.weight'], st[pre + '.bias'], training=True, eps=eps)


def _bn_eval(x, st, pre, eps=1e-5):
    """nn.BatchNorm2d in eval mode: normalises with the running statistics st[pre + '.running_mean' / '.running_var']."""
    return F.batch_norm(x, st[pre + '.running_mean'], st[pre + '.running_var'], st[pre + '.weight'], st[pre + '.bias'],
                        training=False, eps=eps)


def bn_batch_stats(x):
    """Per-channel batch statistics of an NCHW tensor as train-mode BatchNorm2d takes them: (mean, biased variance, which
    normalises, unbiased variance, which enters the running average)."""
    mean = x.mean(dim=(0, 2, 3))
    var = x.var(dim=(0, 2, 3), unbiased=False)
    n = x.numel() // x.shape[1]
    return mean, var, var * n / max(n - 1, 1)


def _bottleneck(x, st, pre, stride, has_ds, nl=Plain, bn=_bn_train):
    """Bottleneck.forward (resnet.py:124-144): stride on the 3x3 (v1.5, :116)."""
    out = nl.relu(bn(F.conv2d(x, st[pre + '.conv1.weight']), st, pre + '.bn1'))
    out = nl.relu(bn(F.conv2d(out, st[pre + '.conv2.weight'], stride=stride, padding=1), st, pre + '.bn2'))
    out = bn(F.conv2d(out, st[pre + '.conv3.weight']), st, pre + '.bn3')
    identity = x
    if has_ds:
        identity = bn(F.conv2d(x, st[pre + '.downsample.0.weight'], stride=stride), st, pre + '.downsample.1')
    return nl.relu(out + identity)


def resnet_stem(x, st, prefix='backbone.', nl=Plain, bn=_bn_train):
    """conv1 (7x7/s2), bn1, relu, maxpool (3x3/s2) of ResNet._forward_impl (resnet.py:235-238)."""
    x = F.conv2d(x, st[prefix + '0.weight'], stride=2, padding=3)
    return nl.maxpool(nl.relu(bn(x, st, prefix + '1')), 3, 2, 1)


def resnet_block_plan(layers, prefix='backbone.'):
    """[(state prefix, stride, has downsample)] of every Bottleneck of layer1..4 in forward order (_make_layer,
    resnet.py:208-231): the first block of a layer strides and carries the downsample."""
    return [(f'{prefix}{4 + li}.{b}', stride if b == 0 else 1, b == 0)
            for li, (_, blocks, stride) in enumerate(layers) for b in range(blocks)]


def resnet50_trunk_fwd(x, st, prefix='backbone.', nl=Plain, layers=RESNET50_LAYERS, bn=_bn_train):
    """children()[:-2] of ResNet-50 (MPNCOV.py:28-29): conv1, bn1, relu, maxpool, layer1..4 -> [B,2048,H/32,W/32].
    ``layers`` gives other depths (``resnet_layers((3, 4, 23, 3))`` is ResNet-101); ``bn=_bn_eval`` is the eval-mode trunk."""
    x = resnet_stem(x, st, prefix, nl, bn)
    for pre, stride, has_ds in resnet_block_plan(layers, prefix):
        x = _bottleneck(x, st, pre, stride, has_ds, nl=nl, bn=bn)
    return x


def mpn_forward(x, st, iter_num=5, nl=Plain):
    """MPN.forward (MPNCOV.py:33-38) with dimension_reduction (conv_dr_block, :64-69), is_sqrt, is_vec."""
    f = resnet50_trunk_fwd(x, st, nl=nl)
    f = nl.relu(_bn_train(F.conv2d(f, st['pool.conv_dr_block.0.weight']), st, 'pool.conv_dr_block.1'))
    v = _TriuvecFn.apply(_SqrtmFn.apply(_CovpoolFn.apply(f), iter_num))            # MPNCOV.py:97-101
    return F.linear(v.reshape(v.shape[0], -1), st['classifier.weight'], st['classifier.bias'])


def npairs_loss(feats, labels):
    """NPairsLoss.forward (model/loss/MAMC_loss.py:35-90): [b, p, D] features of p attention branches, one label per sample.
    Anchors = the b*p rows, L2-normalised; for every anchor three log(1 + sum exp(neg - pos)) sums over (positive, negative)
    sets chosen by same/different attention and same/different class (:50-55), looped over anchors exactly as the reference."""
    b, p, _ = feats.shape
    n = b * p
    x = F.normalize(feats.reshape(n, -1), p=2, dim=1)                                  # :41-43
    t = torch.repeat_interleave(labels, p)                                             # :44
    parts = torch.arange(p, device=labels.device).repeat(b)                            # :45
    prod = x @ x.t()                                                                   # :46
    sc = t.expand(n, n).eq(t.expand(n, n).t())                                         # :50
    sa = parts.expand(n, n).eq(parts.expand(n, n).t())                                 # :51
    s_sasc, s_sadc, s_dasc, s_dadc = sc & sa, (~sc) & sa, sc & (~sa), (~sc) & (~sa)    # :53-56
    total = prod.new_zeros(())

    def term(pos, neg):                                                                # :64-70 (and :73-88)
        return torch.log(1 + torch.exp(neg[None, :] - pos[:, None]).sum(dim=1)).sum()
    for i in range(n):
        total = total + term(prod[i][s_sasc[i]], prod[i][s_sadc[i] | s_dasc[i] | s_dadc[i]])
        total = total + term(prod[i][s_sadc[i]], prod[i][s_dadc[i]])
        total = total + term(prod[i][s_dasc[i]], prod[i][s_dadc[i]])
    return total / n                                                                   # :90


def mamc_loss(pred, x_part, labels, lambda_a=0.5):
    """MAMCLoss.forward (MAMC_loss.py:15-21): CE(label_smoothing=0.1) + lambda_a * N-pairs."""
    return F.cross_entropy(pred, labels, label_smoothing=0.1) + lambda_a * npairs_loss(x_part, labels)


# --------------------------------------------------------------------------------------
# OSMENet: ResNet-101 trunk + OSME (model/methods/OSME.py:8-64)
# --------------------------------------------------------------------------------------
RESNET101_LAYERS = resnet_layers((3, 4, 23, 3))


def osme_forward(x, st, prefix='osme.', nl=Plain, linear=F.linear):
    """OSME.forward (OSME.py:36-44) on the trunk map x [N, C, H, W] -> (sum of the attention features [N, D], the features
    stacked [N, P, D]).  Each OSME_block.forward (:19-24): z = the spatial mean (:21), m = sigmoid(Linear(ReLU(Linear(z))))
    (:22, the Sequential of :12-17), s = m * x per channel (:23); then every attention's Linear over s flattened in NCHW
    order (:43).  The bottleneck ReLU goes through ``nl`` so that a MaskTape replays it; ``linear`` computes the
    attention Linears (a caller may evaluate them in row blocks)."""
    N, C = x.shape[:2]
    P = sum(1 for k in st if k.startswith(prefix + 'blocks.') and k.endswith('.block.0.weight'))
    s = []
    for i in range(P):                                                                 # :42
        pre = f'{prefix}blocks.{i}.block.'
        z = x.mean(dim=(2, 3))                                                         # :21
        h = nl.relu(F.linear(z, st[pre + '0.weight'], st[pre + '0.bias']))             # :22 (:13-14)
        m = torch.sigmoid(F.linear(h, st[pre + '2.weight'], st[pre + '2.bias']))       # :22 (:15-16)
        s.append(m.view(N, C, 1, 1) * x)                                               # :23
    feats = [linear(s[i].reshape(N, -1), st[f'{prefix}fcs.{i}.weight'], st[f'{prefix}fcs.{i}.bias'])
             for i in range(P)]                                                        # :43
    return sum(feats), torch.stack(feats, dim=1)                                       # :44


def osmenet_forward(x, st, nl=Plain, layers=RESNET101_LAYERS, linear=F.linear, bn=_bn_train):
    """OSMENet.forward (OSME.py:60-64): the ResNet trunk (children()[:-2], :55-56), OSME, the classifier on the sum of the
    attention features -> (logits, x_part).  Device- and dtype-agnostic: it runs wherever, and in whatever precision,
    x and st are."""
    f = resnet50_trunk_fwd(x, st, nl=nl, layers=layers, bn=bn)                         # :61
    x1, x_part = osme_forward(f, st, 'osme.', nl, linear)                              # :62
    return F.linear(x1, st['classifier.weight'], st['classifier.bias']), x_part       # :63-64
