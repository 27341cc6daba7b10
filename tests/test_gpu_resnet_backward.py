"""Backward and eval-mode parity of the ResNet trunk (hawkeye_b200/ops_resnet.py over csrc/resnet.cu, the GEMM and the 3x3
convolutions) against torch-CPU fp64, in the default single-pass TF32 mode that training runs in and in the 3xTF32 mode.

* Unit by unit: every conv + BN (+ residual) (+ ReLU) unit of a shallow trunk with real ResNet-50/101 widths, fed the fp64
  oracle's input for that unit, forward with save, then backward with a seeded dy (and a seeded addend on the 1x1 units:
  the fused dgrad epilogue for '1x1', the separate add for '1x1s2').  The reference is fp64 autograd of the same unit on the
  same fp32 inputs and weights, with the ReLU mask this forward produced (tests/matched.py explains why).
* The shallow trunk end to end through ResNetTrunkFn's autograd wiring, against the fp64 oracle on the recorded tape: features,
  every parameter gradient, the running statistics and the eval-mode (running statistics) forward.
* ResNet-101 (APINet's trunk) features against fp64, next to a stock PyTorch TF32 run of the same restatement.
"""
import subprocess

import pytest
import torch
import torch.nn.functional as F

import detgen
import matched
from conftest import rel_l2
from kernel_check import nchw, nhwc, precise  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu

SHALLOW = (2, 1, 1, 1)      # stem, 1x1 downsample at stride 1, an identity block, 3x3/s2 + 1x1/s2 units, layer4 at 7x7

# Per unit.  Default mode: the bound of the forward test (test_resnet_units_vs_oracle).  One unit's backward is two
# single-pass TF32 products (dgrad and wgrad, operands rounded to 2^-11, ~3e-4 rms) behind the BN backward, whose
# normalisation statistics already carry the forward's TF32 error; the worst measured on an H100 is 8.7e-4 (a 1x1 dw).
# Precise mode (3xTF32): the worst measured is 8.5e-6 (the 3x3/s2 dw, fp32 accumulation over the pixels).  5e-5 leaves 6x
# above that and stays 5x below the ~3e-4 that a single un-split TF32 operand anywhere in the unit would leave, so a precise
# path that drops to single-pass TF32 fails.
UNIT_TOL = {0: 2e-3, 1: 5e-5}


@pytest.fixture
def stock_tf32():
    """cuDNN / cuBLAS with TF32 allowed, as a stock PyTorch training run has it; the flags are restored afterwards."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _trunk(blocks):
    from hawkeye_b200.backbone.resnet import ResNetTrunk
    trunk = ResNetTrunk(blocks)
    st = detgen.state_like(trunk)
    trunk.load_state_dict(st)
    return trunk.cuda().train(), st


def _walk(trunk, st64, x, blocks):
    """-> (name of the unit's BN, Unit, fp64 input, fp64 residual or None) for every unit of the trunk in forward order.
    Each unit gets the fp64 oracle's input for it; the walk advances along the oracle's own (plain ReLU) forward."""
    from oracle import hop_oracle as O
    plan = trunk._plan
    yield '1', plan.stem, x, None
    cur = F.max_pool2d(F.relu(O._bn_train(F.conv2d(x, st64['0.weight'], stride=2, padding=3), st64, '1')), 3, 2, 1)
    bi = 0
    for li, (_, nblocks, stride) in enumerate(O.resnet_layers(blocks)):
        for b in range(nblocks):
            u1, u2, u3, ds = plan.blocks[bi]
            bi += 1
            pre, s = f'{4 + li}.{b}', (stride if b == 0 else 1)
            yield pre + '.bn1', u1, cur, None
            o1 = F.relu(O._bn_train(F.conv2d(cur, st64[pre + '.conv1.weight']), st64, pre + '.bn1'))
            yield pre + '.bn2', u2, o1, None
            o2 = F.relu(O._bn_train(F.conv2d(o1, st64[pre + '.conv2.weight'], stride=s, padding=1), st64, pre + '.bn2'))
            oid = cur
            if ds is not None:
                yield pre + '.downsample.1', ds, cur, None
                oid = O._bn_train(F.conv2d(cur, st64[pre + '.downsample.0.weight'], stride=s), st64, pre + '.downsample.1')
            yield pre + '.bn3', u3, o2, oid
            cur = F.relu(O._bn_train(F.conv2d(o2, st64[pre + '.conv3.weight']), st64, pre + '.bn3') + oid)


def _unit_errors(unit, x64, r64, seed):
    """Forward (save) + backward of one unit on the fp32 copy of its oracle input -> {quantity: rel-L2 against fp64}."""
    w, g, b = [p.detach() for p in unit.params()]
    x32 = x64.float()
    r32 = r64.float() if r64 is not None else None
    need_dx = unit.kind != 'stem'
    with torch.no_grad():
        xin = x32.cuda() if unit.kind == 'stem' else nhwc(x32).cuda()
        y, rec = unit.forward(xin, w, g, b, nhwc(r32).cuda() if r32 is not None else None, True)
    dy = detgen.det(y.shape, seed)                                  # NHWC, like y
    # fp64 reference on the same fp32 values, on the ReLU branch this forward took
    xd = x32.double().requires_grad_(need_dx)
    wd, gd, bd = (t.cpu().double().requires_grad_(True) for t in (w, g, b))
    rd = r32.double().requires_grad_(True) if r32 is not None else None
    z = F.batch_norm(F.conv2d(xd, wd, stride=unit.conv.stride, padding=unit.conv.padding), None, None, gd, bd,
                     training=True, eps=unit.bn.eps)
    if rd is not None:
        z = z + rd
    if unit.relu:
        z = z * nchw(y > 0).cpu().double()
    inputs = [wd, gd, bd] + ([xd] if need_dx else []) + ([rd] if rd is not None else [])
    ref = dict(zip(['dw', 'dgamma', 'dbeta'] + (['dx'] if need_dx else []) + (['dres'] if rd is not None else []),
                   torch.autograd.grad(z, inputs, nchw(dy).double())))
    # an addend of dx's own size on the 1x1 units: a dropped or doubled addend is an O(1) error, a wrong dx still shows
    addend = None
    if need_dx and unit.kind.startswith('1x1'):
        addend = detgen.det(ref['dx'].shape, seed + 1, ref['dx'].pow(2).mean().sqrt().item())
        ref['dx'] = ref['dx'] + addend.double()
    with torch.no_grad():
        dx, dres, dw, dg, db = unit.backward(rec, dy.cuda(), need_dx=need_dx,
                                             addend=nhwc(addend).cuda() if addend is not None else None)
    torch.cuda.synchronize()
    got = {'dw': dw, 'dgamma': dg, 'dbeta': db}
    if need_dx:
        got['dx'] = nchw(dx)
    if rd is not None:
        got['dres'] = nchw(dres)
    assert set(got) == set(ref)
    return {k: rel_l2(got[k].cpu(), ref[k]) for k in ref}


def _units(trunk, st, x, blocks, only=None):
    """-> {(BN name, kind): {quantity: error}} over the trunk's units (or those whose BN name is in `only`)."""
    st64 = {k: v.double() for k, v in st.items()}
    out = {}
    for i, (name, unit, x64, r64) in enumerate(_walk(trunk, st64, x.double(), blocks)):
        if only is None or name in only:
            out[(name, unit.kind)] = _unit_errors(unit, x64, r64, 700 + 10 * i)
            if only is not None and len(out) == len(only):
                break
    return out


def _by_kind(errs):
    """worst (error, unit, quantity) per unit kind"""
    worst = {}
    for (name, kind), e in errs.items():
        q = max(e, key=e.get)
        if kind not in worst or e[q] > worst[kind][0]:
            worst[kind] = (e[q], name, q)
    return worst


@pytest.mark.parametrize('size,precise', [(224, 0), (224, 1), (448, 0)], indirect=['precise'])
def test_unit_backward(size, precise):
    """224x224 / batch 2: every unit of the shallow trunk.  448x448: the layer1 3x3 at 112x112, the only ResNet map the v2
    forward kernel takes (W % 16 == 0, default mode only)."""
    torch.set_num_threads(16)
    trunk, st = _trunk(SHALLOW)
    x = detgen.det((2, 3, size, size), 61)
    errs = _units(trunk, st, x, SHALLOW, only=None if size == 224 else ['4.0.bn2'])
    worst = _by_kind(errs)
    print(f'unit backward {size}x{size} precise={precise}, worst per kind: ' +
          ', '.join(f'{k} {v[0]:.2e} ({v[1]} {v[2]})' for k, v in sorted(worst.items())))
    bad = {k: e for k, e in errs.items() if not max(e.values()) < UNIT_TOL[precise]}
    assert len(errs) == (20 if size == 224 else 1) and not bad, bad


# Shallow trunk end to end.  Every gradient is formed from forward activations that have passed up to 16 units (the stem,
# then 3 per block), each adding at most UNIT_TOL[0] = 2e-3 of its own, and a random-weight train-mode ResNet amplifies a
# perturbation ~1.3x per bottleneck (test_resnet_units_vs_oracle).  Independent unit errors then add in quadrature with
# gains 1.3^(blocks after the unit): sqrt(1.3^10 + 3 (1 + 1.3^2 + ... + 1.3^8)) = 8.3, so 8.3 x 2e-3 = 1.7e-2, rounded up
# to 2e-2, bounds the default mode; the amplification measured on an H100 (worst trunk gradient over worst unit error) is
# 7.7x.  A plumbing bug (a dropped identity gradient, a wrong stride adjoint, a missing BN term) moves gradients by O(1).
# Precise mode: the matched-activation bound of test_gpu_matched.py.
TRUNK_TOL = {0: 2e-2, 1: 2e-4}


def _oracle_trunk(st, x, G, blocks, tape):
    """fp64 oracle forward on the recorded tape, loss (feat * G).sum() -> (feat, {param: grad}, {BN name: batch stats})"""
    from oracle import hop_oracle as O
    st64 = {k: (v.double().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v)
            for k, v in st.items()}
    stats = {}

    def bn(z, s, pre):
        stats[pre] = O.bn_batch_stats(z.detach())
        return O._bn_train(z, s, pre)
    feat = O.resnet50_trunk_fwd(x.double(), st64, prefix='', nl=tape, layers=O.resnet_layers(blocks), bn=bn)
    keys = [k for k, v in st64.items() if v.requires_grad]
    grads = torch.autograd.grad((feat * G.double()).sum(), [st64[k] for k in keys])
    return feat.detach(), dict(zip(keys, grads)), stats


def _bn_modules(trunk):
    return {name: m for name, m in trunk.named_modules() if isinstance(m, torch.nn.BatchNorm2d)}


@pytest.mark.parametrize('precise', [0, 1], indirect=True)
def test_shallow_trunk_train_and_eval(precise):
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    torch.set_num_threads(16)
    tol = TRUNK_TOL[precise]
    trunk, st = _trunk(SHALLOW)
    x = detgen.det((2, 3, 224, 224), 61)

    # ---- one train step through ResNetTrunkFn (forward with the decision capture, backward of (feat * G).sum())
    ops.CAPTURE = []
    try:
        feat = trunk(x.cuda())
        cap = ops.CAPTURE
    finally:
        ops.CAPTURE = None
    G = detgen.det(feat.shape, 62)
    trunk.zero_grad(set_to_none=True)
    (feat * G.cuda()).sum().backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu() for k, p in trunk.named_parameters()}
    tape = O.MaskTape(matched.tape_items(cap))
    ref_feat, ref, stats = _oracle_trunk(st, x, G, SHALLOW, tape)
    assert tape.done(), 'oracle consumed fewer decisions than the GPU forward recorded'
    ef = rel_l2(feat.detach().cpu(), ref_feat)
    print(f'shallow trunk precise={precise}: features rel {ef:.2e}')
    assert len(grads) == len(ref) == len(list(trunk.parameters()))
    errs = matched.compare_grads(grads, ref, tol, f'shallow trunk precise={precise}')
    assert ef < tol

    # ---- running statistics after that step: momentum 0.1 from (0, 1); the mean's error in units of the batch spread
    bns = _bn_modules(trunk)
    assert set(bns) == set(stats)
    worst_m = worst_v = 0.0
    for name, m in bns.items():
        mean, var, unb = stats[name]
        assert int(m.num_batches_tracked) == 1, name
        worst_m = max(worst_m, ((m.running_mean.cpu().double() - 0.1 * mean).abs() / (0.1 * var.sqrt())).max().item())
        worst_v = max(worst_v, rel_l2(m.running_var.cpu(), 0.9 + 0.1 * unb))
    print(f'shallow trunk precise={precise}: running mean {worst_m:.2e} (batch sigmas), running var {worst_v:.2e}')
    assert worst_m < tol and worst_v < tol

    # ---- per-unit errors on the same batch, for the amplification through the trunk
    unit_worst = max(max(e.values()) for e in _units(trunk, st, x, SHALLOW).values())
    print(f'shallow trunk precise={precise}: worst gradient {max(errs.values()):.2e}, worst unit {unit_worst:.2e}, '
          f'amplification {max(errs.values()) / unit_worst:.1f}x')

    # ---- eval mode: running statistics = the fp64 batch statistics of a second batch (activations stay at training scale)
    x2 = detgen.det((2, 3, 224, 224), 63)
    st64 = {k: (v.double() if v.is_floating_point() else v) for k, v in st.items()}
    stats2 = {}

    def record(z, s, pre):
        stats2[pre] = O.bn_batch_stats(z)
        return O._bn_train(z, s, pre)
    O.resnet50_trunk_fwd(x2.double(), st64, prefix='', layers=O.resnet_layers(SHALLOW), bn=record)
    for name, m in bns.items():
        m.running_mean.copy_(stats2[name][0].float())
        m.running_var.copy_(stats2[name][1].float())
        st64[name + '.running_mean'], st64[name + '.running_var'] = stats2[name][0], stats2[name][1]
    trunk.eval()
    with torch.no_grad():
        feat_e = trunk(x2.cuda()).cpu()
    ref_e = O.resnet50_trunk_fwd(x2.double(), st64, prefix='', layers=O.resnet_layers(SHALLOW), bn=O._bn_eval)
    ee = rel_l2(feat_e, ref_e)
    print(f'shallow trunk precise={precise}: eval-mode features rel {ee:.2e}')
    assert ee < tol


def _gpu_name_and_power():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ', power limit unknown'
    return out


def test_resnet101_features_vs_stock_tf32(stock_tf32):
    """APINet's trunk at 224x224 / batch 4, train mode, default precision: the pooled features of the library and of the
    same restatement run by stock PyTorch in fp32 with TF32 allowed, each against fp64 on the CPU.  A random-weight
    train-mode ResNet-101 amplifies any rounding a lot (see test_resnet_units_vs_oracle), so neither is close to fp64;
    the library must not be more than 2x further from it than the stock run is."""
    from oracle import hop_oracle as O
    from hawkeye_b200 import _lib
    torch.set_num_threads(16)
    assert not _lib.get_precise()
    blocks = (3, 4, 23, 3)
    trunk, st = _trunk(blocks)
    x = detgen.det((4, 3, 224, 224), 64)
    layers = O.resnet_layers(blocks)
    with torch.no_grad():
        ours = trunk(x.cuda()).mean(dim=(2, 3)).cpu()
        stdev = {k: v.cuda() for k, v in st.items()}
        stock = O.resnet50_trunk_fwd(x.cuda(), stdev, prefix='', layers=layers).mean(dim=(2, 3)).cpu()
        exact = O.resnet50_trunk_fwd(x.double(), {k: (v.double() if v.is_floating_point() else v) for k, v in st.items()},
                                     prefix='', layers=layers).mean(dim=(2, 3))
    e_ours, e_stock, e_between = rel_l2(ours, exact), rel_l2(stock, exact), rel_l2(ours, stock)
    print(f'resnet101 224x224 batch 4 pooled features, rel-L2 vs fp64: library {e_ours:.2e}, stock TF32 {e_stock:.2e}; '
          f'library vs stock {e_between:.2e} ({_gpu_name_and_power()})')
    assert e_ours <= 2 * e_stock
