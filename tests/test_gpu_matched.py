"""Gradient parity of the three models, EVERY parameter, including the benchmark 448x448 / batch-2 configuration.

Two complementary checks (tests/matched.py explains why a plain comparison cannot work for a TF32 forward):
  * matched-activation: the fp64 oracle is evaluated on the branch (ReLU masks, pool arg-maxes, signed-sqrt bins) the GPU
    forward took.  Default TF32 mode: <= 3e-3 (the accumulated rounding of ~17 chained single-pass TF32 products; a
    plumbing bug is O(1)).  Precise mode (hk_set_precise(1), 3xTF32 on the same kernels): <= 2e-4.
  * reference fixtures: precise mode against logits / loss / gradients of the UNMODIFIED fp32 reference
    (tests/golden/reference_448.npz, made by tests/golden/make_golden_448.py): logits, loss and the head gradients at
    1e-3; backbone gradients at 1e-3 + 8u, where u (stored in the fixture) is how far the reference's own fp32 gradient is
    from an exact fp64 evaluation — its own rounding flips ReLU / pool decisions, up to 4e-3 at conv1_1.
The 64x64 input (a 2x2 feature map, HW = 4 << C) is a badly conditioned bilinear backward — a 8e-4 forward difference
becomes 6e-3 in d(features) — so that size is asserted in precise mode only.
"""
import os

import numpy as np
import pytest
import torch

import detgen
import matched
from matched import TOL
from conftest import rel_l2
from kernel_check import precise  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu


class Cfg(dict):
    __getattr__ = dict.__getitem__


@pytest.fixture(scope='module')
def ref448():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_448.npz'))


@pytest.fixture(scope='module')
def ref224():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_224.npz'))


def _bcnn(stage=2):
    import hawkeye_b200 as hb
    from oracle import hop_oracle as O
    net = hb.MODEL.get('BCNN')(Cfg(name='BCNN', stage=stage, num_classes=200))
    state = detgen.vgg_bcnn_state(O.VGG16_D, 200, seed=100)
    net.load_state_dict(state)
    return net.cuda().train(), state


def _cbcnn(d):
    import hawkeye_b200 as hb
    from oracle import hop_oracle as O
    net = hb.MODEL.get('CBCNN')(Cfg(name='CBCNN', stage=2, num_classes=200, input_channel=512, output_channel=d))
    state = detgen.vgg_bcnn_state(O.VGG16_D, 200, seed=100, head_in=d)
    net.load_state_dict(state)
    return net.cuda().train(), state


def _mpn():
    import hawkeye_b200 as hb
    net = hb.MODEL.get('MPN')(Cfg(name='MPN', iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048,
                                  dimension_reduction=256, num_classes=200))
    state = detgen.state_like(net)
    net.load_state_dict(state)
    return net.cuda().train(), state


@pytest.mark.parametrize('size,precise', [(64, 1), (448, 0), (448, 1)], indirect=['precise'])
def test_bcnn_s2_all_gradients(size, precise):
    from oracle import hop_oracle as O
    torch.set_num_threads(16)
    net, state = _bcnn()
    x, labels = detgen.det((2, 3, size, size), 41), detgen.det_labels(2, 200, 42)
    logits, loss, grads, items = matched.gpu_step(net, x, labels)
    ref_logits, ref_loss, ref = matched.oracle_step(lambda xx, st, nl: O.bcnn_forward(xx, st, 2, nl=nl), x, labels, state,
                                                    items, grads.keys())
    e = rel_l2(logits, ref_logits)
    print(f'bcnn {size} precise={precise}: logits rel {e:.2e} loss {loss:.6f} vs {ref_loss:.6f}')
    assert len(grads) == 28 and e < 1e-3 and abs(loss - ref_loss) < 1e-4
    matched.compare_grads(grads, ref, TOL[precise], f'bcnn_s2 {size}x{size} precise={precise}')


@pytest.mark.parametrize('precise', [0, 1], indirect=True)
@pytest.mark.parametrize('size,d', [(128, 8192), (448, 8192), (448, 6000)])
def test_cbcnn_all_gradients(size, d, precise):
    from oracle import hop_oracle as O
    torch.set_num_threads(16)
    net, state = _cbcnn(d)
    x, labels = detgen.det((2, 3, size, size), 41), detgen.det_labels(2, 200, 42)
    logits, loss, grads, items = matched.gpu_step(net, x, labels)
    ref_logits, ref_loss, ref = matched.oracle_step(lambda xx, st, nl: O.cbcnn_forward(xx, st, d, 2, nl=nl), x, labels,
                                                    state, items, grads.keys())
    e = rel_l2(logits, ref_logits)
    print(f'cbcnn {size} d={d} precise={precise}: logits rel {e:.2e} loss {loss:.6f} vs {ref_loss:.6f}')
    assert len(grads) == 28 and e < 1e-3 and abs(loss - ref_loss) < 1e-4
    matched.compare_grads(grads, ref, TOL[precise], f'cbcnn {size}x{size} d={d} precise={precise}')


@pytest.mark.parametrize('precise', [1], indirect=True)
@pytest.mark.parametrize('size,B', [(128, 4), (448, 2)])
def test_mpn_all_gradients(size, B, precise):
    """A random-weight train-mode ResNet-50 amplifies a perturbation of its input ~170x by the last block (measured in fp64),
    so single-pass TF32 (5e-4 per layer) cannot track ANY reference run of it; the 3xTF32 mode can.
    fp32 itself is only reproducible to ~2e-4 here (fp32 vs fp64 oracle on the same branch), hence the looser bound."""
    from oracle import hop_oracle as O
    torch.set_num_threads(16)
    net, state = _mpn()
    x, labels = detgen.det((B, 3, size, size), 51), detgen.det_labels(B, 200, 52)
    logits, loss, grads, items = matched.gpu_step(net, x, labels)
    ref_logits, ref_loss, ref = matched.oracle_step(lambda xx, st, nl: O.mpn_forward(xx, st, 5, nl=nl), x, labels, state,
                                                    items, grads.keys())
    e = rel_l2(logits, ref_logits)
    print(f'mpn {size} B={B} precise={precise}: logits rel {e:.2e} loss {loss:.6f} vs {ref_loss:.6f}')
    assert len(grads) == len(list(net.parameters()))
    errs = matched.compare_grads(grads, ref, 1e-3, f'mpn {size}x{size} precise={precise}')
    assert e < 1e-3 and abs(loss - ref_loss) < 1e-4, (e, errs)


# ------------------------------------------------------------------------------------------------------------------
# precise mode vs the UNMODIFIED reference at the benchmark configuration (fixtures: tests/golden/make_golden_448.py)
# ------------------------------------------------------------------------------------------------------------------
def _slice_like(g, k, ref):
    """apply the fixture's slicing rule to a full gradient"""
    if k.endswith('classifier.weight_slice'):
        return g[:, ::(4099 if g.shape[1] == 512 * 512 else 61)]
    if k.endswith('weight_slice'):
        if g.dim() == 4 and g.shape[2] == 1:
            return g[:, ::8, 0, 0] if 'conv_dr_block' in k else g[::4, ::4, 0, 0]
        return g[::8, ::8] if 'backbone.5.0' not in k else g[::4, ::4]
    return g


def _check_fixture(tag, ref448, logits, loss, grads, tol=1e-3):
    e = rel_l2(logits, ref448[f'{tag}_logits'])
    print(f'{tag}: logits rel {e:.2e} loss {loss:.6f} vs {float(ref448[f"{tag}_loss"]):.6f}')
    assert e < tol and abs(loss - float(ref448[f'{tag}_loss'])) < 1e-4
    errs, bad = {}, {}
    for key in ref448.files:
        if not key.startswith(tag + '_g_'):
            continue
        name = key[len(tag) + 3:]
        pname = name[:-len('_slice')] if name.endswith('_slice') else name
        err = rel_l2(_slice_like(grads[pname], name, ref448[key]), ref448[key])
        # u: the reference's own distance from an exact evaluation (branch flips caused by ITS fp32 rounding, ~1e-6 forward
        # noise).  Flip-induced error grows like sqrt(forward noise); the 3xTF32 forward carries ~2e-5 (operand split plus the
        # tensor core's truncating fp32 accumulation), i.e. ~sqrt(20) ~ 4.5 u on average; flips are discrete events, so
        # the bound leaves headroom: 1e-3 + 8 u.
        bound = tol + 8 * float(ref448[f'{tag}_u_{name}'])
        errs[name] = (err, bound)
        if not err < bound:
            bad[name] = (err, bound)
    print(f'{tag}: {len(errs)} reference gradients (err / bound): ' +
          ', '.join(f'{k} {v[0]:.1e}/{v[1]:.1e}' for k, v in sorted(errs.items(), key=lambda kv: -kv[1][0] / kv[1][1])[:6]))
    assert errs and not bad, bad


@pytest.mark.parametrize('precise', [1], indirect=True)
@pytest.mark.parametrize('stage', [1, 2])
def test_bcnn_448_vs_reference(stage, precise, ref448):
    net, _ = _bcnn(stage)
    x, labels = detgen.det((2, 3, 448, 448), 41), detgen.det_labels(2, 200, 42)
    logits, loss, grads, _ = matched.gpu_step(net, x, labels)
    _check_fixture(f'bcnn_s{stage}', ref448, logits, loss, grads)
    if stage == 1:
        assert set(grads) == {'classifier.weight', 'classifier.bias'}


@pytest.mark.parametrize('precise', [1], indirect=True)
@pytest.mark.parametrize('d', [8192, 6000])
def test_cbcnn_448_vs_reference(d, precise, ref448):
    """Logits, loss and the classifier gradients at 1e-3.  The backbone gradients pass through the signed square root
    d/dv = 1/(2 sqrt(|v|+1e-10)) of 2*d sketch bins: a relative perturbation eps of the Gram changes them by ~1000 eps
    (tests/diag/cbp_sensitivity.py: 3e-7 -> 3e-4), and the tensor core's truncating fp32 accumulation leaves ~2e-5 in
    the 3xTF32 forward, so against the fp32 reference they are only bounded at 5e-2 here; the matched test above pins
    them at 2e-4 with the derivative taken at the bins this forward produced."""
    net, _ = _cbcnn(d)
    x, labels = detgen.det((2, 3, 448, 448), 41), detgen.det_labels(2, 200, 42)
    logits, loss, grads, _ = matched.gpu_step(net, x, labels)
    tag = f'cbcnn_{d}'
    e = rel_l2(logits, ref448[f'{tag}_logits'])
    print(f'{tag}: logits rel {e:.2e} loss {loss:.6f} vs {float(ref448[f"{tag}_loss"]):.6f}')
    assert e < 1e-3 and abs(loss - float(ref448[f'{tag}_loss'])) < 1e-4
    assert rel_l2(grads['classifier.bias'], ref448[f'{tag}_g_classifier.bias']) < 1e-3
    assert rel_l2(grads['classifier.weight'][:, ::61], ref448[f'{tag}_g_classifier.weight_slice']) < 1e-3
    errs = {k: rel_l2(grads[k], ref448[f'{tag}_g_{k}']) for k in ('backbone.0.bias', 'backbone.14.bias', 'backbone.28.bias')}
    print(tag, {k: f'{v:.2e}' for k, v in errs.items()})
    assert max(errs.values()) < 5e-2


@pytest.mark.parametrize('precise', [1], indirect=True)
def test_mpn_448_vs_reference(precise, ref448):
    net, _ = _mpn()
    x, labels = detgen.det((2, 3, 448, 448), 51), detgen.det_labels(2, 200, 52)
    logits, loss, grads, _ = matched.gpu_step(net, x, labels)
    _check_fixture('mpn', ref448, logits, loss, grads)


# ------------------------------------------------------------------------------------------------------------------
# 224x224 inputs: 7x7 feature maps, H*W = 49 is not a multiple of 4 (the reference's stock MPN / CBCNN / PeerLearning
# configs).  The pooling heads zero-pad the map to a 16-byte row pitch; results must be those of the reference.
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precise', [0, 1], indirect=True)
@pytest.mark.parametrize('model', ['bcnn_s2', 'cbcnn_6000', 'mpn'])
def test_224_vs_reference(model, precise, ref224):
    if model == 'bcnn_s2':
        net, _ = _bcnn(2)
        x, labels = detgen.det((2, 3, 224, 224), 41), detgen.det_labels(2, 200, 42)
    elif model == 'cbcnn_6000':
        net, _ = _cbcnn(6000)
        x, labels = detgen.det((2, 3, 224, 224), 41), detgen.det_labels(2, 200, 42)
    else:
        net, _ = _mpn()
        x, labels = detgen.det((2, 3, 224, 224), 51), detgen.det_labels(2, 200, 52)
    logits, loss, grads, _ = matched.gpu_step(net, x, labels)
    e = rel_l2(logits, ref224[f'{model}_logits'])
    eb = rel_l2(grads['classifier.bias'], ref224[f'{model}_g_classifier.bias'])
    print(f'{model} 224 precise={precise}: logits rel {e:.2e} loss {loss:.6f} vs {float(ref224[f"{model}_loss"]):.6f} '
          f'classifier.bias grad {eb:.2e}')
    if model == 'mpn' and not precise:
        return        # single-pass TF32 cannot track a random-weight train-mode ResNet-50 (see test_mpn_all_gradients)
    assert e < 1e-3 and abs(loss - float(ref224[f'{model}_loss'])) < 1e-4 and eb < (2e-3 if not precise else 1e-3)
    if precise:
        _check_fixture(model, ref224, logits, loss, grads) if model != 'cbcnn_6000' else None
