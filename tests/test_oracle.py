"""Pin the oracle restatement (oracle/hop_oracle.py) against outputs of the UNMODIFIED reference
(tests/golden/reference_outputs.npz, made by tests/golden/make_golden.py) and the numpy-RNG
known answers of the reference streams.  CPU only."""
import hashlib

import numpy as np
import torch

import detgen
from conftest import rel_l2
from oracle import hop_oracle as O


def test_cbp_hash_known_answers(golden):
    # Known answers (numpy legacy RNG, seeds 1/3/5/7 — CBCNN.py:76-91): bit-exact
    h1, s1, h2, s2 = O.cbp_hashes(512, 8192)
    assert h1[:8].tolist() == [5157, 235, 3980, 5192, 7935, 905, 2763, 7813]
    assert s1[:8].tolist() == [-1, -1, 1, 1, -1, -1, -1, 1]
    assert h2[:8].tolist() == [2915, 2254, 4079, 1725, 3046, 7286, 5520, 2121]
    assert s2[:8].tolist() == [1, -1, 1, -1, 1, 1, 1, 1]
    sha = hashlib.sha256(np.concatenate([h1, s1, h2, s2]).astype(np.int64).tobytes()).hexdigest()
    assert sha == '5fe0585bec221dd6600895705b0748dc12d9459156708dcbb58046d0bdf1e314'
    g1, _, g2, _ = O.cbp_hashes(512, 6000)
    assert g1[:8].tolist() == [5157, 235, 3980, 5192, 905, 2763, 2895, 5056]
    assert g2[:8].tolist() == [2915, 2254, 4079, 1725, 3046, 5520, 2121, 1032]
    for d in (8192, 6000):
        hs = O.cbp_hashes(512, d)
        for name, arr in zip(('h1', 's1', 'h2', 's2'), hs):
            assert np.array_equal(arr, golden[f'cbp_{name}_{d}'])
        sha = hashlib.sha256(np.concatenate(hs).astype(np.int64).tobytes()).digest()
        assert np.array_equal(np.frombuffer(sha, dtype=np.uint8), golden[f'cbp_hash_sha256_{d}'])


def test_bilinear_pool_matches_reference(golden):
    for tag, shape in (('bp_small', (2, 32, 4, 7)), ('bp_c128', (2, 128, 14, 14))):
        x = detgen.det_uniform(shape, 11)
        y = O.bilinear_pool_fwd(x)
        assert rel_l2(y, golden[f'{tag}_y']) < 1e-6
        dx = O.bilinear_pool_bwd(x, detgen.det(y.shape, 12))
        assert rel_l2(dx, golden[f'{tag}_dx']) < 2e-5
    x = detgen.det_uniform((1, 512, 14, 14), 13)
    y = O.bilinear_pool_fwd(x)
    assert rel_l2(y[0, ::997], golden['bp_full_y_slice']) < 1e-6
    assert abs(y.double().sum().item() - float(golden['bp_full_y_sum'])) < 1e-2
    assert abs(y.norm().item() - 1.0) < 1e-5
    dx = O.bilinear_pool_bwd(x, detgen.det(y.shape, 14))
    assert rel_l2(dx, golden['bp_full_dx']) < 1e-4


def test_bilinear_norm_closed_form():
    # ||z||^2 = sum_p (sum_c x_cp)^2 / HW + C^2 * 1e-5 — what kernel K0 computes
    x = detgen.det_uniform((2, 64, 5, 5), 3).double()
    xf = x.reshape(2, 64, 25)
    z2 = (torch.bmm(xf, xf.transpose(1, 2)) / 25 + 1e-5).reshape(2, -1).sum(1)
    cf = (xf.sum(1) ** 2).sum(1) / 25 + 64 * 64 * 1e-5
    assert torch.allclose(z2, cf, rtol=1e-12)


def test_cbp_matches_reference(golden):
    for d in (8192, 6000):
        x = detgen.det_uniform((2, 512, 3, 3), 21)
        y = O.cbp_fwd(x, d)
        assert rel_l2(y, golden[f'cbp_y_{d}']) < 1e-5
        # Gram-scatter identity == FFT route (what kernel K2 uses)
        pre = O.cbp_presqrt_gram_scatter(x.double(), d)
        y2 = torch.nn.functional.normalize(torch.sign(pre) * torch.sqrt(pre.abs() + 1e-10))
        assert rel_l2(y2, golden[f'cbp_y_{d}']) < 1e-4


def test_mpncov_matches_reference(golden):
    for tag, shape, it in (('mpn_small', (2, 16, 3, 3), 5), ('mpn_it3', (2, 24, 4, 4), 3), ('mpn_c256', (1, 256, 14, 14), 5)):
        x = detgen.det_uniform(shape, 31)
        c = O.covpool_fwd(x)
        assert rel_l2(c, golden[f'{tag}_cov']) < 1e-5
        s, saved = O.sqrtm_fwd(c, it)
        assert rel_l2(s, golden[f'{tag}_sqrt']) < 1e-4
        v = O.triuvec_fwd(s)
        assert v.shape == (shape[0], shape[1] * (shape[1] + 1) // 2, 1)
        if f'{tag}_vec' in golden:
            assert rel_l2(v, golden[f'{tag}_vec']) < 1e-4
        dx = O.mpncov_pool_bwd(x, detgen.det(v.shape, 32), it)
        assert rel_l2(dx, golden[f'{tag}_dx']) < 2e-3, tag


def test_bcnn_model_matches_reference(golden):
    torch.set_num_threads(8)
    state = detgen.vgg_bcnn_state(O.VGG16_D, 200, seed=100)
    x = detgen.det((2, 3, 64, 64), 41)
    labels = detgen.det_labels(2, 200, 42)
    for stage in (1, 2):
        keys = None if stage == 2 else {'classifier.weight', 'classifier.bias'}
        logits, loss, grads = O.loss_and_grads(lambda xx, st: O.bcnn_forward(xx, st, stage), x, labels, state, keys)
        assert rel_l2(logits, golden[f'bcnn_s{stage}_logits']) < 1e-5
        assert abs(loss.item() - float(golden[f'bcnn_s{stage}_loss'])) < 1e-5
        assert rel_l2(grads['classifier.bias'], golden[f'bcnn_s{stage}_gb']) < 1e-4
        assert rel_l2(grads['classifier.weight'][:, ::4099], golden[f'bcnn_s{stage}_gW_slice']) < 1e-4
        if stage == 2:
            assert rel_l2(grads['backbone.0.weight'], golden['bcnn_s2_g_backbone.0.weight']) < 1e-3
            assert rel_l2(grads['backbone.28.bias'], golden['bcnn_s2_g_backbone.28.bias']) < 1e-3


def test_cbcnn_model_matches_reference(golden):
    torch.set_num_threads(8)
    state = detgen.vgg_bcnn_state(O.VGG16_D, 200, seed=100, head_in=8192)
    x = detgen.det((2, 3, 128, 128), 41)
    labels = detgen.det_labels(2, 200, 42)
    logits, loss, grads = O.loss_and_grads(lambda xx, st: O.cbcnn_forward(xx, st, 8192, 2), x, labels, state)
    assert rel_l2(logits, golden['cbcnn_logits']) < 1e-4
    assert abs(loss.item() - float(golden['cbcnn_loss'])) < 1e-5
    assert rel_l2(grads['backbone.28.bias'], golden['cbcnn_g_backbone.28.bias']) < 5e-3


def test_mpn_model_matches_reference():
    """ResNet-50 trunk + MPN-COV head restatement vs the UNMODIFIED reference (tests/golden/reference_mpn.npz)."""
    import os
    torch.set_num_threads(8)
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_mpn.npz'))
    import hawkeye_b200 as hb

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    net = hb.MODEL.get('MPN')(Cfg(name='MPN', iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048,
                                  dimension_reduction=256, num_classes=200))
    st = detgen.state_like(net)          # same keys/shapes as the reference model => same deterministic values
    x = detgen.det((4, 3, 128, 128), 51)
    labels = detgen.det_labels(4, 200, 52)
    feat = O.resnet50_trunk_fwd(x, st)
    assert rel_l2(feat[:, ::16], g['feat_slice']) < 1e-4
    logits = O.mpn_forward(x, st)
    assert rel_l2(logits, g['logits']) < 1e-3
    assert abs(O.cross_entropy_ls(logits, labels).item() - float(g['loss'])) < 1e-4
