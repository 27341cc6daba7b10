"""Compact bilinear pooling + CBCNN vs the oracle and the reference-generated fixtures."""
import hashlib

import numpy as np
import pytest
import torch

import detgen
from conftest import rel_l2


def test_hashes_bit_exact(golden):
    """CPU: the count-sketch hash/sign vectors are bit-identical to the reference's numpy streams (CBCNN.py:76-91)."""
    from hawkeye_b200 import ops
    for d in (8192, 6000):
        hs = ops.count_sketch_hashes(512, d)
        for name, arr in zip(('h1', 's1', 'h2', 's2'), hs):
            assert np.array_equal(arr, golden[f'cbp_{name}_{d}'])
        sha = hashlib.sha256(np.concatenate(hs).astype(np.int64).tobytes())
        assert np.array_equal(np.frombuffer(sha.digest(), dtype=np.uint8), golden[f'cbp_hash_sha256_{d}'])
    assert hashlib.sha256(np.concatenate(ops.count_sketch_hashes(512, 8192)).astype(np.int64).tobytes()).hexdigest() \
        == '5fe0585bec221dd6600895705b0748dc12d9459156708dcbb58046d0bdf1e314'


@pytest.mark.gpu
@pytest.mark.parametrize('d', [8192, 6000])
def test_cbp_golden(golden, d):
    from hawkeye_b200.methods.cbcnn import CompactBilinearPooling
    # fixture shape is 3x3 (HW=9, not a multiple of 4): embed it in a zero-padded 3x4 map — zero columns add nothing
    x = detgen.det_uniform((2, 512, 3, 3), 21)
    xp = torch.zeros(2, 512, 3, 4)
    xp[..., :3] = x
    xg = xp.cuda().requires_grad_(True)
    y = CompactBilinearPooling(512, 512, d)(xg)
    e = rel_l2(y.detach().cpu(), golden[f'cbp_y_{d}'])
    (dx,) = torch.autograd.grad(y, xg, detgen.det(y.shape, 22).cuda())
    eb = rel_l2(dx.cpu()[..., :3], golden[f'cbp_dx_{d}'])
    print(f'cbp d={d}: fwd {e:.2e} bwd {eb:.2e} (arbitrary fp32 inputs: operands are truncated to tf32)')
    assert e < 1e-3
    # The signed-sqrt gradient 1/(2 sqrt(|v|+1e-10)) is ill-conditioned near empty bins: with arbitrary
    # fp32 inputs the tf32 operand truncation perturbs near-zero bins and their gradients by O(1), so dX is only
    # compared in direction here ...
    a, b = dx.cpu()[..., :3].double().flatten(), torch.as_tensor(golden[f'cbp_dx_{d}']).double().flatten()
    cos = (a @ b / (a.norm() * b.norm())).item()
    print(f'cbp d={d}: dX cosine {cos:.4f}')
    assert cos > 0.9
    # ... and tightly on TF32-representable inputs (what the op sees inside the model, where the trunk rounds its
    # activations to tf32): the tensor-core Gram is then exact up to fp32 summation order.
    xt = detgen.tf32_rna(detgen.det_uniform((2, 512, 3, 4), 23)).cuda().requires_grad_(True)
    yt = CompactBilinearPooling(512, 512, d)(xt)
    (dxt,) = torch.autograd.grad(yt, xt, detgen.det(yt.shape, 24).cuda())
    et, ebt = rel_l2(yt.detach().cpu(), golden[f'cbp_tf32in_y_{d}']), rel_l2(dxt.cpu(), golden[f'cbp_tf32in_dx_{d}'])
    print(f'cbp d={d} tf32-representable inputs: fwd {et:.2e} bwd {ebt:.2e}')
    assert et < 1e-3 and ebt < 5e-3


@pytest.mark.gpu
def test_cbp_vs_oracle_14x14():
    from hawkeye_b200.methods.cbcnn import CompactBilinearPooling
    from oracle import hop_oracle as O
    x = detgen.det_uniform((2, 512, 14, 14), 5)
    xg = x.cuda().requires_grad_(True)
    y = CompactBilinearPooling(512, 512, 8192)(xg)
    y_ref = O.cbp_fwd(x.double(), 8192)
    e = rel_l2(y.detach().cpu(), y_ref)
    print('cbp 14x14 fwd', e)
    assert e < 1e-3
    n = y.norm(dim=1)
    assert torch.allclose(n, torch.ones_like(n), atol=1e-4)


@pytest.mark.gpu
def test_cbcnn_model_golden(golden):
    import hawkeye_b200 as hb
    from hawkeye_b200 import ops
    from oracle.hop_oracle import VGG16_D

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    # 128x128 input -> 4x4 feature map (HW=16)
    net = hb.MODEL.get('CBCNN')(Cfg(name='CBCNN', stage=2, num_classes=200, input_channel=512, output_channel=8192))
    net.load_state_dict(detgen.vgg_bcnn_state(VGG16_D, 200, seed=100, head_in=8192))
    net = net.cuda().train()
    logits = net(detgen.det((2, 3, 128, 128), 41).cuda())
    loss = ops.CrossEntropyLS(0.1)(logits, detgen.det_labels(2, 200, 42).cuda())
    loss.backward()
    e = rel_l2(logits.detach().cpu(), golden['cbcnn_logits'])
    print(f'cbcnn logits rel {e:.2e} loss {loss.item():.6f} vs {float(golden["cbcnn_loss"]):.6f}')
    assert e < 1e-3 and abs(loss.item() - float(golden['cbcnn_loss'])) < 1e-4
    assert net.backbone[28].bias.grad is not None
