"""Generate golden fixtures by running the UNMODIFIED reference (imported through oracle/ref_harness: $HAWKEYE_REF or baseline/_ref).

Run here (authoring container) only:  python tests/golden/make_golden.py
Machines without the reference tree run the tests from the committed .npz files.
Inputs are regenerated from tests/detgen.py seeds, so fixtures carry outputs only.
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from conftest import save_golden  # noqa: E402

from oracle import ref_harness as rh  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
from model.methods.BCNN import BilinearPooling  # noqa: E402
from model.methods.CBCNN import CompactBilinearPooling  # noqa: E402
from model.methods.MPNCOV import Covpool, Sqrtm, Triuvec, MPNCOV  # noqa: E402
from model.registry import MODEL  # noqa: E402

torch.set_num_threads(8)
out = {}

# ---- bilinear pooling (BCNN.py:8-27): fwd + autograd bwd ---------------------------------
for tag, shape in (('bp_small', (2, 32, 4, 7)), ('bp_c128', (2, 128, 14, 14))):
    x = detgen.det_uniform(shape, 11).requires_grad_(True)
    y = BilinearPooling()(x)
    dy = detgen.det(y.shape, 12)
    (dx,) = torch.autograd.grad(y, x, dy)
    out[f'{tag}_y'] = y.detach().numpy()
    out[f'{tag}_dx'] = dx.numpy()

# full-size BCNN shape: keep only summaries + a slice (output is 1 MB/img)
x = detgen.det_uniform((1, 512, 14, 14), 13).requires_grad_(True)
y = BilinearPooling()(x)
dy = detgen.det(y.shape, 14)
(dx,) = torch.autograd.grad(y, x, dy)
out['bp_full_y_slice'] = y.detach().numpy()[0, ::997]
out['bp_full_y_sum'] = np.float64(y.detach().double().sum().item())
out['bp_full_dx'] = dx.numpy()

# ---- compact bilinear pooling (CBCNN.py:38-164) -------------------------------------------
for d in (8192, 6000):
    cbp = CompactBilinearPooling(512, 512, d)
    h = cbp.sparse_sketch_matrix1.abs().argmax(1).numpy()
    s = cbp.sparse_sketch_matrix1.sum(1).numpy()
    h2 = cbp.sparse_sketch_matrix2.abs().argmax(1).numpy()
    s2 = cbp.sparse_sketch_matrix2.sum(1).numpy()
    blob = np.concatenate([h, s, h2, s2]).astype(np.int64).tobytes()
    out[f'cbp_hash_sha256_{d}'] = np.frombuffer(hashlib.sha256(blob).digest(), dtype=np.uint8)
    out[f'cbp_h1_{d}'] = h.astype(np.int64)
    out[f'cbp_h2_{d}'] = h2.astype(np.int64)
    out[f'cbp_s1_{d}'] = s.astype(np.int64)
    out[f'cbp_s2_{d}'] = s2.astype(np.int64)
    x = detgen.det_uniform((2, 512, 3, 3), 21).requires_grad_(True)
    y = cbp(x)
    dy = detgen.det(y.shape, 22)
    (dx,) = torch.autograd.grad(y, x, dy)
    out[f'cbp_y_{d}'] = y.detach().numpy()
    out[f'cbp_dx_{d}'] = dx.numpy()
    # same op on TF32-representable inputs (what the op sees inside the model: the trunk rounds its activations to tf32):
    # the tensor-core Gram is then exact, so the ill-conditioned signed-sqrt gradient can be compared tightly
    x = detgen.tf32_rna(detgen.det_uniform((2, 512, 3, 4), 23)).requires_grad_(True)
    y = cbp(x)
    (dx,) = torch.autograd.grad(y, x, detgen.det(y.shape, 24))
    out[f'cbp_tf32in_y_{d}'] = y.detach().numpy()
    out[f'cbp_tf32in_dx_{d}'] = dx.numpy()

# ---- MPN-COV (MPNCOV.py:105-230) -------------------------------------------------------------
for tag, shape, it in (('mpn_small', (2, 16, 3, 3), 5), ('mpn_it3', (2, 24, 4, 4), 3), ('mpn_c256', (1, 256, 14, 14), 5)):
    x = detgen.det_uniform(shape, 31).requires_grad_(True)
    c = Covpool.apply(x)
    s = Sqrtm.apply(c, it)
    v = Triuvec.apply(s)
    dv = detgen.det(v.shape, 32)
    (dx,) = torch.autograd.grad(v, x, dv)
    out[f'{tag}_cov'] = c.detach().numpy()
    out[f'{tag}_sqrt'] = s.detach().numpy()
    if shape[1] <= 64:
        out[f'{tag}_vec'] = v.detach().numpy()
    out[f'{tag}_dx'] = dx.numpy()

# ---- full BCNN (BCNN.py:30-55) with deterministic weights, 64x64 input ----------------------------
for stage in (1, 2):
    net = MODEL.get('BCNN')(rh.cfg(name='BCNN', stage=stage, num_classes=200))
    from oracle.hop_oracle import VGG16_D
    state = detgen.vgg_bcnn_state(VGG16_D, 200, seed=100)
    net.load_state_dict(state)
    net.train()
    x = detgen.det((2, 3, 64, 64), 41)
    labels = detgen.det_labels(2, 200, 42)
    logits = net(x)
    loss = torch.nn.CrossEntropyLoss(label_smoothing=0.1)(logits, labels)
    net.zero_grad()
    loss.backward()
    out[f'bcnn_s{stage}_logits'] = logits.detach().numpy()
    out[f'bcnn_s{stage}_loss'] = np.float32(loss.item())
    out[f'bcnn_s{stage}_gW_slice'] = net.classifier.weight.grad.numpy()[:, ::4099]
    out[f'bcnn_s{stage}_gb'] = net.classifier.bias.grad.numpy()
    if stage == 2:
        for k, p in net.named_parameters():
            if k.startswith('backbone') and k.endswith('bias'):
                out[f'bcnn_s2_g_{k}'] = p.grad.numpy()
        out['bcnn_s2_g_backbone.0.weight'] = net.backbone[0].weight.grad.numpy()
        out['bcnn_s2_g_backbone.28.weight_slice'] = net.backbone[28].weight.grad.numpy()[::8, ::8]

# ---- full CBCNN (CBCNN.py:12-35), d=8192 --------------------------------------------------------
net = MODEL.get('CBCNN')(rh.cfg(name='CBCNN', stage=2, num_classes=200, input_channel=512, output_channel=8192))
state = detgen.vgg_bcnn_state(VGG16_D, 200, seed=100, head_in=8192)
net.load_state_dict(state)
x = detgen.det((2, 3, 128, 128), 41)   # 4x4 feature map
labels = detgen.det_labels(2, 200, 42)
logits = net(x)
loss = torch.nn.CrossEntropyLoss(label_smoothing=0.1)(logits, labels)
net.zero_grad()
loss.backward()
out['cbcnn_logits'] = logits.detach().numpy()
out['cbcnn_loss'] = np.float32(loss.item())
out['cbcnn_g_backbone.28.bias'] = net.backbone[28].bias.grad.numpy()
out['cbcnn_g_backbone.0.bias'] = net.backbone[0].bias.grad.numpy()

save_golden('reference_outputs', out)                 # parts of under 1 MB: tests/golden/reference_outputs.<i>.npz
print('wrote', len(out), 'arrays')
