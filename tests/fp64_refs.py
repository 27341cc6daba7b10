"""fp64 restatements that more than one kernel suite compares with, and the measured constants of their bounds.

The 3x3 convolution references (test_gpu_conv_vgg16.py, test_gpu_conv_first.py, test_gpu_conv_bwd_fused.py): the inputs
are TF32-representable (detgen.tf32_rna), so every tensor-core product is exact and a kernel's output may differ from
the fp64 result only by its fp32 accumulation and, where it stores TF32, one rounding on store.  Each reference comes
with its fp32 scale, the same operation applied to |inputs| and |weights|; the c constants below bound the
accumulation relative to it (test_gpu_conv_vgg16.py gives the measurements).

The classifier (hk_linear_*) references: test_gpu_mpncov_head.py measures C_LIN, test_gpu_osme_head.py uses it.
"""
import contextlib

import torch
import torch.nn.functional as F

import detgen
from kernel_check import U, nchw, nhwc

BATCH = 32
# (name, H = W, Cin, Cout, max-pool follows) of the VGG-16 3x3 convolutions behind conv1_1 at 448x448
VGG16_LAYERS = [('conv1_2', 448, 64, 64, True),
                ('conv2_1', 224, 64, 128, False), ('conv2_2', 224, 128, 128, True),
                ('conv3_1', 112, 128, 256, False), ('conv3_2', 112, 256, 256, False), ('conv3_3', 112, 256, 256, True),
                ('conv4_1', 56, 256, 512, False), ('conv4_2', 56, 512, 512, False), ('conv4_3', 56, 512, 512, True),
                ('conv5_1', 28, 512, 512, False), ('conv5_2', 28, 512, 512, False), ('conv5_3', 28, 512, 512, True)]

C_TF32 = 2.0 ** -17           # forward and data gradient (9 Cin terms per output), single-pass TF32
C_TF32_WGRAD = 2.0 ** -15     # weight and bias gradients (a sum over every pixel of the batch), single-pass TF32
CHUNK = 4                     # images per fp64 reference evaluation
C_LIN = 2.0 ** -19            # classifier forward, data and weight gradient products


def gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def randn(shape, g, scale=1.0):
    return torch.randn(shape, device='cuda', generator=g) * scale


# ------------------------------------------------------------------------------------------------ 3x3 convolution
@contextlib.contextmanager
def fp32_exact():
    """fp32 convolutions without TF32 (the scale references)"""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def pack(w):
    """hk_conv3x3_pack_weights: the forward and data-gradient weight layouts of w [Cout, Cin, 3, 3]"""
    from hawkeye_b200 import _lib
    cout, cin = w.shape[:2]
    wf = torch.empty(9 * cout * cin, device='cuda')
    wd = torch.empty(9 * cout * cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, _lib.stream_ptr())
    return wf, wd


def conv_ref(x, w, b):
    """fp64 pre-activation conv2d and its fp32 scale conv2d(|x|, |w|) + |b|, NHWC, of an NHWC chunk"""
    xc = nchw(x)
    ref = nhwc(F.conv2d(xc.double(), w.double(), None if b is None else b.double(), padding=1))
    with fp32_exact():
        absref = nhwc(F.conv2d(xc.abs(), w.abs(), None if b is None else b.abs(), padding=1))
    return ref, absref


def dgrad_ref(dy, w):
    """fp64 input gradient of conv2d(., w, padding=1) (conv_transpose2d) and its fp32 scale, NHWC"""
    dc = nchw(dy)
    ref = nhwc(F.conv_transpose2d(dc.double(), w.double(), padding=1))
    with fp32_exact():
        absref = nhwc(F.conv_transpose2d(dc.abs(), w.abs(), padding=1))
    return ref, absref


def wgrad_ref(x, dy, cin, cout, chunk=CHUNK):
    """fp64 weight and bias gradients of conv2d(x, ., padding=1) against dy, summed chunk by chunk, and their fp32
    scales computed from |x|, |dy|"""
    gw = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda')
    aw = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda')
    gb = torch.zeros(cout, dtype=torch.float64, device='cuda')
    ab = torch.zeros(cout, dtype=torch.float64, device='cuda')
    for n0 in range(0, x.shape[0], chunk):
        xc, dc = nchw(x[n0:n0 + chunk]), nchw(dy[n0:n0 + chunk])
        gw += torch.nn.grad.conv2d_weight(xc.double(), gw.shape, dc.double(), padding=1)
        gb += dc.double().sum((0, 2, 3))
        with fp32_exact():
            aw += torch.nn.grad.conv2d_weight(xc.abs(), gw.shape, dc.abs(), padding=1).double()
        ab += dc.abs().double().sum((0, 2, 3))
        del xc, dc
    return gw, aw, gb, ab


# ------------------------------------------------------------------------------------------------ classifier
def linear_splits(F):
    """hk_linear_fwd's K slices (head.cu)"""
    S = min(max(F // 1024, 1), 512)
    while F % S or (F // S) % 4:
        S -= 1
        if S <= 1:
            return 1
    return S


def classifier_inputs(B, F, N, seed, device):
    """tf32 x, w, dy and an fp32 bias; the last 4 columns of every K slice of x and w (a partial k-block: 1028 = 32 x 32
    + 4) are 16x larger, so that leaving them out cannot hide"""
    g = torch.Generator(device=device).manual_seed(seed)
    S = linear_splits(F)
    x = torch.relu(torch.randn(B, F, generator=g, device=device))
    w = torch.randn(N, F, generator=g, device=device) * F ** -0.5
    tail = torch.zeros(F, dtype=torch.bool, device=device)
    for s in range(S):
        tail[(s + 1) * (F // S) - 4:(s + 1) * (F // S)] = True
    x[:, tail] *= 16
    w[:, tail] *= 16
    b = torch.randn(N, generator=g, device=device) * 0.1
    dy = torch.randn(B, N, generator=g, device=device) * 0.01
    return detgen.tf32_rna(x), detgen.tf32_rna(w), b, detgen.tf32_rna(dy), S


def linear_refs(x, w, b, dy, S):
    """fp64 y, dx, dw, db and their (fixed, scale) bounds"""
    xd, wd, bd, dd = (t.to(torch.float64) for t in (x, w, b, dy))
    sy = xd.abs() @ wd.abs().T + bd.abs()
    out = {'y': (xd @ wd.T + bd, (S + 1) * U * sy, sy),
           'dx': (dd @ wd, 0 * xd, dd.abs() @ wd.abs()),
           'dw': (dd.T @ xd, 0 * wd, dd.abs().T @ xd.abs())}
    out['db'] = (dd.sum(0), 2.0 ** -19 * dd.abs().sum(0), dd.abs().sum(0))
    return out
