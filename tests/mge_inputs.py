"""Seeded inputs shared by tests/golden/make_golden_mge.py and the MGE-CNN tests, so fixtures need not carry them."""
import numpy as np

E2E_IMAGE, E2E_BATCH, E2E_CLASSES = 128, 4, 12
E2E_LAYERS = (1, 1, 1, 3)          # the shallowest trunk the reference builds: GradCam hooks layer4 block "2"
BOX_THRED = 0.2                    # configs/MGE_CNN.yaml
E2E_THRED = 0.6                    # the end-to-end step's box_thred: high enough that its random trunks' boxes are not the whole image
CAM_C = 256                        # channels of the get_bbox maps (any count works; the CAM is summed over them)

# get_bbox cases: name -> (image size, images, kind, seed, rate).  'rand' maps are seeded ReLU'd normals with positive
# random weights; 'int' maps hold integers 0..7 with power-of-two weights, so the CAM is exact in any summation order;
# 'const' gives a constant CAM (0 / 0 = NaN everywhere); 'peak' one pixel; 'row' / 'col' keep a single row / column.
BBOX_CASES = {
    'rand224': (224, 5, 'rand', 5100, BOX_THRED),
    'rand224_r5': (224, 3, 'rand', 5101, 0.5),
    'rand448': (448, 3, 'rand', 5102, 0.4),
    'int224': (224, 6, 'int', 5103, BOX_THRED),
    'int224_r6': (224, 4, 'int', 5104, 0.6),
    'int448': (448, 4, 'int', 5105, 0.5),
    'const224': (224, 2, 'const', 5106, BOX_THRED),
    'peak224': (224, 1, 'peak', 5107, BOX_THRED),
    'peak448': (448, 1, 'peak', 5108, BOX_THRED),
    'row224': (224, 2, 'row', 5109, 0.99),
    'col448': (448, 2, 'col', 5110, 0.99),
}
EXACT_CASES = tuple(k for k, v in BBOX_CASES.items() if v[2] != 'rand')


def bbox_case(name):
    """-> (conv5 float32 [N, C, h, h] NCHW, layer weights float32 [N, C] >= 0, rate, image size)."""
    size, n, kind, seed, rate = BBOX_CASES[name]
    h = size // 32
    C = CAM_C
    rs = np.random.RandomState(seed)
    if kind in ('rand', 'int'):
        # sparse maps (about one pixel in six active per channel), so that the boxes are not the whole image
        active = rs.random_sample((n, C, h, h)) < 0.15
        if kind == 'rand':
            x = (np.abs(rs.standard_normal((n, C, h, h))) * active).astype(np.float32)
            lw = (np.maximum(rs.standard_normal((n, C)), 0) / (h * h)).astype(np.float32)
        else:
            x = (rs.randint(1, 8, size=(n, C, h, h)) * active).astype(np.float32)
            lw = np.ldexp(1.0, -rs.randint(0, 7, size=(n, C))).astype(np.float32)
        lw[rs.random_sample((n, C)) < 0.97] = 0          # a few channels carry the CAM
    else:
        x = np.zeros((n, C, h, h), dtype=np.float32)
        lw = np.zeros((n, C), dtype=np.float32)
        lw[:, :4] = 0.25
        if kind == 'const':
            x[:, :4] = 1.0
        elif kind == 'peak':
            x[:, :4, 3, 3] = 1.0
        elif kind == 'row':
            x[:, :4, 0, :] = 1.0
            x[1, :4, h - 1, :] = 1.0
        elif kind == 'col':
            x[:, :4, :, 2] = 1.0
    return x, lw, rate, size


def crop_box(xy, size):
    """The reference's [x1, x2, y1, y2] of get_bbox -> the (y0, x0, y1, x1) box its crop reads (the whole image when
    x1 == x2 or y1 == y2)."""
    x1, x2, y1, y2 = (int(v) for v in xy)
    if x1 == x2 or y1 == y2:
        return (0, 0, size, size)
    return (y1, x1, y2, x2)


def gradcam_input(seed=5200):
    """A conv4-shaped input [2, 1024, 8, 8] for the reference GradCam on the shallow model (8x8: a 256 image's layer3)."""
    rs = np.random.RandomState(seed)
    return np.maximum(rs.standard_normal((2, 1024, 8, 8)), 0).astype(np.float32)
