"""S3N, selective sparse sampling (Ding et al., ICCV 2019), with the reference's surface (model/methods/S3N.py).

Same modules as the reference — ``backbone`` (a ResNet-50 with its unused 1000-way ``fc``) and ``features`` (its children
without avgpool and fc, the same modules again), ``radius`` / ``radius_inv`` (ScaleLayer), ``filter`` (the 61x61 Gaussian
conv), ``raw_classifier``, ``sampler_buffer`` / ``sampler_buffer1`` (3x3 stride-2 conv, BatchNorm, ReLU),
``sampler_classifier`` / ``sampler_classifier1``, ``con_classifier`` and ``map_origin`` (a 1x1 conv that never gets a
gradient) — so the reference's ``state_dict`` loads strictly, in both directions.  ``P_basis`` stays a plain attribute.
``forward(x, p)`` returns ``(aggregation, agg_origin, agg_sampler, agg_sampler1)``.

The trunk runs on ops_resnet three times per call — the images, the zoomed images, the complementary images — so
BatchNorm updates its running statistics three times per training step, in that order.  The class response maps are one
GEMM over the trunk's NHWC map with map_origin's weights, copied from raw_classifier at every forward as in the reference;
the sampler, the grid and the warp run on hk_s3n_* (ops_s3n).  ``radius``, ``radius_inv`` and ``filter`` get their gradients
through the warp's grid gradient, which needs the trunk's gradient at its input image (hk_stem_dgrad).

Deliberate deviations from the reference:

- Random draws: the reference draws ``random.uniform(0, 1)`` on the host, one per peak (p = 1).  Here the forward draws
  ``torch.rand(N, 961)`` on the device, one per grid position, and a peak uses the draw at its own position: the same
  distribution, no host round trip, and PyTorch's generator keeps the draws right under CUDA-graph capture.
- Maps with no peaks: the reference appends nothing to ``xs_inv`` for such an image, and its ``torch.cat`` fails (a
  constant decision map normalises to NaN and has no peaks either).  Here such an image gets ``base_ratio`` in both maps.
- The value of ``p``: ``p`` may be a Python int or an int32 device tensor of one element, which the sampler kernel reads.
  One captured graph then serves every epoch: the trainer writes the epoch's ``p`` into its tensor before each step.
"""
import numpy as np
import torch
import torch.nn as nn

from .. import ops, ops_resnet, ops_s3n
from ..backbone.resnet import RESNET_NAMES
from ..registry import MODEL
from .resnet import _build


def make_gaussian(size, fwhm=3):
    """makeGaussian(size, fwhm) of S3N.py:12-22, centred."""
    x = np.arange(0, size, 1, float)
    y = x[:, np.newaxis]
    x0 = y0 = size // 2
    return np.exp(-4 * np.log(2) * ((x - x0) ** 2 + (y - y0) ** 2) / fwhm ** 2)


class ScaleLayer(nn.Module):
    def __init__(self, init_value=1e-3):
        super().__init__()
        self.scale = nn.Parameter(torch.FloatTensor([init_value]))


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _buffer():
    return nn.Sequential(nn.Conv2d(2048, 2048, kernel_size=3, stride=2, padding=1, bias=False), nn.BatchNorm2d(2048),
                         nn.ReLU())


@MODEL.register
class S3N(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        num_classes = config.num_classes
        ops.check_num_classes(num_classes)
        if int(config.image_size) <= 0 or int(config.image_size) % 64:
            raise ValueError(f'S3N: image_size={config.image_size} must be a positive multiple of 64 (the sampler buffers\' '
                             'stride-2 conv takes an even layer4 map)')
        self.backbone = _build(_Cfg(num_classes=1000), (3, 4, 6, 3), 'HAWKEYE_RESNET50_PTH', 'resnet50')
        self.features = nn.Sequential(*[getattr(self.backbone, n) for n in RESNET_NAMES])
        self.num_features = 2048
        self.grid_size = ops_s3n.GRID
        self.padding_size = ops_s3n.PAD
        self.global_size = self.grid_size + 2 * self.padding_size
        self.input_size_net = config.image_size
        self.base_ratio = config.base_ratio
        self.radius = ScaleLayer(config.radius)
        self.radius_inv = ScaleLayer(config.radius_inv)
        self.filter = nn.Conv2d(1, 1, kernel_size=(2 * self.padding_size + 1, 2 * self.padding_size + 1), bias=False)
        with torch.no_grad():
            self.filter.weight[0].copy_(torch.FloatTensor(make_gaussian(2 * self.padding_size + 1, fwhm=13)))
        g = torch.arange(self.global_size, dtype=torch.float64)
        basis = (g - self.padding_size) / (self.grid_size - 1.0)
        self.P_basis = torch.stack([basis.expand(self.global_size, -1), basis[:, None].expand(-1, self.global_size)]).float()
        self.raw_classifier = nn.Linear(2048, num_classes)
        self.sampler_buffer = _buffer()
        self.sampler_classifier = nn.Linear(2048, num_classes)
        self.sampler_buffer1 = _buffer()
        self.sampler_classifier1 = nn.Linear(2048, num_classes)
        self.con_classifier = nn.Linear(self.num_features * 3, num_classes)
        self.avg = nn.AdaptiveAvgPool2d(1)
        self.max_pool = nn.AdaptiveMaxPool2d(1)
        self.map_origin = nn.Conv2d(2048, num_classes, 1, 1, 0)
        self.__dict__['_plan'] = self.backbone._plan
        self.__dict__['_units'] = (ops_resnet.Unit('3x3s2', self.sampler_buffer[0], self.sampler_buffer[1], True),
                                   ops_resnet.Unit('3x3s2', self.sampler_buffer1[0], self.sampler_buffer1[1], True))
        self.__dict__['_p'] = {}

    def no_grad_parameters(self):
        """The parameters no loss reaches: ``backbone.fc`` (never called) and ``map_origin`` (copied from raw_classifier
        at every forward and used without gradient)."""
        return list(self.backbone.fc.parameters()) + list(self.map_origin.parameters())

    def device_p(self, p, device):
        """p as the int32 device scalar the sampler reads: a tensor is used as it is; an int is written into a tensor the
        model keeps per device (outside a graph capture, or the capture would freeze its value)."""
        if isinstance(p, torch.Tensor):
            return p
        t = self._p.get(device)
        if t is None:
            t = self._p[device] = torch.zeros(1, dtype=torch.int32, device=device)
        t.fill_(int(p))
        return t

    def branch(self, x, unit):
        feat = ops_resnet.resnet_trunk(x, self._plan, self.training)
        if unit is not None:
            feat = ops_resnet.unit(feat, unit, self.training)
        return ops.NHWCMeanFn.apply(feat), feat

    def forward(self, x, p):
        with torch.no_grad():                                        # S3N.py:288-289
            self.map_origin.weight.copy_(self.raw_classifier.weight[:, :, None, None])
            self.map_origin.bias.copy_(self.raw_classifier.bias)
        N = x.shape[0]
        pooled_raw, feature_raw = self.branch(x, None)
        agg_origin = ops.linear(pooled_raw, self.raw_classifier.weight, self.raw_classifier.bias)
        with torch.no_grad():
            _, h, w, C = feature_raw.shape
            K = self.map_origin.out_channels
            crm = ops.gemm_tf32(feature_raw.reshape(-1, C), self.map_origin.weight.reshape(K, C),
                                D=self.map_origin.bias.reshape(1, K), beta=1.0).view(N, h, w, K)
        rnd = torch.rand(N, self.grid_size * self.grid_size, device=x.device)
        x_zoom, x_inv = ops_s3n.sample_images(x, crm, rnd, self.device_p(p, x.device), self.radius.scale,
                                              self.radius_inv.scale, self.filter.weight, self.base_ratio)
        pooled_d, _ = self.branch(x_zoom, self._units[0])
        agg_sampler = ops.linear(pooled_d, self.sampler_classifier.weight, self.sampler_classifier.bias)
        pooled_c, _ = self.branch(x_inv, self._units[1])
        agg_sampler1 = ops.linear(pooled_c, self.sampler_classifier1.weight, self.sampler_classifier1.bias)
        aggregation = ops.linear(torch.cat([pooled_raw, pooled_d, pooled_c], 1), self.con_classifier.weight,
                                 self.con_classifier.bias)
        return aggregation, agg_origin, agg_sampler, agg_sampler1

    def prediction(self, outputs):
        return outputs[0]
