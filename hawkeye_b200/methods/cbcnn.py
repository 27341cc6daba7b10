"""CBCNN with the reference's surface (model/methods/CBCNN.py:12-164)."""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..backbone.vgg import vgg16
from ..registry import MODEL
from ..utils import initialize_weights


class CompactBilinearPooling(nn.Module):
    """Tensor-Sketch pooling (CBCNN.py:38-135).  Same constructor; hash/sign vectors are the bit-exact numpy streams of
    CBCNN.py:76-91.  Like the reference's sketch matrices they are plain attributes (not in the state_dict)."""

    def __init__(self, input_dim1, input_dim2, output_dim, sum_pool=True, rand_h_1=None, rand_s_1=None, rand_h_2=None,
                 rand_s_2=None):
        super().__init__()
        if input_dim1 != input_dim2 or not sum_pool:
            raise NotImplementedError('hawkeye_b200: compact bilinear pooling of one feature map with sum_pool=True')
        self.input_dim1, self.input_dim2, self.output_dim, self.sum_pool = input_dim1, input_dim2, output_dim, sum_pool
        h1, s1, h2, s2 = ops.count_sketch_hashes(input_dim1, output_dim)
        h1 = np.asarray(rand_h_1) if rand_h_1 is not None else h1
        s1 = np.asarray(rand_s_1) if rand_s_1 is not None else s1
        h2 = np.asarray(rand_h_2) if rand_h_2 is not None else h2
        s2 = np.asarray(rand_s_2) if rand_s_2 is not None else s2
        assert np.all(h1 >= 0) and np.all(h1 < output_dim) and np.all(h2 >= 0) and np.all(h2 < output_dim)
        self.rand_h_1, self.rand_s_1, self.rand_h_2, self.rand_s_2 = h1, s1, h2, s2
        self._dev = {}

    def _tables(self, device):
        if device not in self._dev:
            self._dev[device] = (torch.from_numpy(self.rand_h_1.astype(np.int32)).to(device),
                                 torch.from_numpy(self.rand_h_2.astype(np.int32)).to(device),
                                 torch.from_numpy(self.rand_s_1.astype(np.float32)).to(device),
                                 torch.from_numpy(self.rand_s_2.astype(np.float32)).to(device))
        return self._dev[device]

    def forward(self, bottom1, bottom2=None):
        if bottom2 is not None and bottom2 is not bottom1:
            raise NotImplementedError('hawkeye_b200: two distinct bottoms are not on the CBCNN path (CBCNN.py:33)')
        assert bottom1.size(1) == self.input_dim1
        h1, h2, s1, s2 = self._tables(bottom1.device)
        return ops.CompactBilinearPoolFn.apply(bottom1, h1, h2, s1, s2, self.output_dim)


@MODEL.register
class CBCNN(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        in_channel, out_channel = config.input_channel, config.output_channel   # CBCNN.py:18-19
        self.backbone = vgg16(pretrained=True)
        self.bilinear_pooling = CompactBilinearPooling(in_channel, in_channel, out_channel)
        ops.check_num_classes(config.num_classes)
        self.classifier = nn.Linear(out_channel, config.num_classes)
        self.classifier.apply(initialize_weights)

    def features(self, x):
        x = self.backbone(x)
        return x.detach() if self.config.stage == 1 else x                      # CBCNN.py:31-32

    def head(self, feat):
        return ops.linear(self.bilinear_pooling(feat), self.classifier.weight, self.classifier.bias)

    def forward(self, x):
        return self.head(self.features(x))
