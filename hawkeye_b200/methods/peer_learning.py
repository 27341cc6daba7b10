"""PeerLearningNet with the reference's surface (model/methods/PeerLearningNet.py:8-20): two copies of a base model built
through the registry (``config.base_model.name`` — BCNN in configs/PeerLearning_BCNN_S{1,2}.yaml), the second with a freshly
initialised classifier; ``forward`` returns both logit tensors.  The base model is whatever ``MODEL`` holds under that name,
i.e. the native BCNN / CBCNN / MPN, so this caller of the hot path inherits the kernels unchanged."""
import copy

import torch.nn as nn

from ..registry import MODEL
from ..utils import initialize_weights


@MODEL.register
class PeerLearningNet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.base_model = MODEL.get(config.base_model.name)(config.base_model)     # PeerLearningNet.py:13
        self.base_model2 = copy.deepcopy(self.base_model)                           # :14
        self.base_model2.classifier.apply(initialize_weights)                       # :15

        self._shared_key = None

    def _backbones_identical(self):
        """Stage 1 of the BCNN / CBCNN base models freezes the backbone and detaches its output: the second network's
        backbone is a deep copy that never changes, so ONE backbone pass serves both heads.  Verified, not assumed: the
        two parameter sets are compared once per (version) state and re-checked whenever either changes."""
        m1, m2 = self.base_model, self.base_model2
        if not (hasattr(m1, 'features') and hasattr(m1, 'head') and getattr(m1, 'stage', getattr(getattr(m1, 'config', None), 'stage', 2)) == 1):
            return False
        p1, p2 = list(m1.backbone.parameters()), list(m2.backbone.parameters())
        if any(p.requires_grad for p in p1 + p2) or len(p1) != len(p2):
            return False
        key = tuple((p.data_ptr(), p._version) for p in p1 + p2)
        if key != self._shared_key:
            import torch
            self._shared_ok = all(a.shape == b.shape and torch.equal(a, b) for a, b in zip(p1, p2))
            self._shared_key = key
        return self._shared_ok

    def forward(self, x):
        if self._backbones_identical():
            feat = self.base_model.features(x)
            return self.base_model.head(feat), self.base_model2.head(feat)
        return self.base_model(x), self.base_model2(x)                              # :17-20

    def prediction(self, outputs):
        return tuple(outputs)
