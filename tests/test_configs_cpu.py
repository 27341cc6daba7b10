"""The shipped yamls load through hawkeye_b200.config (yacs-compatible CfgNode) and build their models through the registry
with the parameter counts of the reference models."""
import os

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('name,total,trainable', [('BCNN_S1', 67143688, 52429000), ('BCNN_S2', 67143688, 67143688),
                                                   ('CBCNN_S1', 14714688 + 8192 * 200 + 200, None), ('MPN', 30612232, 30612232)])
def test_yaml_builds_model(name, total, trainable):
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', name + '.yaml'))
    assert 'model' in cfg and cfg['model'] is cfg.model and cfg.train.optimizer.lr > 0      # attribute and item access
    net = hb.MODEL.get(cfg.model.name)(cfg.model)
    assert sum(p.numel() for p in net.parameters()) == total
    if trainable is not None:
        assert sum(p.numel() for p in net.parameters() if p.requires_grad) == trainable
    for attr in ('backbone', 'classifier'):
        assert hasattr(net, attr)
