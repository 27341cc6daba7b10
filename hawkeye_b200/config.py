"""Entry point mirror of the reference's config.py:5-31: ONE yaml via ``--config`` -> frozen CfgNode."""
import argparse

try:
    from yacs.config import CfgNode as CN
except Exception:  # yacs is not installed in this image
    from .cfgnode import CfgNode as CN


def load_config(path):
    with open(path) as f:
        cfg = CN.load_cfg(f)
    cfg.freeze()
    return cfg


def setup_config(argv=None):
    parser = argparse.ArgumentParser(description='Hawkeye (H100-native hot path)')
    parser.add_argument('--config', default='configs/Baseline.yaml', type=str, help='path to config file')
    arg, _ = parser.parse_known_args(argv)
    return load_config(arg.config)
