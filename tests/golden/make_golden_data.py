"""Golden fixtures of the host-side surfaces, recorded from the UNMODIFIED reference:
  reference_checkpoint_layout.json — key order, shapes and dtypes of the state_dict the reference's BCNN / MPN write
                                     (read by tests/test_checkpoint_cpu.py);
  reference_data.npz               — the reference's dataset / transforms / sampler outputs on the generated image folder
                                     of tests/test_data_cpu.py (tests/test_data_cpu.py::reference_data_outputs).
Needs the reference tree ($HAWKEYE_REF or baseline/_ref):  python tests/golden/make_golden_data.py"""
import importlib
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
from oracle import ref_harness as rh  # noqa: E402
import test_data_cpu  # noqa: E402

rh.load_reference()
from model.registry import MODEL as REF  # noqa: E402

layout = {}
for (name, kw) in [('BCNN', dict(stage=2, num_classes=200)),
                   ('MPN', dict(iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048, dimension_reduction=256,
                                num_classes=200))]:
    torch.manual_seed(1)
    m = REF.get(name)(rh.cfg(name=name, **kw))
    layout[name] = [[k, list(v.shape), str(v.dtype).replace('torch.', '')] for k, v in m.state_dict().items()]
json.dump(layout, open(os.path.join(HERE, 'reference_checkpoint_layout.json'), 'w'), indent=0)

root = rh.find_reference_root()
if root not in sys.path:
    sys.path.insert(0, root)
rd, rt, rs = (importlib.import_module(m) for m in ('dataset.dataset', 'dataset.transforms', 'dataset.sampler'))


class _TmpFactory:
    def mktemp(self, name):
        return tempfile.mkdtemp(prefix=name)


folder, meta = test_data_cpu.folder.__wrapped__(_TmpFactory())
np.savez_compressed(test_data_cpu.REFERENCE_DATA, **test_data_cpu.reference_data_outputs(folder, meta, rd, rt, rs))
print('wrote reference_checkpoint_layout.json and reference_data.npz')
