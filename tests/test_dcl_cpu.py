"""DCL on CPU: the registry model against the reference's state_dict layout and parameter count, DCLTrainer's parameter
groups and StepLR schedule, the jigsaw data path (RandomSwap, DCLDataset, the collate functions) bit for bit, and the fp64
oracle, all against fixtures of the unmodified reference (tests/golden/make_golden_dcl.py)."""
import json
import os
import random

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2
from oracle import dcl_oracle as D

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = load_golden('reference_dcl')


class Cfg(dict):
    __getattr__ = dict.__getitem__


def _net(monkeypatch, **kw):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'DCL.yaml'))
    mc = cfg.model if not kw else Cfg(dict(name='DCL', num_classes=200, cls_2=False, cls_2xmul=False), **kw)
    return hb.MODEL.get('DCL')(mc), cfg


def test_yaml_builds_dcl_with_reference_layout(monkeypatch):
    net, cfg = _net(monkeypatch)
    ref = json.loads(bytes(G['state_keys_json']).decode())
    assert len(ref) == 322
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == ref
    assert sum(p.numel() for p in net.parameters()) == int(G['params_cls2'])
    for attr in ('backbone', 'Convmask', 'avgpool2', 'avgpool', 'classifier', 'classifier_swap'):
        assert hasattr(net, attr)
    sd = {k: torch.full(s, 0.25) if not k.endswith('num_batches_tracked') else torch.tensor(3) for k, s in ref.items()}
    net.load_state_dict(sd, strict=True)                                    # a reference checkpoint loads as is
    assert torch.equal(net.classifier_swap.weight, torch.full((2, 2048), 0.25))
    mul, _ = _net(monkeypatch, cls_2xmul=True)
    assert sum(p.numel() for p in mul.parameters()) == int(G['params_cls2xmul'])
    both, _ = _net(monkeypatch, cls_2=True, cls_2xmul=True)                # cls_2xmul wins, as in DCL.py:25-28
    assert both.classifier_swap.weight.shape == (400, 2048)


def test_dcl_needs_a_swap_classifier(monkeypatch):
    import hawkeye_b200 as hb
    with pytest.raises(hb._lib.HawkeyeLibError, match='cls_2'):
        _net(monkeypatch, cls_2=False)
    with pytest.raises(hb._lib.HawkeyeLibError):
        _net(monkeypatch, cls_2=True, num_classes=202)


def test_dcl_trainer_groups_lrs_and_no_weight_decay(monkeypatch):
    from hawkeye_b200 import engine, examples
    net, cfg = _net(monkeypatch)
    t = object.__new__(examples.DCLTrainer)
    t.model, t.config = net, cfg
    groups = t.param_groups()
    opt_cfg = cfg.train.optimizer
    assert [m for _, m in groups] == [1.0, opt_cfg.lr_ratio, opt_cfg.lr_ratio, opt_cfg.lr_ratio]
    assert groups[1][0] == [net.classifier.weight] and groups[2][0] == [net.classifier_swap.weight]
    assert groups[3][0] == [net.Convmask.weight, net.Convmask.bias]
    assert sum(p.numel() for g, _ in groups for p in g) == sum(p.numel() for p in net.parameters())

    class FakeFlat:
        flat = torch.zeros(4)
    FakeFlat.groups = [g for g, _ in groups]
    t.flat = FakeFlat()
    opt = t.get_optimizer(opt_cfg)
    assert isinstance(opt, engine.FusedSGD) and opt_cfg.weight_decay > 0
    assert [g['lr'] for g in opt.param_groups] == pytest.approx([8e-4, 8e-3, 8e-3, 8e-3])
    assert all(g['weight_decay'] == 0.0 and g['momentum'] == 0.9 for g in opt.param_groups)
    assert examples.ALL_TRAINERS['DCL'] is examples.DCLTrainer and 'DCL' not in examples.TRAINERS
    assert type(t.get_criterion(cfg.train.criterion)).__name__ == 'DCLLoss'
    data = (torch.zeros(4, 3, 8, 8), torch.zeros(4).long(), torch.ones(4).long(), torch.zeros(4, 49), ['a', 'b'])
    images, targets = t.batch_tensors(data)
    assert images is data[0] and targets == data[1:4]


def test_step_scheduler_matches_torch_steplr():
    from hawkeye_b200.train import _Step
    p = [torch.nn.Parameter(torch.zeros(1)) for _ in range(2)]
    opt = torch.optim.SGD([dict(params=[p[0]], lr=8e-4), dict(params=[p[1]], lr=8e-3)], momentum=0.9)
    sch = torch.optim.lr_scheduler.StepLR(opt, step_size=60, gamma=0.1)

    class FakeOpt:
        param_groups = [dict(lr=8e-4, initial_lr=8e-4), dict(lr=8e-3, initial_lr=8e-3)]
    ours = _Step(FakeOpt(), 60, 0.1)
    for epoch in range(185):
        assert np.allclose([g['lr'] for g in FakeOpt.param_groups], [g['lr'] for g in opt.param_groups], rtol=1e-12), epoch
        opt.step()
        sch.step()
        ours.step()
        if epoch == 100:
            sd = ours.state_dict()
            ours = _Step(FakeOpt(), 60, 0.1)
            ours.load_state_dict(sd)


@pytest.mark.parametrize('tag', ['sq', 'rect'])
def test_random_swap_matches_reference(tag):
    from PIL import Image
    from hawkeye_b200.data import RandomSwap
    random.seed(int(G[f'swap_{tag}_seed']))
    out = RandomSwap(tuple(int(v) for v in G[f'swap_{tag}_size']))(Image.fromarray(G[f'swap_{tag}_in']))
    assert np.array_equal(np.asarray(out), G[f'swap_{tag}_out'])


def _dataset_dir(tmp_path):
    from PIL import Image
    lines = []
    seed = int(G['data_seed'])
    for i in range(22):
        label = 0 if i < 10 else 1
        name = f'c{label}/img{i:02d}.png'
        (tmp_path / f'c{label}').mkdir(exist_ok=True)
        w, h, s = 70 + i, 60 + (i % 5), seed + i
        rs = np.random.RandomState(s)
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 127 // max(w + h - 2, 1)], -1)
        Image.fromarray(np.clip(base + rs.randint(-30, 31, size=(h, w, 3)), 0, 255).astype(np.uint8)).save(tmp_path / name)
        lines.append(f'{label} {name}')
    (tmp_path / 'meta.txt').write_text('\n'.join(lines) + '\n')
    return str(tmp_path), str(tmp_path / 'meta.txt')


def _u8(t):
    return (t * 255).round().clamp(0, 255).to(torch.uint8).numpy()


def test_dcl_dataset_and_collate_match_reference(tmp_path):
    from torchvision.transforms import transforms
    from hawkeye_b200.data import DCLDataset, RandomSwap, collate_fn4train, collate_fn4val
    root, meta = _dataset_dir(tmp_path)
    seed = int(G['data_seed'])
    tf = {'swap': transforms.Compose([RandomSwap((7, 7))]), 'common_aug': transforms.Compose([transforms.Resize((56, 56))]),
          'train_totensor': transforms.Compose([transforms.Resize((56, 56)), transforms.ToTensor()]),
          'val_totensor': transforms.Compose([transforms.Resize((56, 56)), transforms.ToTensor()]), 'None': None}
    for tag, cls_2, cls_2xmul in (('cls2', True, False), ('cls2xmul', False, True)):
        random.seed(seed)
        ds = DCLDataset(root, meta, transforms=tf, mode='train', cls_2=cls_2, cls_2xmul=cls_2xmul)
        items = [ds[i] for i in (0, 13, 21)]
        for j, it in enumerate(items):
            assert np.array_equal(_u8(it[0]), G[f'ds_{tag}_{j}_img']) and np.array_equal(_u8(it[1]), G[f'ds_{tag}_{j}_swap'])
            assert it[2] == G[f'ds_{tag}_{j}_label'] and it[3] == G[f'ds_{tag}_{j}_label_swap']
            assert np.array_equal(np.array(it[4]), G[f'ds_{tag}_{j}_law1'])
            assert np.array_equal(np.array(it[5]), G[f'ds_{tag}_{j}_law2'])
        imgs, lab, lab_swap, law, names = collate_fn4train(items)
        assert np.array_equal(_u8(imgs), G[f'col_{tag}_imgs']) and np.array_equal(lab.numpy(), G[f'col_{tag}_labels'])
        assert np.array_equal(lab_swap.numpy(), G[f'col_{tag}_labels_swap'])
        assert lab.dtype == lab_swap.dtype == torch.int64 and law.dtype == torch.float32
        assert np.array_equal(law.numpy(), G[f'col_{tag}_law'])
        assert names == json.loads(bytes(G[f'col_{tag}_names']).decode())
    assert G['col_cls2_labels_swap'].tolist() == [1, 0] * 3
    random.seed(seed + 1)
    val = DCLDataset(root, meta, transforms=tf, mode='val')
    assert val.paths == json.loads(bytes(G['val_paths']).decode()) and len(val) == 2
    assert np.array_equal(np.array(val.labels), G['val_labels'])
    imgs, lab, lab_swap, law, _ = collate_fn4val([val[i] for i in range(len(val))])
    assert np.array_equal(_u8(imgs), G['val_imgs']) and np.array_equal(lab.numpy(), G['val_col_labels'])
    assert np.array_equal(lab_swap.numpy(), G['val_col_labels_swap']) and np.array_equal(law.numpy(), G['val_col_law'])


@pytest.mark.parametrize('S,seed', [(14, 501), (7, 511)])
def test_oracle_head_matches_reference(S, seed):
    import detgen
    import torch.nn as nn
    st = {k: torch.as_tensor(v) for k, v in detgen.state_like(nn.ModuleDict(dict(
        Convmask=nn.Conv2d(2048, 1, 1), classifier=nn.Linear(2048, 200, bias=False),
        classifier_swap=nn.Linear(2048, 2, bias=False)))).items()}
    x = detgen.det((4, 2048, S, S), seed, positive=True).double().requires_grad_(True)
    w = st['Convmask.weight'].double().requires_grad_(True)
    b = st['Convmask.bias'].double().requires_grad_(True)
    wc = st['classifier.weight'].double().requires_grad_(True)
    ws = st['classifier_swap.weight'].double().requires_grad_(True)
    pooled, mask = D.head(x, w, b)
    logits, swap = D.classifiers(pooled, wc, ws)
    assert mask.shape == (4, (S // 2) ** 2)
    for got, key in ((logits, 'logits'), (swap, 'swap'), (mask, 'mask')):
        assert rel_l2(got.detach(), G[f'head{S}_{key}']) < 1e-5, key
    r = [detgen.det(t.shape, seed + 1 + i).double() for i, t in enumerate((logits, swap, mask))]
    ((logits * r[0]).sum() + (swap * r[1]).sum() + (mask * r[2]).sum()).backward()
    assert rel_l2(x.grad[:, ::16], G[f'head{S}_dx']) < 1e-5
    assert rel_l2(w.grad, G[f'head{S}_dconvmask_w']) < 1e-5 and rel_l2(b.grad, G[f'head{S}_dconvmask_b']) < 1e-5
    assert rel_l2(wc.grad[:, ::8], G[f'head{S}_dclassifier']) < 1e-5
    assert rel_l2(ws.grad, G[f'head{S}_dclassifier_swap']) < 1e-5


@pytest.mark.parametrize('tag', ['cls2', 'cls2xmul'])
def test_oracle_loss_matches_reference(tag):
    alpha, beta, gamma = G['loss_weights'].tolist()
    t = {k: torch.as_tensor(G[f'loss_{tag}_{k}']).double().requires_grad_(True) for k in ('logits', 'swap', 'mask')}
    loss = D.loss(t['logits'], t['swap'], t['mask'], G[f'loss_{tag}_labels'], G[f'loss_{tag}_labels_swap'],
                  G[f'loss_{tag}_law'], alpha, beta, gamma)
    loss.backward()
    assert abs(loss.item() - float(G[f'loss_{tag}_value'])) < 1e-5 * abs(float(G[f'loss_{tag}_value']))
    for k in ('logits', 'swap', 'mask'):
        assert rel_l2(t[k].grad, G[f'loss_{tag}_d{k}']) < 1e-5, k
    assert (t['mask'].grad[0, :5] == 0).all()


def test_oracle_end_to_end_matches_reference(monkeypatch):
    """ResNet-50 trunk restatement + the DCL oracle on the reference's own end-to-end run (train mode, 128x128)."""
    import detgen
    from oracle import hop_oracle as O
    torch.set_num_threads(8)
    net, _ = _net(monkeypatch)
    st = detgen.state_like(net)                   # same keys/shapes as the reference model => same deterministic values
    x = detgen.det((4, 3, 128, 128), 560)
    feat = O.resnet50_trunk_fwd(x, st)
    assert rel_l2(feat[:, ::16], G['e2e_feat_slice']) < 1e-4
    pooled, mask = D.head(feat, st['Convmask.weight'], st['Convmask.bias'])
    logits, swap = D.classifiers(pooled, st['classifier.weight'], st['classifier_swap.weight'])
    assert rel_l2(logits, G['e2e_logits']) < 1e-3 and rel_l2(swap, G['e2e_swap']) < 1e-3
    assert rel_l2(mask, G['e2e_mask']) < 1e-3
    loss = D.loss(logits, swap, mask, G['e2e_labels'], G['e2e_labels_swap'], G['e2e_law'])
    assert abs(loss.item() - float(G['e2e_loss'])) < 1e-4


def test_stacked_logits_reads_only_whole_column_views():
    """The loss reads DCL's classifier output in place only when both logit tensors are its full-height column views; a
    row slice (the source images only, the first half of the batch) is concatenated, so every row of what the loss kernel
    reads belongs to the labels and laws it is given."""
    from hawkeye_b200.losses import dcl_stacked_logits
    base = torch.arange(8 * 204, dtype=torch.float32).reshape(8, 204).clone()     # a root tensor, as the GEMM output is
    logits, swap = base[:, :200], base[:, 200:202]
    assert dcl_stacked_logits(logits, swap) is base
    for rows in (slice(None, None, 2), slice(0, 4), slice(4, 8)):
        got = dcl_stacked_logits(logits[rows], swap[rows])
        assert got is not base and got.shape == (len(range(8)[rows]), 202)
        assert torch.equal(got, torch.cat([base[rows, :200], base[rows, 200:202]], 1))
    assert dcl_stacked_logits(base[:, :200].clone(), swap).shape == (8, 202)


def test_loss_rejects_inputs_whose_rows_or_width_differ():
    from hawkeye_b200 import _lib
    from hawkeye_b200.losses import DCLLoss
    crit = DCLLoss(Cfg(alpha=1.0, beta=1.0, gamma=1.0))
    z, s, m = torch.zeros(8, 200), torch.zeros(8, 2), torch.zeros(8, 49)
    y, ys, law = torch.zeros(8, dtype=torch.int64), torch.zeros(8, dtype=torch.int64), torch.zeros(8, 49)
    for args, what in (((y[:4], ys, law), 'labels has 4'), ((y, ys[:4], law), 'labels_swap has 4'),
                       ((y, ys, law[:4]), 'swap_law has 4')):
        with pytest.raises(_lib.HawkeyeLibError, match=what):
            crit([z, s, m], *args)
    with pytest.raises(_lib.HawkeyeLibError, match='mask has 4'):
        crit([z, s, m[:4]], y, ys, law)
    with pytest.raises(_lib.HawkeyeLibError, match=r'448x448 inputs for swap_num \[7, 7\]'):
        crit([z, s, m[:, :9]], y, ys, law)
    with pytest.raises(_lib.HawkeyeLibError, match='ops need CUDA'):     # shapes fine: only then the device check
        crit([z, s, m], y, ys, law)
