"""DenseNet training, what needs no GPU: the fp64 restatement of the train-mode step (densenet_train_oracle.py) against the executed
reference (tests/golden/densenet_train.npz) and its fp16 rounding model, the trainer's parameter order, the new entry points in the header and the ctypes table, and the
train-mode refusals."""
import os
import re

import numpy as np
import pytest
import torch

import densenet_oracle as D
import densenet_train_oracle as T
from oracle import yolo2_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ENTRIES = ('yb_conv1x1_preact_stats_fwd', 'yb_conv1x1_preact_wgrad', 'yb_bn_batch_fold', 'yb_bn_preact_bwd', 'yb_bn_running_update_batch')


def build(name, seed=0, **kwargs):
    import configparser
    import model
    import model.densenet
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'}})
    net = getattr(model.densenet, name)(model.ConfigChannels(config), O.anchors_yolo_voc(), 20, **kwargs)
    if name != 'densenet161':
        net.load_state_dict(D.make_densenet_state_dict(name, seed), strict=False)
    return net


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'densenet_train.npz'))


def test_restatement_vs_reference_golden(golden):
    """The restatement of the step against one executed train()-mode step of the reference's densenet121, both in float32 (the fixture's
    arithmetic: in float64 the 121 train-mode BatchNorms move the stem's gradient norm by 4e-4 relative)."""
    b, h, w = (int(v) for v in golden['shape'])
    sd = D.make_densenet_state_dict('densenet121', 0)
    x = O.synth_images(b, h, w, seed=int(golden['image_seed']))
    loss, _, grads, run = T.step(sd, x, name='densenet121', dtype=torch.float32)
    ref = float(golden['loss'])
    assert abs(loss.item() - ref) <= 1e-5 * abs(ref)
    names = [k[len('gnorm_'):] for k in golden.files if k.startswith('gnorm_')]
    assert set(names) == set(grads)
    for k in names:
        n = float(golden['gnorm_' + k])
        assert abs(grads[k].norm().item() - n) <= 1e-4 * n, k
        head = torch.from_numpy(golden['ghead_' + k]).double()
        assert torch.allclose(grads[k].flatten()[:head.numel()].double(), head, rtol=1e-4, atol=1e-4 * n), k
    stats = [k[len('stat_'):] for k in golden.files if k.startswith('stat_')]
    assert set(stats) == set(run)
    for k in stats:
        v = torch.from_numpy(golden['stat_' + k]).double()
        assert (run[k].double() - v).abs().max().item() <= 1e-5 * max(v.abs().max().item(), 1.0), k


def test_rounding_model_budget():
    """The fp16 rounding model moves the step by the fp16 floor and no more (the budget the GPU step is held to is neither empty nor chaos)."""
    sd = D.make_densenet_state_dict('densenet121', 0)
    x = O.synth_images(2, 64, 96, seed=4)
    ref = T.step(sd, x)
    got = T.step(sd, x, rnd=T.Rounding(1024.0))
    e = T.step_errors(got[1], got[2], got[3], ref[1], ref[2], ref[3], sorted(ref[2]))
    assert 1e-5 < e['feature'] < 0.1 and e['grad_cosine'][0] > 0.8, e


@pytest.mark.parametrize('name', ['densenet121', 'densenet169', 'densenet201'])
def test_grad_order_covers_every_parameter_once(name):
    from b200 import train_engine
    net = build(name)
    order = train_engine.DenseNetTrainer(net).grad_order()
    assert len(order) == len(set(order))
    assert set(order) == set(n for n, _ in net.named_parameters())


def test_new_entries_declared_and_bound():
    from b200 import lib
    with open(os.path.join(ROOT, 'include', 'yolo2_b200.h')) as fh:
        header = fh.read()
    for name in NEW_ENTRIES:
        m = re.search(r'int %s\(([^;]*)\);' % name, header)
        assert m is not None, name
        args = [a for a in m.group(1).split(',') if a.strip()]
        assert len(args) == len(lib.SIGNATURES[name]), name
    assert re.search(r'typedef struct yb_bn_running \{\s*float\* running_mean;\s*float\* running_var;\s*int channels;\s*float momentum;\s*\} yb_bn_running;',
                     header)


def test_cpu_tensor_refused_in_train_mode():
    net = build('densenet121').train()
    with pytest.raises(NotImplementedError, match='CPU tensor'):
        net(torch.zeros(1, 3, 64, 64))


def test_drop_rate_refused_in_train_mode(monkeypatch):
    """drop_rate > 0 in train mode raises NotImplementedError naming drop_rate (eval mode is unaffected)."""
    net = build('densenet121', drop_rate=0.2).train()
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))      # the refusal comes before any kernel runs
    with pytest.raises(NotImplementedError, match='drop_rate'):
        net(torch.zeros(1, 3, 64, 64))


def test_densenet161_refused_in_both_modes(monkeypatch):
    net = build('densenet161').eval()
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    with pytest.raises(NotImplementedError, match='96-channel stem.*growth rate 48'):
        net(torch.zeros(1, 3, 64, 64))
    net.train()
    with pytest.raises(NotImplementedError, match='96-channel stem.*growth rate 48'):
        net(torch.zeros(1, 3, 64, 64))
