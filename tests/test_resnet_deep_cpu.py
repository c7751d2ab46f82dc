"""resnet101 / resnet152 without a GPU: the constructors against the executed reference (state_dict keys and shapes), the eval and train-mode
restatements against resnet_deep.npz (tests/golden/make_golden_resnet_deep.py), the trainer's plan and gradient order, and the loss scale
chosen per depth."""
import os

import numpy as np
import pytest
import torch

import resnet_deep_oracle  # noqa: F401  (registers resnet101 / 152 in the oracle's ResNet table)
import resnet_train_oracle as RT
from oracle import yolo2_oracle as O
from test_resnet_train import make_net, oracle_step

DEEP = ('resnet101', 'resnet152')
TRAIN_CASE = ('resnet101', 2, 64, 42, 43)           # as make_golden_resnet_deep.py


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'resnet_deep.npz'))


@pytest.mark.parametrize('name', DEEP)
def test_deep_resnet_state_dict_matches_reference(golden, name):
    """Same keys, in the same order, with the same shapes as the reference's constructor, and the oracle's synthetic state_dict loads."""
    sd = make_net(name).state_dict()
    assert list(sd) == golden['%s_keys' % name].tolist()
    assert [';'.join(str(d) for d in v.shape) for v in sd.values()] == golden['%s_shapes' % name].tolist()
    n_bn = sum(1 for k in sd if k.endswith('running_mean'))
    assert n_bn == {'resnet101': 104, 'resnet152': 155}[name]
    make_net(name, O.make_resnet_state_dict(name, 0))


@pytest.mark.parametrize('name', DEEP)
def test_deep_resnet_restatement_matches_reference(golden, name):
    """The eval restatement (oracle.yolo2_oracle.resnet_forward) against the executed reference's heads to 1e-5, and, for resnet101 at 64^2,
    every block output (its L2 norm to 1e-5 and its first 64 elements; the generator compared the whole tensors)."""
    sd = O.make_resnet_state_dict(name, 0)
    sizes = [(64, 10), (416, 0)] if name == 'resnet101' else [(64, 10)]
    for size, seed in sizes:
        collect = {}
        with torch.no_grad():
            f = O.resnet_forward(sd, O.synth_images(1, size, size, seed=seed), name, collect=collect)
        ref = torch.from_numpy(golden['%s_feature%d' % (name, size)])
        assert ((f - ref).norm() / ref.norm()).item() < 1e-5, (name, size)
        if name != 'resnet101' or size != 64:
            continue
        keys = golden['resnet101_blocks'].tolist()
        assert sorted(keys) == sorted([b['prefix'] for b in O.resnet_blocks(name)] + ['maxpool'])
        for key, norm, head in zip(keys, golden['resnet101_actnorm'], golden['resnet101_acthead']):
            got = collect[key].double()
            assert abs(got.norm().item() - norm) <= 1e-5 * norm, key
            np.testing.assert_allclose(got.flatten()[:64].numpy(), head, rtol=1e-5, atol=1e-5 * float(got.abs().max()), err_msg=key)


def test_deep_resnet_train_restatement_matches_reference(golden):
    """One train() step of the restatement (batch statistics, decode, region loss, autograd) against the reference's own resnet101 at
    2 x 64^2: loss terms 1e-5, every parameter gradient (norm 1e-4 and first elements; the stem's, layer1's and the head's small tensors in
    full) and the running statistics (norm and first elements of every BatchNorm's, the stem's and layer1's in full)."""
    name, b, size, seed_x, seed_t = TRAIN_CASE
    sd0 = O.make_resnet_state_dict(name, 0)
    s = size // 32
    x = O.synth_images(b, size, size, seed=seed_x)
    data = O.norm_data(O.synth_targets(b, size, size, slots=6, seed=seed_t), size, size, s, s)
    _, losses, grads, stats, counts = oracle_step(name, sd0, x, data)
    for k, v in losses.items():
        ref = float(golden['%s_loss_%s' % (name, k)])
        assert abs(v.item() - ref) <= 1e-5 * abs(ref), (k, v.item(), ref)
    params = golden[name + '_params'].tolist()
    assert sorted(grads) == sorted(params)
    assert sum(1 for k in golden.files if '_gfull_' in k) == 1 + 2 + 2 * 10      # head bias, stem BatchNorm, layer1's 10 BatchNorms
    for pname, ref_norm, head in zip(params, golden[name + '_gnorm'], golden[name + '_ghead']):
        gr = grads[pname]
        assert abs(gr.double().norm().item() - ref_norm) <= 1e-4 * ref_norm + 1e-12, pname
        np.testing.assert_allclose(gr.flatten()[:16].numpy(), head, rtol=1e-3, atol=1e-3 * float(np.abs(head).max()) + 1e-12, err_msg=pname)
        key = '%s_gfull_%s' % (name, pname)
        if key in golden.files:
            assert np.linalg.norm(gr.numpy() - golden[key]) <= 1e-4 * np.linalg.norm(golden[key]) + 1e-12, pname
    bns = golden[name + '_bns'].tolist()
    assert sorted(stats) == sorted(bns) and len(bns) == 104
    for prefix, norms, heads in zip(bns, golden[name + '_bufnorm'], golden[name + '_bufhead']):
        mean, var = stats[prefix]
        for exp, norm, head, kind in zip(RT.expected_running(sd0, prefix, mean, var, counts[prefix]), norms, heads, ('running_mean', 'running_var')):
            assert abs(exp.double().norm().item() - norm) <= 1e-4 * norm, (prefix, kind)
            np.testing.assert_allclose(exp[:16].numpy(), head, rtol=1e-4, atol=1e-6, err_msg='%s.%s' % (prefix, kind))
            key = '%s_buf_%s.%s' % (name, prefix, kind)
            if key in golden.files:
                np.testing.assert_allclose(exp.numpy(), golden[key], rtol=1e-4, atol=1e-6, err_msg=key)
    assert sum(1 for k in golden.files if '_buf_' in k) == 2 * 11                   # the stem's and layer1's 10 BatchNorms


@pytest.mark.parametrize('name', DEEP)
def test_deep_resnet_trainer_plan_and_grad_order(name):
    """The trainer's plan holds every block of layer1-layer4 with its units and downsample, each parameter belongs to exactly one planned
    unit, and grad_order() lists every parameter exactly once, head first and stem last.  Building the trainer needs no GPU."""
    from b200 import train_engine
    net = make_net(name)
    tr = train_engine.ResNetTrainer(net)
    blocks = tr._plan()
    assert [p for p, _, _ in blocks] == [b['prefix'] for b in O.resnet_blocks(name)]
    owned = []
    for u in [tr._stem, tr._head] + tr._conv_units():
        owned += [n for n in u.pnames if n is not None]
    owned.append('conv.bias')
    params = {n for n, _ in net.named_parameters()}
    assert len(owned) == len(set(owned)) and set(owned) == params
    order = tr.grad_order()
    assert len(order) == len(set(order)) == len(params) and set(order) == params
    assert order[:2] == ['conv.bias', 'conv.weight'] and order[-3:] == ['bn1.weight', 'bn1.bias', 'conv1.weight']
    assert net.trainer.grad_order() == order


@pytest.mark.parametrize('name, scale', [('resnet18', 16384.0), ('resnet34', 16384.0), ('resnet50', 16384.0), ('resnet101', 4096.0),
                                         ('resnet152', 1024.0)])
def test_resnet_loss_scale_per_depth(name, scale):
    """The static loss scale is chosen from the block count (DESIGN §6): resnet18 / 34 / 50 keep 16384, resnet101 takes 4096 and resnet152
    1024; an explicit grad_scale still wins."""
    from b200 import train_engine
    net = make_net(name)
    assert net.trainer.grad_scale == scale
    assert train_engine.ResNetTrainer(net).grad_scale == scale
    assert train_engine.ResNetTrainer(net, grad_scale=512.0).grad_scale == 512.0
