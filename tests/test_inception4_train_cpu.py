"""Inception-v4 training (b200.train_engine.Inception4Trainer), what needs no GPU: the train-mode restatement in inception4_train_oracle.py
against one executed train() step of the reference with BatchNorm on and off (inception4_train.npz), the trainer's parameter order and block
plan, the refusal of channel-pruned and ratio != 1 models, the excl-pool backward's entry point in the header and the ctypes table, and the
error budget's rounding model of that pool."""
import os

import numpy as np
import pytest
import torch

import inception4_oracle as I
import inception4_train_oracle as T4
from oracle import yolo2_oracle as O
from test_inception4 import build

MODES = {'bn': True, 'nobn': False}


def build_mode(mode, seed=None):
    return build(0 if seed is None else seed) if MODES[mode] else build(tag='nobn')


@pytest.mark.parametrize('mode', sorted(MODES))
def test_train_restatement_vs_reference_golden(golden_dir, mode):
    bn = MODES[mode]
    gold = np.load(os.path.join(golden_dir, 'inception4_train.npz'))
    b, h, w = (int(v) for v in gold['shape'])
    x = O.synth_images(b, h, w, seed=int(gold['image_seed']))
    sd = I.make_state_dict(int(gold['seed_' + mode]), bn=bn)
    _, loss, grads, stats = T4.train_step(sd, x, dtype=torch.float32)
    ref = float(gold['loss_' + mode])
    assert abs(loss.item() - ref) <= 1e-5 * abs(ref), (loss.item(), ref)
    params = [k for k in sd if 'running' not in k]
    pre = 'gnorm_%s_' % mode
    assert sorted(params) == sorted(k[len(pre):] for k in gold.files if k.startswith(pre))
    for k in params:
        n = float(gold[pre + k])
        assert abs(grads[k].norm().item() - n) <= 1e-4 * n, k
        head = gold['ghead_%s_%s' % (mode, k)]
        assert np.allclose(grads[k].flatten()[:len(head)].numpy(), head, rtol=1e-3, atol=1e-4 * n), k
    stat_keys = [k for k in gold.files if k.startswith('stat_%s_' % mode)]
    assert len(stat_keys) == len(stats) and (len(stats) > 0) == bn
    for k, v in stats.items():
        r = torch.from_numpy(gold['stat_%s_%s' % (mode, k)])
        assert (v - r).abs().max().item() <= 1e-5 * max(r.abs().max().item(), 1.0), k


@pytest.mark.parametrize('mode', sorted(MODES))
def test_grad_order_names_every_parameter_once(mode):
    net, _ = build_mode(mode)
    order = net.trainer.grad_order()
    names = [n for n, _ in net.named_parameters()]
    assert len(order) == len(set(order)) == len(names) and set(order) == set(names)
    assert order[:2] == ['features.22.bias', 'features.22.weight'] and order[-1] == 'features.0.conv.weight'
    # backward order: the last block's units before the one before it, every unit's BatchNorm (or bias) before its conv weight
    first = 'features.21.branch3.1.bn.weight' if mode == 'bn' else 'features.21.branch3.1.conv.bias'
    assert order.index(first) < order.index('features.20.branch0.conv.weight')
    second = 'features.6.branch0.bn.bias' if mode == 'bn' else 'features.6.branch0.conv.bias'
    assert order.index(second) < order.index('features.6.branch0.conv.weight')


def cat_offsets(net):
    """Output channel offset of every concatenated unit and of every max-pool branch, computed from the model's CAT and the module widths."""
    f = net.features
    units, pools = {}, {}
    cin = f[2].conv.out_channels
    for i in range(3, 22):
        m = f[i]
        off = 0
        for name in m.CAT:
            if name in m.POOLS:
                pools[i] = off
                off += cin
            else:
                units['features.%d.%s' % (i, name)] = off
                off += m.get_submodule(name).conv.out_channels
        cin = off
    return units, pools


def test_block_plan_offsets_follow_cat():
    net, _ = build()
    tr = net.trainer
    units, pools = cat_offsets(net)
    got_units, got_pools = {}, {}
    for index, m, recs, maxpool in tr.block_plan():
        for key, _, _, off in recs:
            if off is not None:
                got_units[key] = off
        if maxpool is not None:
            got_pools[index] = maxpool
    assert got_units == units
    assert got_pools == pools == {3: 0, 5: 192, 10: 640, 18: 512}
    assert len(tr._plan()) == 149
    assert all(u.cout % 32 == 0 and u.cout_pad == u.cout for u in tr._plan().values())
    # the block buffers' widths and every unit's input width at full width (the identity layout)
    assert [net.blocks[i - 3][2].width for i in (3, 4, 5, 6, 10, 11, 18, 21)] == [160, 192, 384, 384, 1024, 1024, 1536, 1536]
    srcs = {key: src for _, _, recs, _ in tr.block_plan() for key, _, src, _ in recs}
    assert srcs['features.21.branch1_1a'] == srcs['features.21.branch1_1b'] == 'branch1_0'
    assert srcs['features.21.branch2_3a'] == srcs['features.21.branch2_3b'] == 'branch2_2'
    assert srcs['features.6.branch3.1'] == 'pool' and srcs['features.6.branch0'] == 'x'


@pytest.mark.parametrize('tag', ['pruned', 'ratio05'])
def test_pruned_and_ratio_models_are_refused_in_training(tag):
    net, _ = build(tag=tag)
    net.train()
    x = torch.zeros(2, 3, 107, 139)
    with pytest.raises(ValueError, match='training needs the full-width model'):
        net.trainer._check(x)
    with pytest.raises(NotImplementedError):          # a CPU tensor never reaches the trainer
        net(x)
    net.eval()
    with pytest.raises(RuntimeError):
        net(x)


def test_full_width_model_passes_the_check():
    for mode in MODES:
        net, _ = build_mode(mode)
        net.trainer._check(torch.zeros(2, 3, 75, 75))
        with pytest.raises(ValueError):
            net.trainer._check(torch.zeros(2, 3, 74, 139))


def test_train_eval_drops_the_cache():
    net, _ = build()
    net._cache['x'] = 1
    net.train()
    assert net._cache == {}
    net._cache['x'] = 1
    net.eval()
    assert net._cache == {}


def test_new_entry_point_is_declared():
    from b200 import lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'yolo2_b200.h')).read()
    name = 'yb_avgpool3x3_s1_excl_bwd_f16'
    assert name in lib.SIGNATURES and ('int %s(' % name) in header
    from b200 import ops
    assert callable(ops.avgpool3x3_s1_excl_bwd)


def test_rounding_model_stores_the_pool_gradient_in_fp16():
    """The restatement's pool branch with the GPU path's roundings: the pooled values are stored as fp16, and so is the gradient the pool
    hands back to the block input (loss-scaled)."""
    r = T4.Rounding(1024.0)
    x = torch.full((1, 1, 3, 3), 1.0 + 2.0 ** -12, dtype=torch.float64, requires_grad=True)
    y = r.a(I.avg_pool(r.g(x)))
    assert bool((y == 1.0).all())
    y.backward(torch.full_like(y, 1.0 + 2.0 ** -20))
    corner = x.grad[0, 0, 0, 0].item()          # 1/4 + 2 * 1/6 + 1/9 of the output gradients, rounded once at the loss scale
    exact = (1.0 + 2.0 ** -20) * (1 / 4 + 2 / 6 + 1 / 9)
    assert corner != exact and abs(corner - exact) <= exact * 2.0 ** -10
    assert abs(corner * 1024 - float(torch.tensor(exact * 1024).half())) == 0
