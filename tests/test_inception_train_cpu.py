"""Inception-v3 training (b200.train_engine.InceptionTrainer), what needs no GPU: the train-mode restatement in inception_train_oracle.py
against one executed train() step of the reference (inception_train.npz), the trainer's parameter order, the BatchNorm channel chunks, and
the new C entry points in the header and the ctypes table."""
import os

import numpy as np
import torch

import inception_oracle as I
import inception_train_oracle as T
from oracle import yolo2_oracle as O
from test_inception import build

NEW_ENTRIES = ('yb_conv2d_wgrad', 'yb_unpack_wgrad_khw', 'yb_pack_weight_dgrad_khw_f16', 'yb_stem3x3_s2_raw_fwd', 'yb_stem3x3_s2_wgrad',
               'yb_maxpool3x3_s2_valid_bwd_f16', 'yb_join_f16', 'yb_pack_weights_khw_batch')


def test_train_restatement_vs_reference_golden(golden_dir):
    gold = np.load(os.path.join(golden_dir, 'inception_train.npz'))
    b, h, w = (int(v) for v in gold['shape'])
    x = O.synth_images(b, h, w, seed=int(gold['image_seed']))
    sd = I.make_inception_state_dict(0)
    _, loss, grads, stats = T.train_step(sd, x, dtype=torch.float32)
    ref = float(gold['loss'])
    assert abs(loss.item() - ref) <= 1e-5 * abs(ref), (loss.item(), ref)
    params = [k for k in sd if 'running' not in k]
    assert sorted('gnorm_' + k for k in params) == sorted(k for k in gold.files if k.startswith('gnorm_'))
    for k in params:
        n = float(gold['gnorm_' + k])
        assert abs(grads[k].norm().item() - n) <= 1e-4 * n, k
        head = gold['ghead_' + k]
        assert np.allclose(grads[k].flatten()[:len(head)].numpy(), head, rtol=1e-3, atol=1e-4 * n), k
    for k, v in stats.items():
        r = torch.from_numpy(gold['stat_' + k])
        assert (v - r).abs().max().item() <= 1e-5 * max(r.abs().max().item(), 1.0), k


def test_grad_order_names_every_parameter_once():
    net = build()
    order = net.trainer.grad_order()
    names = [n for n, _ in net.named_parameters()]
    assert len(order) == len(set(order)) == len(names) and set(order) == set(names)
    assert order[:2] == ['conv.bias', 'conv.weight'] and order[-1] == 'Conv2d_1a_3x3.conv.weight'
    # backward order: Mixed_7c's units before Mixed_7b's, every unit's BatchNorm before its conv weight
    assert order.index('Mixed_7c.branch_pool.bn.weight') < order.index('Mixed_7b.branch1x1.conv.weight')
    assert order.index('Mixed_5b.branch1x1.bn.bias') < order.index('Mixed_5b.branch1x1.conv.weight')


def test_trainer_plan_widths():
    """The buffer width each unit reads: the padded 80- and 48-filter outputs, and every Mixed block's input width."""
    units = build().trainer._plan()
    assert len(units) == 94
    assert (units['Conv2d_3b_1x1'].cout_pad, units['Conv2d_4a_3x3'].cin_pad) == (96, 96)
    assert (units['Mixed_5b.branch5x5_1'].cout_pad, units['Mixed_5b.branch5x5_2'].cin_pad) == (64, 64)
    widths = {'Mixed_5b': 192, 'Mixed_5c': 256, 'Mixed_5d': 288, 'Mixed_6a': 288, 'Mixed_6b': 768, 'Mixed_7a': 768, 'Mixed_7b': 1280,
              'Mixed_7c': 2048}
    for name, c in widths.items():
        assert units[name + ('.branch3x3' if name == 'Mixed_6a' else '.branch3x3_1' if name == 'Mixed_7a' else '.branch1x1')].cin_pad == c, name


def test_bn_chunks_cover_every_width():
    from b200.train_engine import _bn_chunks
    for c in sorted({cout for _, cout, _, _, _, _, _ in I.units().values()}):
        chunks = _bn_chunks(c)
        assert sum(n for _, n in chunks) == c and all(256 % (n // 8) == 0 for _, n in chunks), c
        assert [o for o, _ in chunks] == [sum(n for _, n in chunks[:i]) for i in range(len(chunks))]


def test_new_entry_points_are_declared():
    from b200 import lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'yolo2_b200.h')).read()
    for name in NEW_ENTRIES:
        assert name in lib.SIGNATURES and ('int %s(' % name) in header, name


def test_khw_pack_table_matches_the_header_struct():
    """b200.train_engine.KhwPackPlan builds the device table of yb_pack_weights_khw_batch with numpy: field order, sizes and the 56-byte stride
    must be those of `yb_pack_khw_unit` in include/yolo2_b200.h (3 pointers, a long long, 6 ints on LP64)."""
    import re
    from b200.train_engine import KhwPackPlan
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'yolo2_b200.h')).read()
    body = re.search(r'typedef struct yb_pack_khw_unit \{(.*?)\} yb_pack_khw_unit;', header, re.S).group(1)
    fields = []
    for decl in body.split(';'):
        decl = decl.strip()
        if not decl:
            continue
        m = re.match(r'(const float\*|void\*|long long|int) (.*)', decl)
        assert m, decl
        for name in m.group(2).split(','):
            fields.append(({'const float*': 'ptr', 'void*': 'ptr'}.get(m.group(1), m.group(1)), name.strip()))
    assert [k for k, _ in fields] == ['ptr'] * 3 + ['long long'] + ['int'] * 6, fields
    assert [n for _, n in fields] == ['w_oihw', 'out_fwd', 'out_dgrad', 'elem0', 'cout', 'cin', 'kh', 'kw', 'cout_pad', 'cin_pad']
    dt = KhwPackPlan.DTYPE
    assert dt.itemsize == 56 and len(dt.names) == len(fields)
    assert dt.names == ('w', 'f', 'd', 'e0', 'cout', 'cin', 'kh', 'kw', 'cp', 'cip')
    assert [dt.fields[n][1] for n in dt.names] == [0, 8, 16, 24, 32, 36, 40, 44, 48, 52]
    assert [dt.fields[n][0].itemsize for n in dt.names] == [8, 8, 8, 8, 4, 4, 4, 4, 4, 4]


def test_error_budget_rounding_model():
    """inception_train_oracle.Rounding, the error budget's model of the GPU path: values stored as fp16, weights read as fp16 with their
    gradient passed straight through, and stored gradients rounded to fp16 at the loss scale."""
    r = T.Rounding(1024.0)
    x = torch.tensor([1.0 + 2.0 ** -12, 3.0], dtype=torch.float64, requires_grad=True)
    y = r.a(x)
    assert y.tolist() == [1.0, 3.0]
    y.backward(torch.tensor([1.0 + 2.0 ** -20, 1e-11], dtype=torch.float64))
    assert x.grad.tolist() == [1.0, 0.0]                    # 1e-11 * 1024 rounds to zero below half of fp16's smallest subnormal
    w = torch.tensor([1.0 + 2.0 ** -12], dtype=torch.float64, requires_grad=True)
    (r.w(w) * 3.0).sum().backward()
    assert r.w(w).item() == 1.0 and w.grad.item() == 3.0
    z = torch.tensor([1.0 + 2.0 ** -12], dtype=torch.float64, requires_grad=True)
    g = r.g(z)
    assert g.item() == z.item()
    g.backward(torch.tensor([1.0 + 2.0 ** -20], dtype=torch.float64))
    assert z.grad.item() == 1.0
