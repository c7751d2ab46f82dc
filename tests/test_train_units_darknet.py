"""Train-mode parity of the Darknet-19 and Tiny trainers one unit at a time, against an fp64 restatement fed its own activations and gradients,
and the weight-gradient and BatchNorm-backward reductions at the lengths of the C3 batch (64 x 416^2).

Same method as test_train_units.py (which holds the shared teacher, figures and bounds): an fp64 teacher runs one train-mode step of
`O.darknet_forward(train=True)` / `O.tiny_forward(train=True)` with autograd and records, for every conv + BatchNorm unit, the input the GPU
unit reads and the loss gradient at its output -- for a unit followed by a max-pool, the gradient at the pooled output; for the branch point
layers1.16 both parts (direct from the passthrough, pooled from layers2).  Each trainer unit (`DarknetTrainer._first_forward /
_first_backward / _bn_unit_forward / _unit_backward / _reorg_* / _head_backward`, `TinyTrainer._first_forward / _chain_unit_forward /
_tiny_unit0_backward / _tiny_padded_unit_backward / _head_backward`) then runs on exactly those operands, stored the way the GPU stores them,
and is compared with an fp64 recomputation of that unit.  The leaky slope and each pool window's winner are the GPU's own decisions, taken
from y = z16 * sc + sh recomputed in fp32 from the GPU's stored z, mean and invstd (the rule of train_ops.cu bn_act_bwd).

CPU: the teacher's records chain into the float32 restatement.  GPU: every unit at several sizes and both code paths of the first layer's
weight gradient and of the forward statistics; the whole `DarknetTrainer.backward()` checked unit by unit on the gradients it hands itself
(the wiring: concat slices, reorg, the branch point); the long reductions of the C3 batch.
"""
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import yolo2_oracle as O
from test_train_units import (DEV, SCALE, TOL, Figures, Teacher, _bn_figures, _case_inputs, _grad_figures, _head_check, _leaf_sd,
                              _snap, first_max, make_config, nhwc16, nchw, record, rel_err, rel_l2, unit_ref)

SLOPE = 0.1              # LeakyReLU(0.1) of model/yolo2.py's Conv2d units


# ------------------------------------------------------------------------------------------------
# fp64 teachers
# ------------------------------------------------------------------------------------------------
def _pool(t, key, a):
    p = F.max_pool2d(a, 2)
    p.retain_grad()
    t.pools[key] = p
    return p


def darknet_teacher(sd0, x, data, dtype=torch.float64, device='cpu'):
    """The arithmetic of O.darknet_forward(train=True) with every unit, every max-pool output (t.pools; 'layers1.16' is layers2's leading
    pool), the passthrough's reorg (t.reorg), the concat (t.cat) and the head recorded."""
    t = Teacher()
    t.sd = _leaf_sd(sd0, dtype, device)
    t.pools = {}
    layers = O.darknet19_layers()
    ks = {l['key']: l['k'] for l in layers}

    def unit(key, inp):
        return t.unit(key, inp, key + '.conv.weight', key + '.bn', 1, ks[key], True, slope=SLOPE)

    cur = x.to(device, dtype)
    for l in layers:
        if l['group'] == 'layers1':
            cur = unit(l['key'], cur)
            if l['pool_after']:
                cur = _pool(t, l['key'], cur)
    x1 = cur
    pt = unit('passthrough', x1)
    r = O.reorg(pt)
    r.retain_grad()
    cur = _pool(t, 'layers1.16', x1)
    for l in layers:
        if l['group'] == 'layers2':
            cur = unit(l['key'], cur)
    cat = torch.cat([r, cur], 1)
    cat.retain_grad()
    t.reorg, t.cat = dict(inp=pt, out=r), cat
    a30 = unit('layers3.0', cat)
    t.head = dict(a=a30, w='layers3.1.conv.weight', b='layers3.1.conv.bias')
    return t.finish(F.conv2d(a30, t.sd['layers3.1.conv.weight'], t.sd['layers3.1.conv.bias']), data)


def tiny_teacher(sd0, x, data, dtype=torch.float64, device='cpu'):
    """The arithmetic of O.tiny_forward(train=True) with every unit, the max-pool outputs (t.pools), the pad + stride-1 pool output
    (t.pools_s1) and the head recorded."""
    t = Teacher()
    t.sd = _leaf_sd(sd0, dtype, device)
    t.pools, t.pools_s1 = {}, {}
    cur = x.to(device, dtype)
    layers = O.tiny_layers()
    for l in layers[:-1]:
        key = l['key']
        cur = t.unit(key, cur, key + '.conv.weight', key + '.bn', 1, l['k'], True, slope=SLOPE)
        if l['after'] == 'pool':
            cur = _pool(t, key, cur)
        elif l['after'] == 'pool_s1':
            cur = F.max_pool2d(F.pad(cur, (0, 1, 0, 1), value=O.FLOAT32_MIN), 2, stride=1)
            cur.retain_grad()
            t.pools_s1[key] = cur
    head = layers[-1]['key']
    t.head = dict(a=cur, w=head + '.conv.weight', b=head + '.conv.bias')
    return t.finish(F.conv2d(cur, t.sd[head + '.conv.weight'], t.sd[head + '.conv.bias']), data)


def reorg_t(g):
    """The transpose (= inverse) of O.reorg's permutation: [B,4C,h,w] -> [B,C,2h,2w]."""
    b, c4, h, w = g.shape
    return g.reshape(b, 2, 2, c4 // 4, h, w).permute(0, 3, 4, 1, 5, 2).reshape(b, c4 // 4, 2 * h, 2 * w)


def unit_grads(t, key):
    """(gradient at the unit's output -- pooled when a max-pool follows --, gradient at its unpooled activation from a second consumer, pooled)"""
    if key == 'layers1.16':
        return t.pools[key].grad, t.units['passthrough']['src'].grad, True
    if key in t.pools:
        return t.pools[key].grad, None, True
    return t.units[key]['out'].grad, None, False


# ------------------------------------------------------------------------------------------------
# CPU: the teachers are the restatement, and their records chain
# ------------------------------------------------------------------------------------------------
# fp64 teacher vs fp32 restatement, measured on the CPU: Darknet at 2 x 96^2 feature 1.8e-5, worst parameter gradient 3.0e-5 (rel L2,
# layers1.2.bn.bias); Tiny at 8 x 160^2 feature 3.4e-6, worst parameter gradient 7.7e-6
CPU_CASES = {'darknet': (2, 96, 46, 47), 'tiny': (8, 160, 70, 71)}
FEATURE_FP32 = {'darknet': 1e-4, 'tiny': 1e-4}
GRAD_FP32 = {'darknet': 2e-4, 'tiny': 1e-4}


def _restated_step(net, x, data):
    sd0 = O.make_state_dict(0) if net == 'darknet' else O.make_tiny_state_dict(0)
    sd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v.clone()) for k, v in sd0.items()}
    f32 = O.darknet_forward(sd, x, train=True) if net == 'darknet' else O.tiny_forward(sd, x, train=True)
    pred = O.decode(f32, O.anchors_yolo_voc())
    pred['feature'] = f32
    l32, _ = O.loss(O.anchors_yolo_voc(), data, pred, 0.6)
    O.loss_total(l32).backward()
    return sd0, sd, f32, l32


@pytest.mark.parametrize('net', ['darknet', 'tiny'])
def test_teacher_records_chain_to_the_fp32_restatement(net):
    """The fp64 teacher is the restatement: feature, losses and every parameter gradient agree with the float32 restatement to fp32 rounding;
    every unit recomputed alone by `unit_ref` (leaky 0.1, fused max-pool, the branch point's two gradients) reproduces its records; and the
    records chain: each unit's input is its producer's (pooled) output, reorg backward is the exact transpose of O.reorg, the concat's
    gradient splits exactly into the reorg's and layers2.7's, and at layers1.16 the direct and the pooled part add up to the total."""
    b, size, seed_x, seed_t = CPU_CASES[net]
    x, _, data = _case_inputs(b, size, seed_x, seed_t)
    sd0, sd, f32, l32 = _restated_step(net, x, data)
    t = darknet_teacher(sd0, x, data) if net == 'darknet' else tiny_teacher(sd0, x, data)
    e_f = rel_err(t.feature, f32)
    for k, v in t.losses.items():
        assert abs(v.item() - l32[k].item()) <= 1e-4 * abs(l32[k].item()) + 1e-9, ('loss', k)
    params = [k for k, v in sd.items() if v.requires_grad]
    worst = max((rel_l2(t.sd[k].grad, sd[k].grad), k) for k in params)
    print('%s: fp64 teacher vs fp32 restatement: feature %.2e, worst gradient rel L2 %.2e (%s)' % (net, e_f, *worst))
    assert e_f <= FEATURE_FP32[net], ('feature', e_f)
    assert worst[0] <= GRAD_FP32[net], worst
    # each unit alone, from its own records
    owned = set()
    for key, u in t.units.items():
        gout, gdir, pool = unit_grads(t, key)
        r = unit_ref(u['src'], t.sd[u['conv']], t.sd[u['bn'] + '.weight'], t.sd[u['bn'] + '.bias'], 1, u['k'], True, gout, slope=SLOPE,
                     pool=pool, gdir=gdir)
        assert r['flips'] == 0, key
        assert rel_err(r['act'], u['out']) <= 1e-10 and rel_err(r['z'], u['z']) <= 1e-10, key
        if pool:
            assert rel_err(r['out'], t.pools[key]) <= 1e-12, ('pool', key)
        assert rel_err(r['mean'], u['mean']) <= 1e-8 and rel_err(r['var'], u['var']) <= 1e-10 and r['count'] == u['count'], key
        assert u['src'].grad is None or rel_err(r['dx'], u['src'].grad) <= 1e-9, ('dx', key)
        for name, got in ((u['conv'], r['dw']), (u['bn'] + '.weight', r['dgamma']), (u['bn'] + '.bias', r['dbeta'])):
            assert rel_err(got, t.sd[name].grad) <= 1e-9, (name, key)
            owned.add(name)
    head = t.head
    hr_w, hr_b, hr_a = (v.detach().clone().requires_grad_(True) for v in (t.sd[head['w']], t.sd[head['b']], head['a']))
    F.conv2d(hr_a, hr_w, hr_b).backward(t.feature.grad)
    assert rel_err(hr_w.grad, t.sd[head['w']].grad) <= 1e-9 and rel_err(hr_b.grad, t.sd[head['b']].grad) <= 1e-9
    assert rel_err(hr_a.grad, head['a'].grad) <= 1e-9
    owned |= {head['w'], head['b']}
    assert owned == set(params), sorted(set(params) ^ owned)
    # chaining
    keys = list(t.units)
    if net == 'tiny':
        outs = {**t.pools, **t.pools_s1}
        for prev, key in zip(keys, keys[1:]):
            assert t.units[key]['inp'] is outs.get(prev, t.units[prev]['out']), key
        assert head['a'] is t.units[keys[-1]]['out']
        key = next(iter(t.pools_s1))
        xs = t.units[key]['out'].detach().clone().requires_grad_(True)
        F.max_pool2d(F.pad(xs, (0, 1, 0, 1), value=O.FLOAT32_MIN), 2, stride=1).backward(t.pools_s1[key].grad)
        assert rel_err(xs.grad, t.units[key]['out'].grad) <= 1e-12, 'pad + stride-1 pool backward'
        return
    l1 = [k for k in keys if k.startswith('layers1.')]
    l2 = [k for k in keys if k.startswith('layers2.')]
    for prev, key in zip(l1, l1[1:]):
        assert t.units[key]['inp'] is t.pools.get(prev, t.units[prev]['out']), key
    assert t.units['passthrough']['inp'] is t.units['layers1.16']['out'] and t.units[l2[0]]['inp'] is t.pools['layers1.16']
    for prev, key in zip(l2, l2[1:]):
        assert t.units[key]['inp'] is t.units[prev]['out'], key
    assert t.units['layers3.0']['inp'] is t.cat and head['a'] is t.units['layers3.0']['out']
    # reorg: the transpose is the inverse permutation, and the recorded gradients obey it exactly
    pt = t.reorg['inp'].detach()
    assert torch.equal(reorg_t(O.reorg(pt)), pt)
    assert torch.equal(t.units['passthrough']['out'].grad, reorg_t(t.reorg['out'].grad))
    cpt4 = t.reorg['out'].shape[1]
    assert torch.equal(t.cat.grad[:, :cpt4], t.reorg['out'].grad) and torch.equal(t.cat.grad[:, cpt4:], t.units[l2[-1]]['out'].grad)
    # the branch point: direct + pooled = total
    x1 = t.units['layers1.16']['out']
    xs = x1.detach().clone().requires_grad_(True)
    F.max_pool2d(xs, 2).backward(t.pools['layers1.16'].grad)
    assert rel_err(xs.grad + t.units['passthrough']['src'].grad, x1.grad) <= 1e-12, 'layers1.16 gradient parts'


# ------------------------------------------------------------------------------------------------
# GPU: teacher-forced units
# ------------------------------------------------------------------------------------------------
# about 2x the worst unit measured on an H100 (Darknet at 8 x 160^2, 2 x 416^2, 2 x 608^2, the backward chain at 4 x 128^2, Tiny at 8 x 160^2
# and 2 x 416^2; DESIGN.md section 2), never above TOL of test_train_units.py
DK_TOL = dict(z=1.7e-3, act=2.7e-3, mean=9e-5, var=2.7e-4, running=5e-4, dgamma=8e-4, dbeta=2e-6, dbias=2e-7, dw_l2=1.2e-3, dw_max=1.5e-3,
              dx_l2=6e-4, dx_max=1.1e-3, pool_dx_l2=4e-4, pool_dx_max=8e-4)
assert all(v <= TOL[q] for q, v in DK_TOL.items())


def nchw_d(t):
    """NHWC -> NCHW fp64 on the device (the fp64 references run on the GPU: a 608^2 Darknet unit is too large for the host)."""
    return t.detach().permute(0, 3, 1, 2).double()


def _gout16d(t):
    g16 = nhwc16(t * SCALE)
    return g16, nchw_d(g16) / SCALE


def gpu_y(s, bn, c=None):
    """y = fmaf(z16, sc, sh) with sc = gamma * invstd, sh = beta - mean * sc in fp32 from the GPU's own stored z, mean and invstd: the value
    whose sign picks the leaky slope and whose first maximum takes a window's pooled gradient in bn_act_bwd (train_ops.cu)."""
    c = bn.weight.shape[0] if c is None else c
    z = nchw_d(s.z[..., :c])
    sc = bn.weight.detach().float() * s.invstd.float()
    sh = (bn.bias.detach().double() - s.mean.double() * sc.double()).float()
    return (z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)).float().double()


def ref_unit(s, bn, src, w, k, gout, gdir=None, pool=False):
    """fp64 unit (conv, train-mode BN, leaky 0.1, optional fused max-pool) on the GPU's operands with the GPU's slope and window decisions;
    returned on the host."""
    y = gpu_y(s, bn)
    r = unit_ref(src, w, bn.weight, bn.bias, 1, k, True, gout, round_z=True, mask=(y > 0).double(), slope=SLOPE, pool=pool,
                 win=first_max(y) if pool else None, gdir=gdir)
    return {q: (v.cpu() if torch.is_tensor(v) else v) for q, v in r.items()}


def _darknet_net(sd0):
    import model
    import model.yolo2
    dnn = model.yolo2.Darknet(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    dnn.load_state_dict(sd0, strict=False)
    return dnn.to(DEV).train()


def _darknet_unit_map(eng):
    return dict(zip(eng._k1 + eng._k2 + ['passthrough', 'layers3.0'], eng.units1 + eng.units2 + [eng.unit_pt, eng.units3[0]]))


def _darknet_trainer(dnn):
    tr = dnn.trainer
    tr._repack(torch.device(DEV))
    tr._ensure_arena(dnn, torch.device(DEV))
    tr._main = torch.cuda.current_stream()
    return tr, _darknet_unit_map(dnn.engine)


def _darknet_units(b, size, seed, fuse_stats=True):
    from b200 import ops
    sd0 = O.make_state_dict(0)
    x, _, data = _case_inputs(b, size, seed, seed + 1, slots=5)
    t = darknet_teacher(sd0, x, data, device=DEV)
    dnn = _darknet_net(sd0)
    tr, units = _darknet_trainer(dnn)
    tr.fuse_stats = fuse_stats
    fig = Figures('darknet_%dx%d%s' % (b, size, '' if fuse_stats else '_stats_unfused'), DK_TOL)
    # layers1.0: the fp32 image and fp32 weights, BN, leaky, fused max-pool; weight gradient from the image (fused or two-kernel)
    u0 = units['layers1.0']
    rm0, rv0 = _snap(u0.bn)
    xg = x.to(DEV).float().contiguous()
    s0, a0 = tr._first_forward(xg)
    g16, g64 = _gout16d(t.pools['layers1.0'].grad)
    # the first-layer kernels pack the fp32 image and weights to fp16 (conv0_tc.cu): those are the operands
    ref = ref_unit(s0, u0.bn, xg.half().double(), sd0['layers1.0.conv.weight'].to(DEV).half().double(), 3, g64, pool=True)
    _bn_figures(fig, 'layers1.0', s0, ref, u0.bn, rm0, rv0, a0, ref['out'])
    fig.add('layers1.0', flips=ref['flips'])
    tr._first_backward(xg, s0, None, g16, {})
    _grad_figures(fig, 'layers1.0', tr.arena, tr._pnames('layers1.0', u0), ref)
    cat_ch = t.cat.shape[1]
    dcat16, _ = _gout16d(t.cat.grad)
    for key, tu in t.units.items():
        if key == 'layers1.0':
            continue
        u = units[key]
        rm0, rv0 = _snap(u.bn)
        inp16 = nhwc16(tu['inp'])
        bb, hh, ww = inp16.shape[:3]
        gout, gdir, pool = unit_grads(t, key)
        pool_fwd = pool and key != 'layers1.16'
        if key == 'layers2.7':
            # the trunk's last unit writes its activation into channels [256, 1280) of the concat buffer
            a_off = cat_ch - u.cout
            cat = torch.full((bb, hh, ww, cat_ch), float('nan'), dtype=torch.float16, device=DEV)
            _, s = tr._bn_unit_forward(key, u, inp16, bb, hh, ww, False, out=cat, a_off=a_off)
            assert bool(torch.isnan(cat[..., :a_off]).all()), '%s: activation written outside channels [%d, %d)' % (key, a_off, cat_ch)
            a = cat[..., a_off:]
        else:
            a, s = tr._bn_unit_forward(key, u, inp16, bb, hh, ww, pool_fwd)
        if key == 'passthrough':
            # reorg forward and backward are permutations of fp16 values: bit-exact against the teacher's reorg of the same operands
            a_pt = nhwc16(tu['out'])
            buf = torch.full((bb, hh // 2, ww // 2, cat_ch), float('nan'), dtype=torch.float16, device=DEV)
            tr._reorg_forward(a_pt, buf)
            assert torch.equal(buf[..., :4 * u.cout], nhwc16(O.reorg(nchw_d(a_pt)))), 'reorg forward (yb_reorg_f16) is not the exact permutation'
            assert bool(torch.isnan(buf[..., 4 * u.cout:]).all()), 'reorg forward wrote outside its slice'
            g16 = tr._reorg_backward(dcat16, bb, hh, ww, u.cout)
            assert torch.equal(g16, nhwc16(reorg_t(nchw_d(dcat16)[:, :4 * u.cout]))), \
                'passthrough: reorg backward (yb_reorg_bwd_f16) is not the exact transpose of the concat gradient channels [0, %d)' % (4 * u.cout)
            g64 = nchw_d(g16) / SCALE
        elif key == 'layers2.7':
            g16, g64 = dcat16, nchw_d(dcat16)[:, a_off:] / SCALE
        else:
            g16, g64 = _gout16d(gout)
        gd16, gd64 = _gout16d(gdir) if gdir is not None else (None, None)
        w16 = t.sd[tu['conv']].detach().half().double()
        ref = ref_unit(s, u.bn, nchw_d(inp16), w16, tu['k'], g64, gdir=gd64, pool=pool)
        _bn_figures(fig, key, s, ref, u.bn, rm0, rv0, a, ref['out'] if pool_fwd else ref['act'])
        if pool:
            fig.add(key, flips=ref['flips'])
        grads = {}
        if key == 'layers2.7':
            dx = tr._unit_backward(key, s, bb, grads, da=g16, da_off=a_off)
        elif key == 'layers1.16':
            dx = tr._unit_backward(key, s, bb, grads, da=gd16, dap=g16)
        elif pool:
            dx = tr._unit_backward(key, s, bb, grads, dap=g16)
        else:
            dx = tr._unit_backward(key, s, bb, grads, da=g16)
        _grad_figures(fig, key, tr.arena, tr._pnames(key, u), ref, dx, ref['dx'])
    # the head: bias, weight gradient from the 128-wide padded dz, padded data gradient
    a16 = nhwc16(t.head['a'])
    bb, hh, ww = a16.shape[:3]
    _head_check(fig, tr, t, a16, sd0['layers3.1.conv.weight'].half().double(), hh, ww)
    # yb_head_grad_prepare: exact fp16 of the scaled gradient in channels [0, 125), exact zeros in the padding of a NaN-prefilled buffer
    df = (t.feature.grad.float() * SCALE).contiguous()
    dzh = torch.full((bb, hh, ww, 128), float('nan'), dtype=torch.float16, device=DEV)
    dbias = torch.empty(125, dtype=torch.float32, device=DEV)
    ops.call('yb_head_grad_prepare', df, dzh, dbias, bb, 125, 128, hh * ww)
    assert bool((dzh[..., 125:] == 0).all()), 'yb_head_grad_prepare: padding channels 125..127 are not zero'
    assert torch.equal(dzh[..., :125], df.permute(0, 2, 3, 1).half()), 'yb_head_grad_prepare: dz is not the fp16 of the scaled gradient'
    assert len(fig.units) == len(t.units) + 1 == 23
    return fig


DARKNET_UNIT_CASES = [(8, 160, 'fused'), (8, 160, 'unfused'), (2, 416, 'fused'), (2, 608, 'fused')]


@pytest.mark.gpu
@pytest.mark.parametrize('case', DARKNET_UNIT_CASES, ids=['%dx%d_%s' % c for c in DARKNET_UNIT_CASES])
def test_darknet_units_on_teacher_operands(case, monkeypatch):
    """Every unit of the Darknet-19 trainer on the fp64 teacher's own input and output gradient: layers1.0 (fp32 image, fused max-pool; its
    weight gradient by the fused yb_conv0_wgrad_bn, or with 'unfused' by yb_bn_act_bwd + yb_conv0_wgrad, and the forward statistics by
    yb_bn_stats instead of the conv epilogue), every pooled and plain unit of layers1, the branch point layers1.16 (direct plus pooled
    gradient), the passthrough after reorg backward, layers2.7 writing / reading at channel 256 of the 1280-wide concat, layers3.0 on the
    concat and the padded head.  z, batch and running statistics, activation, dgamma, dbeta, dW and dx per unit.  8 x 160^2, 2 x 416^2 and
    2 x 608^2 give 5^2, 13^2 and 19^2 head grids."""
    b, size, path = case
    if path == 'unfused':
        monkeypatch.setenv('YB_CONV0_WGRAD_FUSED', '0')
    fig = _darknet_units(b, size, 60 + size % 97, fuse_stats=path == 'fused')
    fig.check()


def _tiny_units(b, size, seed):
    import model
    import model.yolo2
    sd0 = O.make_tiny_state_dict(0)
    x, _, data = _case_inputs(b, size, seed, seed + 1, slots=5)
    t = tiny_teacher(sd0, x, data, device=DEV)
    dnn = model.yolo2.Tiny(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    dnn.load_state_dict(sd0, strict=False)
    dnn = dnn.to(DEV).train()
    tr = dnn.trainer
    plan = dnn.unit_keys()
    for i, (_, u, _) in enumerate(plan):
        u.refresh(first_layer=(i == 0), force=True)
    tr._ensure_arena(dnn, torch.device(DEV))
    tr._main = torch.cuda.current_stream()
    fig = Figures('tiny_%dx%d' % (b, size), DK_TOL)
    # unit 0: 16 filters on the 32-filter first-layer kernels; the padding channels of z, a and dz stay exactly zero
    key0, u0, _ = plan[0]
    c0 = u0.cout
    rm0, rv0 = _snap(u0.bn)
    xg = x.to(DEV).float().contiguous()
    tr._x = xg
    s0, a0 = tr._first_forward(xg)
    assert bool((s0.z[..., c0:] == 0).all()) and bool((a0[..., c0:] == 0).all()), 'Tiny %s: padding channels of z / a are not zero' % key0
    sv = types.SimpleNamespace(z=s0.z[..., :c0], mean=s0.mean, invstd=s0.invstd)
    g16, g64 = _gout16d(t.pools[key0].grad)
    ref = ref_unit(sv, u0.bn, xg.half().double(), sd0[key0 + '.conv.weight'].to(DEV).half().double(), 3, g64, pool=True)
    _bn_figures(fig, key0, sv, ref, u0.bn, rm0, rv0, a0[..., :c0], ref['out'])
    fig.add(key0, flips=ref['flips'])
    tr._tiny_unit0_backward(key0, s0, b, {}, g16)
    assert bool((tr._zero_bufs[('dz0', b, size, size)][..., c0:] == 0).all()), 'Tiny %s: padding channels of dz are not zero' % key0
    assert tuple(tr.arena.views[key0 + '.conv.weight'].shape) == (c0, 3, 3, 3)
    _grad_figures(fig, key0, tr.arena, tr._pnames(key0, u0), ref)
    for key, u, after in plan[1:-1]:
        tu = t.units[key]
        rm0, rv0 = _snap(u.bn)
        inp16 = nhwc16(tu['inp'])
        bb, hh, ww, cin = inp16.shape
        cur = inp16
        if tu['inp'] is t.pools[key0]:
            cur = torch.zeros(bb, hh, ww, 32, dtype=torch.float16, device=DEV)       # the first layer's 32-wide buffer
            cur[..., :cin] = inp16
        a, s = tr._chain_unit_forward(key, u, after, cur, bb, hh, ww)
        pool = after == 'pool'
        if after == 'pool_s1':
            # ConstantPad2d + MaxPool2d(2, stride 1): forward exact, backward (first maximum of each window) against fp64 autograd
            au = nchw(s.a_unpooled).requires_grad_(True)
            pooled = F.max_pool2d(F.pad(au, (0, 1, 0, 1), value=O.FLOAT32_MIN), 2, stride=1)
            assert torch.equal(nchw(a), pooled.detach()), '%s: pad + stride-1 max-pool forward is not exact' % key
            gs16, gs64 = _gout16d(t.pools_s1[key].grad)
            pooled.backward(gs64.cpu())
            g16 = torch.empty_like(s.a_unpooled)
            from b200 import ops
            ops.call('yb_maxpool2x2_s1_bwd_f16', s.a_unpooled, gs16, g16, bb, hh, ww, u.cout)
            fig.add(key, pool_dx_l2=rel_l2(nchw(g16) / SCALE, au.grad), pool_dx_max=rel_err(nchw(g16) / SCALE, au.grad))
            g64 = nchw_d(g16) / SCALE
        else:
            g16, g64 = _gout16d(t.pools[key].grad if pool else tu['out'].grad)
        w16 = sd0[key + '.conv.weight'].half().double().to(DEV)
        ref = ref_unit(s, u.bn, nchw_d(inp16), w16, 3, g64, pool=pool)
        _bn_figures(fig, key, s, ref, u.bn, rm0, rv0, s.a_unpooled if after == 'pool_s1' else a, ref['out'])
        if pool:
            fig.add(key, flips=ref['flips'])
        grads = {}
        if s.cin_pad != u.cin:
            # input side zero-padded 16 -> 32: the weight gradient over the padded width, cut back to the 16 real inputs
            dx = tr._tiny_padded_unit_backward(key, s, bb, grads, g16, pool)
            assert tuple(tr.arena.views[key + '.conv.weight'].shape) == (u.cout, cin, 3, 3)
        else:
            dx = tr._unit_backward(key, s, bb, grads, da=None if pool else g16, dap=g16 if pool else None)
        _grad_figures(fig, key, tr.arena, tr._pnames(key, u), ref, dx, ref['dx'])
    a16 = nhwc16(t.head['a'])
    _head_check(fig, tr, t, a16, sd0[t.head['w']].half().double(), a16.shape[1], a16.shape[2])
    assert len(fig.units) == len(t.units) + 1 == 9
    return fig


TINY_UNIT_CASES = [(8, 160), (2, 416)]


@pytest.mark.gpu
@pytest.mark.parametrize('case', TINY_UNIT_CASES, ids=['%dx%d' % c for c in TINY_UNIT_CASES])
def test_tiny_units_on_teacher_operands(case):
    """Every unit of the Tiny trainer on the fp64 teacher's own input and output gradient: the 16-filter first layer on the 32-filter kernels
    (padding channels of z, a and dz exactly zero, weight gradient cut back to 16 filters), unit 1 on the zero-padded 32-wide input (weight
    gradient cut back to 16 inputs), the pooled units, the pad + stride-1 pool and its backward inside the chain, and the head."""
    b, size = case
    _tiny_units(b, size, 74 if size == 160 else 76).check()


# ------------------------------------------------------------------------------------------------
# GPU: DarknetTrainer.backward() as a whole, each unit on the gradient the chain hands it
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_darknet_backward_chain_unit_by_unit():
    """One real step (`forward` + `backward` through the plugin), with every unit's backward recorded.  Each unit's dgamma, dbeta, dW and dx
    are then compared with an fp64 recomputation of that unit from the operands the chain itself saved (its input, z, mean, invstd) and the
    gradient the network's wiring says it must receive, built from the other units' recorded outputs: layers2.7 reads channels [256, 1280) of
    layers3.0's data gradient, the passthrough reads the exact transpose of its channels [0, 256), layers1.16 gets the passthrough's data
    gradient directly plus layers2.1's through the max-pool, every pooled unit of layers1 its consumer's gradient through its pool."""
    import model
    sd0 = O.make_state_dict(0)
    b, size = 4, 128
    x, _, data = _case_inputs(b, size, 62, 63, slots=5)
    dnn = _darknet_net(sd0)
    tr = dnn.trainer
    rec = {}
    unit_bw, first_bw, head_bw = tr._unit_backward, tr._first_backward, tr._head_backward

    def rec_unit(key, s, bb, grads, **kw):
        dx = unit_bw(key, s, bb, grads, **kw)
        rec[key] = dict(s=s, dx=dx)
        return dx

    def rec_first(xx, s0, g_da, g_dap, grads):
        first_bw(xx, s0, g_da, g_dap, grads)
        rec['layers1.0'] = dict(s=s0, dx=None)

    def rec_head(a_last, hh, ww, dfeature, grads):
        rec['head'] = dict(dx=head_bw(a_last, hh, ww, dfeature, grads))
        return rec['head']['dx']

    tr._unit_backward, tr._first_backward, tr._head_backward = rec_unit, rec_first, rec_head
    inference = model.Inference(make_config(), dnn, O.anchors_yolo_voc()).train()
    pred = model._inference(inference, x.to(DEV))
    losses, _ = model.loss(O.anchors_yolo_voc(), {k: v.to(DEV) for k, v in data.items()}, pred, 0.6)
    sum(losses[k] * O.HPARAM_DEFAULT[k] for k in losses).backward()
    torch.cuda.synchronize()
    eng = dnn.engine
    units = _darknet_unit_map(eng)
    k1, k2 = eng._k1, list(eng._k2[:len(eng.units2)])
    cpt4 = eng.unit_pt.cout * 4
    pooled1 = {k for k, p in zip(k1, eng.pools1) if p}

    def grad(key):
        return nchw_d(rec[key]['dx']) / SCALE

    dcat = grad('layers3.0')
    wiring = {'layers3.0': (grad('head'), None, False), k2[-1]: (dcat[:, cpt4:], None, False),
              'passthrough': (reorg_t(dcat[:, :cpt4]), None, False), k1[-1]: (grad(k2[0]), grad('passthrough'), True)}
    for key, nxt in zip(k2, k2[1:]):
        wiring[key] = (grad(nxt), None, False)
    for key, nxt in zip(k1, k1[1:]):
        wiring[key] = (grad(nxt), None, key in pooled1)
    fig = Figures('darknet_backward_chain_%dx%d' % (b, size), DK_TOL)
    params = dict(dnn.named_parameters())
    for key, (gout, gdir, pool) in wiring.items():
        s, u = rec[key]['s'], units[key]
        if key == 'layers1.0':
            src, w = x.to(DEV).half().double(), params[key + '.conv.weight'].detach().half().double()
        else:
            src, w = nchw_d(s.ain), params[key + '.conv.weight'].detach().half().double()
        ref = ref_unit(s, u.bn, src, w, u.ksize, gout, gdir=gdir, pool=pool)
        _grad_figures(fig, key, tr.arena, tr._pnames(key, u), ref, rec[key]['dx'], ref['dx'] if rec[key]['dx'] is not None else None)
    assert len(fig.units) == 22
    fig.check()


# ------------------------------------------------------------------------------------------------
# GPU: the reductions of the C3 batch (64 x 416^2)
# ------------------------------------------------------------------------------------------------
C3_CHUNK = 8             # images per fp64 reference chunk: peak memory of a few GB


def _wgrad_ref(x16, dz16, k, chunk=C3_CHUNK):
    """fp64 dW[cout, k, k, cin] = sum over pixels of dz * shifted x (zero padding), on the device, chunked over images."""
    b, h, w, cin = x16.shape
    cout = dz16.shape[-1]
    p = (k - 1) // 2
    dw = torch.zeros(cout, k, k, cin, dtype=torch.float64, device=DEV)
    for i in range(0, b, chunk):
        xs = F.pad(x16[i:i + chunk].double(), (0, 0, p, p, p, p))
        dz = dz16[i:i + chunk].double().reshape(-1, cout)
        for ky in range(k):
            for kx in range(k):
                dw[:, ky, kx, :] += dz.t() @ xs[:, ky:ky + h, kx:kx + w, :].reshape(-1, cin)
    return dw


def _synth_grad(shape, seed):
    """fp16 gradient with a per-channel mean that is not zero (so a dropped or doubled partial sum shows in every channel)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = shape[-1]
    bias = torch.randn(c, generator=g, device=DEV) * 0.5
    return ((torch.randn(shape, generator=g, device=DEV) + bias) * 0.05 * SCALE / 64).half()


@pytest.mark.gpu
def test_c3_reduction_lengths(monkeypatch):
    """The C3 batch's reductions against fp64 references on the same operands: layers1.0's BatchNorm backward reduce pass (sums of dy and of
    dy * xhat over 64 * 416^2 = 11.1 M rows, routed through the max-pool by the GPU's own window decisions) and its dgamma / dbeta, the
    fused yb_conv0_wgrad_bn weight gradient over the same rows, and yb_conv_wgrad for layers1.2 (2.77 M pixels, 32 -> 64, 3x3) and layers1.4
    (692 k pixels, 64 -> 128, 3x3) at the cost model's split count, one split (the no-atomics store), a ragged last split and 512 splits.
    z, mean and invstd are the GPU's own forward of the C3 input."""
    from b200 import ops
    sd0 = O.make_state_dict(0)
    dnn = _darknet_net(sd0)
    tr, units = _darknet_trainer(dnn)
    b, size = 64, 416
    x = O.synth_images(b, size, size, seed=64).to(DEV)
    with torch.no_grad():
        s0, a0 = tr._first_forward(x)
        a2, s2 = tr._bn_unit_forward('layers1.2', units['layers1.2'], a0, b, size // 2, size // 2, True)
    figs = {}
    # ---- layers1.0: BatchNorm + leaky + pool backward reduce pass, dgamma / dbeta, fused weight gradient ----
    u0 = s0.u
    h, w = size, size
    gp = _synth_grad((b, h // 2, w // 2, 32), 640)
    sums = torch.zeros(64, dtype=torch.float64, device=DEV)
    bnw, bnb = u0.bn.weight.detach(), u0.bn.bias.detach()
    ops.call('yb_bn_act_bwd', 0, s0.z, 32, s0.mean, s0.invstd, bnw, bnb, SLOPE, None, 0, 0, gp, 32, 0, b, h, w, 32, 1, sums, None, 0, 1)
    dgamma, dbeta = torch.empty(32, device=DEV), torch.empty(32, device=DEV)
    dw0 = torch.empty(32, 3, 3, 3, dtype=torch.float32, device=DEV)
    ops.call('yb_conv0_wgrad_bn', x, s0.z, gp, 32, 0, s0.mean, s0.invstd, bnw, bnb, SLOPE, sums, dw0, b, h, w)
    ops.call('yb_bn_param_grad', sums.clone(), 32, dgamma, dbeta, 0, 1.0 / SCALE)
    rows = b * h * w
    sc = (bnw.float() * s0.invstd.float()).double()
    mean, inv = s0.mean.double(), s0.invstd.double()
    ref_s1 = torch.zeros(32, dtype=torch.float64, device=DEV)
    ref_s2 = torch.zeros(32, dtype=torch.float64, device=DEV)

    def dy_chunk(i):
        sv = types.SimpleNamespace(z=s0.z[i:i + C3_CHUNK], mean=s0.mean, invstd=s0.invstd)
        y = gpu_y(sv, u0.bn)
        win = first_max(y)
        up = F.interpolate(nchw_d(gp[i:i + C3_CHUNK]), scale_factor=2, mode='nearest') * win
        dy = torch.where(y > 0, up, up * SLOPE)
        xhat = (nchw_d(s0.z[i:i + C3_CHUNK]) - mean.view(1, -1, 1, 1)) * inv.view(1, -1, 1, 1)
        return dy, xhat

    for i in range(0, b, C3_CHUNK):
        dy, xhat = dy_chunk(i)
        ref_s1 += dy.sum(dim=(0, 2, 3))
        ref_s2 += (dy * xhat).sum(dim=(0, 2, 3))
    figs['layers1.0'] = dict(sum_dy=rel_err(sums[:32], ref_s1), sum_dy_xhat=rel_err(sums[32:], ref_s2),
                             dbeta=rel_err(dbeta, ref_s1 / SCALE), dgamma=rel_err(dgamma, ref_s2 / SCALE))
    # dz = sc * (dy - mean(dy) - xhat * mean(dy xhat)) in fp64 from the exact sums, then dW = sum dz * shifted image
    dw_ref = torch.zeros(32, 3, 3, 3, dtype=torch.float64, device=DEV)
    for i in range(0, b, C3_CHUNK):
        dy, xhat = dy_chunk(i)
        dz = sc.view(1, -1, 1, 1) * (dy - (ref_s1 / rows).view(1, -1, 1, 1) - xhat * (ref_s2 / rows).view(1, -1, 1, 1))
        dw_ref += torch.nn.grad.conv2d_weight(x[i:i + C3_CHUNK].half().double(), (32, 3, 3, 3), dz, padding=1)
        del dy, xhat, dz
    figs['layers1.0'].update(dw_l2=rel_l2(dw0, dw_ref), dw_max=rel_err(dw0, dw_ref))
    del gp
    # ---- yb_conv_wgrad at the long reductions of layers1.2 (input: layers1.0's pooled output) and layers1.4 (layers1.2's) ----
    cases = {'layers1.2': (a0, 64), 'layers1.4': (a2, 128)}
    for key, (xin, cout) in cases.items():
        bb, hh, ww, cin = xin.shape
        dz = _synth_grad((bb, hh, ww, cout), 641 + cout)
        ref = _wgrad_ref(xin, dz, 3)
        res = {}
        kb_total = -(-bb * hh * ww // WGRAD_KP)
        for tag, splits in (('model', None), ('1', 1), ('ragged', 7), ('512', 512)):
            if splits is None:
                monkeypatch.delenv('YB_WGRAD_SPLITS', raising=False)
            else:
                monkeypatch.setenv('YB_WGRAD_SPLITS', str(splits))
            dw = torch.full((cout, 3, 3, cin), float('nan'), dtype=torch.float32, device=DEV)
            ops.call('yb_conv_wgrad', xin, dz, dw, bb, hh, ww, cin, cout, 3, cin, cout)
            res['splits_' + tag] = dict(dw_l2=rel_l2(dw, ref), dw_max=rel_err(dw, ref))
            if splits is not None:
                per_split = -(-kb_total // splits) * WGRAD_KP                # pixels summed by one accumulator (conv_wgrad.cu)
                res['splits_' + tag]['bound'] = 2 * WGRAD_ACC_PER_PIXEL * per_split + 1e-5
                if tag == 'ragged':
                    assert kb_total % (per_split // WGRAD_KP), '%s: %d splits leave no short last split' % (key, splits)
        monkeypatch.delenv('YB_WGRAD_SPLITS', raising=False)
        figs[key] = res
        del dz, ref
    record('c3_reduction_lengths', figs)
    bad = []
    for q in ('sum_dy', 'sum_dy_xhat', 'dbeta', 'dgamma'):
        if figs['layers1.0'][q] > C3_TOL['bn_sums']:
            bad.append('layers1.0 %s = %.3e' % (q, figs['layers1.0'][q]))
    for q in ('dw_l2', 'dw_max'):
        if figs['layers1.0'][q] > C3_TOL['conv0_wgrad_bn']:
            bad.append('layers1.0 yb_conv0_wgrad_bn %s = %.3e' % (q, figs['layers1.0'][q]))
    for key in cases:
        for tag, f in figs[key].items():
            bound = f.get('bound', C3_TOL['conv_wgrad_model'])
            for q in ('dw_l2', 'dw_max'):
                if not f[q] <= bound:
                    bad.append('%s yb_conv_wgrad %s %s = %.3e > %.1e' % (key, tag, q, f[q], bound))
    assert not bad, '; '.join(bad)


# The wgmma accumulators of yb_conv_wgrad lose precision linearly in the number of pixels one accumulator sums (measured on an H100:
# relative error 4.0e-9 per pixel, 1.1e-2 for layers1.2's 2.77 M pixels in one split, 2.1e-5 at 512 splits -- a bias, as of rounding toward
# zero, not a random walk).  The bound of an explicit split count is twice that law; the cost model's own choice is bounded at about twice
# its measured figure.
WGRAD_KP = 128                   # pixels per K-block (conv_wgrad.cu kWgKP)
WGRAD_ACC_PER_PIXEL = 4.0e-9
# measured: reduce-pass sums 2.3e-8, dgamma / dbeta 3.9e-8, yb_conv0_wgrad_bn 4.7e-5, yb_conv_wgrad at the cost model's split count 2.5e-4
# (layers1.2) and 5.6e-5 (layers1.4)
C3_TOL = dict(bn_sums=1e-7, conv0_wgrad_bn=1e-4, conv_wgrad_model=5e-4)
