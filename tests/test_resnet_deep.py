"""resnet101 / resnet152 on the GPU: inference against the executed reference (resnet_deep.npz) and the eval oracle, and the training step
of b200.train_engine.ResNetTrainer at these depths -- unit by unit on the fp64 teacher's operands (the method of test_train_units.py, so
each bound is independent of depth), the whole step against the fp16 error budget computed in the same run
(tools/resnet_train_error_budget.py), the loss scale's headroom, descent with the eval() hand-over, and train.GraphedStep against the
spread of two eager runs."""
import os
import sys

import numpy as np
import pytest
import torch

import resnet_deep_oracle  # noqa: F401  (registers resnet101 / 152 in the oracle's ResNet table)
import test_train_units as TU
from oracle import yolo2_oracle as O
from test_resnet_train import make_config, make_net, record

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
import resnet_train_error_budget as EB  # noqa: E402

DEV = 'cuda'
FP16_MAX = 65504.0
gpu = pytest.mark.gpu


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def cosine(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (torch.dot(a, b) / (a.norm() * b.norm() + 1e-30)).item()


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'resnet_deep.npz'))


# ------------------------------------------------------------------------------------------------
# inference
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('name', ['resnet101', 'resnet152'])
def test_deep_resnet_heads_and_blocks_vs_golden(golden, name):
    """Heads against the executed reference (64^2 for both, 416^2 for resnet101) within 3e-3, the bound of the other plugins; every
    resnet101 block (`ResNet._block`) fed the eval oracle's own input at 64^2 within 2e-3."""
    sd = O.make_resnet_state_dict(name, 0)
    net = make_net(name, sd).to(DEV).eval()
    heads = {}
    for size, seed in ([(64, 10), (416, 0)] if name == 'resnet101' else [(64, 10)]):
        with torch.no_grad():
            f = net(O.synth_images(1, size, size, seed=seed).to(DEV))
        heads[size] = rel_err(f, torch.from_numpy(golden['%s_feature%d' % (name, size)]))
    blocks = {}
    if name == 'resnet101':
        _, blocks = TU._resnet_eval_blocks(net, sd, O.synth_images(1, 64, 64, seed=10), name)
    record('%s_eval' % name, dict(heads=heads, blocks=blocks))
    for size, e in heads.items():
        assert e <= 3e-3, (name, size, e)
    for p, v in blocks.items():
        assert v['rel'] <= 2e-3, (p, v)


@gpu
@pytest.mark.parametrize('name', ['resnet101', 'resnet152'])
def test_deep_resnet_batch32_416(name):
    """Batch 32 at 416^2 against the eval oracle run in fp32 on the GPU (TF32 off), judged by the worst image; and the forward captured in
    a CUDA graph gives the eager forward's bits."""
    sd = O.make_resnet_state_dict(name, 0)
    net = make_net(name, sd).to(DEV).eval()
    x = O.synth_images(32, 416, 416, seed=3).to(DEV)
    with torch.no_grad():
        f = net(x)
        flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            ref = O.resnet_forward({k: v.to(DEV) for k, v in sd.items()}, x, name)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
        worst = max(rel_err(f[i], ref[i]) for i in range(32))
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fg = net(x)
        graph.replay()
        torch.cuda.synchronize()
    record('%s_batch32_416' % name, dict(worst_image=worst))
    assert worst <= 3e-3, worst
    assert torch.equal(fg, f), 'graphed forward differs from the eager one'


# ------------------------------------------------------------------------------------------------
# training, unit by unit (test_train_units.py's method, at the trainer's own loss scale)
# ------------------------------------------------------------------------------------------------
@gpu
def test_resnet101_units_on_teacher_operands(monkeypatch):
    """Every unit of resnet101 at 8 x 160^2 on the fp64 teacher's own operands, stored as the GPU stores them at resnet101's loss scale:
    the stem, the first block of each stage with its downsample, the 23 layer3 blocks, the 2048-channel layer4 units, every join and the
    head, held to the per-unit bounds resnet50 meets (test_train_units.TOL) except one.  The running-statistics figure is relative to
    |running mean| floored at 1e-3, so a channel whose updated running mean lands near 0 turns a batch-mean error far inside its own bound
    into a large ratio: on an H100 layer4.0.conv2 measured 2.3e-3 there while its batch mean was 2.2e-5 of the channel spread (bound 1e-4)
    and its variance 8.5e-5 (bound 3e-4).  With 104 BatchNorms such a channel is more likely than in resnet50's 53, so that figure is held
    to 4e-3."""
    monkeypatch.setattr(TU, 'SCALE', make_net('resnet101').trainer.grad_scale)
    fig = TU._resnet_units('resnet101', 8, 160, 90)
    for key in ('conv1', 'layer1.0.downsample', 'layer2.0.downsample', 'layer3.0.downsample', 'layer4.0.downsample', 'layer3.11.conv2',
                'layer4.2.conv3', 'head'):
        assert key in fig.units, key
    fig.tol = dict(TU.TOL, running=4e-3)
    fig.check()


@gpu
def test_resnet152_layer3_block_on_teacher_operands():
    """One mid-layer3 block of resnet152 (layer3.17, at 8 x 160^2, resnet152's loss scale): each unit on the fp64 teacher's operands, the
    block join forward and backward, within test_train_units.TOL."""
    name, p = 'resnet152', 'layer3.17'
    sd0 = O.make_resnet_state_dict(name, 0)
    x, _, data = TU._case_inputs(8, 160, 90, 91, slots=5)
    t = TU.resnet_teacher(sd0, x, data, name, device=DEV)
    net = make_net(name, sd0).to(DEV).train()
    tr = net.trainer
    scale = tr.grad_scale
    tr._plan()
    tr._repack(torch.device(DEV))
    tr._ensure_arena(net, torch.device(DEV))
    tr._main = torch.cuda.current_stream()
    fig = TU.Figures('%s_%s_8x160' % (name, p))
    units = {u.key: u for u in tr._conv_units()}
    for key in t.joins[p]['units']:
        tu, u = t.units[key], units[key]
        rm0, rv0 = TU._snap(u.bn)
        inp16 = TU.nhwc16(tu['inp'])
        bb, hh, ww = inp16.shape[:3]
        a, s = tr._unit_forward(u, inp16, bb, hh, ww)
        g16 = TU.nhwc16(tu['out'].grad * scale)
        w16 = t.sd[tu['conv']].detach().half().double().cpu()
        ref = TU.unit_ref(TU.nchw(inp16), w16, sd0[tu['bn'] + '.weight'], sd0[tu['bn'] + '.bias'], tu['stride'], tu['k'], tu['relu'],
                          TU.nchw(g16) / scale, round_z=True, mask=(TU.nchw(a) > 0).double())
        TU._bn_figures(fig, key, s, ref, u.bn, rm0, rv0, a, ref['out'])
        grads = {}
        dx = tr._res_unit_backward(s, bb, grads, g16)
        f = dict(dw_l2=TU.rel_l2(tr.arena.views[u.pnames[0]], ref['dw']), dw_max=TU.rel_err(tr.arena.views[u.pnames[0]], ref['dw']),
                 dgamma=TU.rel_err(tr.arena.views[u.pnames[1]], ref['dgamma']), dbeta=TU.rel_err(tr.arena.views[u.pnames[2]], ref['dbeta']),
                 dx_l2=TU.rel_l2(TU.nchw(dx) / scale, ref['dx']), dx_max=TU.rel_err(TU.nchw(dx) / scale, ref['dx']))
        fig.add(key, **f)
    j = t.joins[p]
    m16, r16 = TU.nhwc16(j['main']), TU.nhwc16(j['res'])
    exp = torch.relu(m16.float() + r16.float()).half()
    tr._join_forward(m16, r16)
    assert torch.equal(m16, exp)
    bb, hh, ww = j['xin'].shape[0], j['xin'].shape[2], j['xin'].shape[3]
    gm16, gb16 = TU.nhwc16(j['xm'].grad * scale), TU.nhwc16(j['skip'].grad * scale)
    g = tr._join_backward(TU.nhwc16(j['xin']), gm16, gb16, 1, bb, hh, ww)
    prev = list(t.joins)[list(t.joins).index(p) - 1]
    fig.add('join ' + p, join_l2=TU.rel_l2(TU.nchw(g) / scale, t.joins[prev]['pre'].grad),
            join_max=TU.rel_err(TU.nchw(g) / scale, t.joins[prev]['pre'].grad))
    assert len(fig.units) == 4
    fig.check()


# ------------------------------------------------------------------------------------------------
# training, whole step
# ------------------------------------------------------------------------------------------------
class Peaks(object):
    """Largest |gradient| the trainer stores in fp16 during a backward, per tensor kind and unit: every unit's dz, every data gradient a
    unit hands back, every block-boundary gradient and the stem's max-pool backward (test-side wrappers of the trainer's methods)."""

    def __init__(self, monkeypatch):
        from b200 import train_engine as TE
        cls = TE.ResNetTrainer
        self.peak = {}
        bn0, ru0, jb0, sb0 = cls._bn_backward, cls._res_unit_backward, cls._join_backward, cls._stem_backward

        def note(key, t):
            self.peak[key] = max(self.peak.get(key, 0.0), float(t.float().abs().max()))

        def bn(tr, key, s, b, grads, dz, *args, **kw):
            bn0(tr, key, s, b, grads, dz, *args, **kw)
            note('dz ' + key, dz)

        def ru(tr, s, b, grads, da):
            g = ru0(tr, s, b, grads, da)
            note('dx ' + s.u.key, g)
            return g

        def jb(mask, gm, gb, stride_b, b, h, w):
            g = jb0(mask, gm, gb, stride_b, b, h, w)
            note('join %dx%dx%d' % (h, w, gm.shape[-1]), g)
            return g

        def sb(tr, x, st, stem_a, g, grads):
            da = sb0(tr, x, st, stem_a, g, grads)
            note('stem pool dx', da)
            return da
        monkeypatch.setattr(cls, '_bn_backward', bn)
        monkeypatch.setattr(cls, '_res_unit_backward', ru)
        monkeypatch.setattr(cls, '_join_backward', staticmethod(jb))
        monkeypatch.setattr(cls, '_stem_backward', sb)

    def top(self):
        k = max(self.peak, key=self.peak.get)
        return k, self.peak[k]


def _stage(pname):
    return pname.split('.')[0] if pname.startswith('layer') else {'conv1.weight': 'stem', 'bn1.weight': 'stem', 'bn1.bias': 'stem'}.get(pname, 'head')


def step_figures(f, grads, f_ref, g_ref, last):
    """Feature (max |d| / max |ref|), median / worst gradient cosine, worst cosine of the head + last block, median cosine per stage."""
    cos = {k: cosine(grads[k], g_ref[k]) for k in g_ref}
    late = [c for k, c in cos.items() if k.startswith('conv.') or k.startswith(last + '.')]
    stages = {}
    for k, c in cos.items():
        stages.setdefault(_stage(k), []).append(c)
    return dict(feature=rel_err(f, f_ref), median_cosine=float(np.median(list(cos.values()))), worst_cosine=min(cos.values()),
                late_cosine=min(late), stage_median_cosine={s: float(np.median(v)) for s, v in stages.items()})


STEP_CASES = [('resnet101', 8, 160), ('resnet152', 8, 160), ('resnet101', 2, 416)]


@gpu
@pytest.mark.parametrize('case', STEP_CASES, ids=['%s_%dx%d' % c for c in STEP_CASES])
def test_deep_resnet_training_step(monkeypatch, case):
    """One train() step through the plugin surface against the fp32 restatement with CPU autograd, held to the error budget of the GPU
    path's fp16 roundings at the trainer's loss scale computed here on the same batch (tools/resnet_train_error_budget.py): feature
    <= 1.5x the budget's, median and head + last block gradient cosine >= the budget's - 0.1, every stage's median cosine >= the budget's
    - 0.2 where the budget keeps at least 0.3.  The loss scale's headroom: the gradient guard does not fire and the largest stored
    |gradient| stays 8-fold below 65504.  For resnet101 at 8 x 160^2, 15 SGD steps then reduce the loss, and eval() runs on the trained
    state: every block fed the eval oracle's own input on the trained state_dict within 2e-3, and the end-to-end feature far closer to the
    oracle on the trained state than to the initial one.  End to end, the per-block errors compound over 33 blocks (measured 0.14 on an
    H100, where stale operands would be 412 off; resnet50 measures 3.2e-2 over 16 blocks)."""
    import model
    import train as yb_train
    name, b, size = case
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    sd0 = O.make_resnet_state_dict(name, 0)
    s = size // 32
    x = O.synth_images(b, size, size, seed=90)
    tgt = O.synth_targets(b, size, size, slots=5, seed=91)
    data = O.norm_data(tgt, size, size, s, s)
    peaks = Peaks(monkeypatch)
    net = make_net(name, sd0).to(DEV).train()
    tr = net.trainer
    inference = model.Inference(cfg, net, anchors).train()
    pred = model._inference(inference, x.to(DEV))
    losses, _ = model.loss(anchors, {k: v.to(DEV) for k, v in data.items()}, pred, 0.6)
    sum(losses[k] * O.HPARAM_DEFAULT[k] for k in losses).backward()
    torch.cuda.synchronize()
    found_inf = float(tr.found_inf)
    grads = {k: p.grad.detach().double().cpu() for k, p in net.named_parameters()}
    assert all(bool(torch.isfinite(g).all()) for g in grads.values())
    assert all(int(v) == 1 for k, v in net.state_dict().items() if k.endswith('num_batches_tracked'))
    f_ref, g_ref = EB.step(sd0, x, data, name, False)
    f_b, g_b = EB.step(sd0, x, data, name, True, tr.grad_scale)
    last = 'layer4.%d' % (len(net.layer4) - 1)
    got = step_figures(pred['feature'], grads, f_ref, g_ref, last)
    bud = step_figures(f_b, g_b, f_ref, g_ref, last)
    where, top = peaks.top()
    record('%s_train_step_%dx%d' % case, dict(gpu=got, budget=bud, grad_scale=tr.grad_scale, found_inf=found_inf, peak_grad=top,
                                                peak_at=where, headroom=FP16_MAX / top))
    assert found_inf == 0.0
    assert top <= FP16_MAX / 8, (where, top)
    assert got['feature'] <= 1.5 * bud['feature'] + 1e-3, (got, bud)
    assert got['median_cosine'] >= bud['median_cosine'] - 0.1, (got, bud)
    assert got['late_cosine'] >= bud['late_cosine'] - 0.1, (got, bud)
    for st, c in bud['stage_median_cosine'].items():
        if c >= 0.3:
            assert got['stage_median_cosine'][st] >= c - 0.2, (st, got, bud)
    if case != ('resnet101', 8, 160):
        return
    opt = torch.optim.SGD(net.parameters(), 1e-3, momentum=0.9)
    batch = dict(tensor=x, yx_min=tgt['yx_min'], yx_max=tgt['yx_max'], cls=tgt['cls'])
    hist = [float(yb_train.iterate(inference, opt, anchors, cfg, batch)['loss_total'].item()) for _ in range(15)]
    net.eval()
    xe = x[:2]
    sd_t = {k: v.detach().float().cpu() for k, v in net.state_dict().items() if not k.endswith('num_batches_tracked')}
    e_eval, blocks = TU._resnet_eval_blocks(net, sd_t, xe, name)
    with torch.no_grad():
        e_stale = rel_err(O.resnet_forward(sd0, xe, name), O.resnet_forward(sd_t, xe, name))
    record('%s_descent_and_eval' % name, dict(losses=hist, vs_trained_state=e_eval, stale_state_would_be=e_stale,
                                              worst_block=max((v['rel'], p) for p, v in blocks.items())))
    assert hist[-1] < 0.9 * hist[0], hist
    for p, v in blocks.items():
        assert v['rel'] <= 2e-3, (p, v)
    assert e_eval <= 0.3 and e_eval <= 0.01 * e_stale, (e_eval, e_stale)


@gpu
def test_resnet101_graphed_step_within_eager_spread():
    """train.GraphedStep on resnet101 against eager train.iterate from the same state, three SGD steps each.  Eager runs differ from each
    other because the batch statistics and weight gradients are summed with float atomics, and 104 train-mode BatchNorms amplify that: on
    an H100 two eager runs measured 1.8 % and 12 % apart in the loss in two sessions, so one pair does not estimate the spread.  The spread
    is therefore the largest distance between any two of four eager runs, and the graphed run's median distance to those four must stay
    within it (losses, parameter-update cosine, running statistics), with small absolute floors."""
    import model
    import train as yb_train
    name = 'resnet101'
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    sd0 = O.make_resnet_state_dict(name, 0)
    b, size = 4, 128
    batches = []
    for i in range(2):
        t = O.synth_targets(b, size, size, slots=6, seed=61 + i)
        batches.append(dict(tensor=O.synth_images(b, size, size, seed=71 + i).to(DEV), yx_min=t['yx_min'].to(DEV), yx_max=t['yx_max'].to(DEV),
                            cls=t['cls'].to(DEV)))

    def run(graphed):
        net = make_net(name, sd0).to(DEV).train()
        inference = model.Inference(cfg, net, anchors).train()
        opt = torch.optim.SGD(net.parameters(), 1e-3, momentum=0.9)
        step = yb_train.GraphedStep(inference, opt, anchors, cfg) if graphed else (lambda d: yb_train.iterate(inference, opt, anchors, cfg, d))
        losses = [float(step(batches[i % 2])['loss_total'].item()) for i in range(3)]
        if graphed:
            assert step.launches > 0 and len(step.graphs) == 1
            step.close()
        assert float(net.trainer.found_inf) == 0.0
        return np.array(losses), {k: v.detach().double().cpu().clone() for k, v in net.state_dict().items()}

    def distance(la, sa, lb, sb):
        upd = [cosine(sa[k] - sd0[k].double(), sb[k] - sd0[k].double()) for k in sd0 if 'running' not in k]
        run = max(((sa[k] - sb[k]).norm() / sa[k].norm().clamp_min(1e-30)).item() for k in sd0 if 'running' in k)
        return dict(loss=float(np.max(np.abs(la - lb) / np.abs(la))), median_update_cosine=float(np.median(upd)), running=run)

    eager = [run(False) for _ in range(4)]
    lg, sg = run(True)
    for k in sg:
        if k.endswith('num_batches_tracked'):
            assert int(sg[k]) == 3 and all(int(s[k]) == 3 for _, s in eager), k
    pairs = [distance(*eager[i], *eager[j]) for i in range(4) for j in range(i + 1, 4)]
    to_graphed = [distance(le, se, lg, sg) for le, se in eager]
    spread = dict(loss=max(d['loss'] for d in pairs), median_update_cosine=min(d['median_update_cosine'] for d in pairs),
                  running=max(d['running'] for d in pairs))
    graphed = {q: float(np.median([d[q] for d in to_graphed])) for q in spread}
    record('%s_graphed_vs_eager' % name, dict(eager_spread=spread, graphed_median=graphed, eager_pairs=pairs, graphed_to_eager=to_graphed,
                                              losses=dict(eager=[le.tolist() for le, _ in eager], graphed=lg.tolist())))
    assert graphed['loss'] <= spread['loss'] + 1e-3, (graphed, spread)
    assert graphed['median_update_cosine'] >= spread['median_update_cosine'] - 0.05, (graphed, spread)
    assert graphed['running'] <= spread['running'] + 1e-3, (graphed, spread)
