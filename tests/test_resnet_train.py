"""Training of the ResNet plugin (model.resnet in train() mode, b200.train_engine.ResNetTrainer).

CPU: the train-mode restatement (tests/resnet_train_oracle.py) against one step executed with the reference's own modules
(tests/golden/make_golden_resnet_train.py), and the trainer's gradient order.  GPU: the five training kernels against torch autograd, one step
of resnet18 / resnet50 against the restatement with CPU autograd plus descent and the eval() hand-over, and the CUDA-graph step against the
eager one."""
import configparser
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resnet_train_oracle as RT
from oracle import yolo2_oracle as O

DEV = 'cuda'
CASES = {'resnet18': (4, 128, 40, 41), 'resnet50': (2, 64, 42, 43)}     # as make_golden_resnet_train.py


def rel_err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def record(name, value):
    """Measured parity figures of this run -> $YB_PARITY_OUT/parity_resnet_train.json when that directory is given."""
    import json
    out = os.environ.get('YB_PARITY_OUT')
    if not out:
        return
    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, 'parity_resnet_train.json')
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[name] = value
    with open(path, 'w') as f:
        json.dump(data, f, indent=1, sort_keys=True)


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                      'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    return config


def make_net(name, sd=None):
    import model
    import model.resnet
    net = getattr(model.resnet, name)(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    if sd is not None:
        res = net.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net


def oracle_step(name, sd0, x, data):
    """One train-mode step of the restatement with CPU autograd: (feature, losses, {param: grad}, {bn: (mean, var)}, {bn: values per channel})."""
    anchors = O.anchors_yolo_voc()
    sd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v.clone()) for k, v in sd0.items()}
    stats, counts = {}, {}
    feature = RT.resnet_train_forward(sd, x, name, stats=stats, counts=counts)
    pred = O.decode(feature, anchors)
    pred['feature'] = feature
    losses, _ = O.loss(anchors, data, pred, 0.6)
    O.loss_total(losses).backward()
    return feature, losses, {k: v.grad for k, v in sd.items() if v.requires_grad}, stats, counts


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_resnet_train_oracle_matches_executed_reference(golden_dir):
    """The train-mode restatement (batch-statistics BatchNorm, decode, region loss, autograd) against one step executed with the reference's
    own resnet18 / resnet50 modules: loss terms, every parameter gradient (norm, first elements, small tensors in full) and the BatchNorm
    running statistics after the step (momentum 0.1, unbiased variance), to fp32 rounding."""
    g = np.load(os.path.join(golden_dir, 'resnet_train.npz'))
    for name, (b, size, seed_x, seed_t) in CASES.items():
        sd0 = O.make_resnet_state_dict(name, 0)
        s = size // 32
        x = O.synth_images(b, size, size, seed=seed_x)
        data = O.norm_data(O.synth_targets(b, size, size, slots=6, seed=seed_t), size, size, s, s)
        _, losses, grads, stats, counts = oracle_step(name, sd0, x, data)
        for k, v in losses.items():
            ref = float(g['%s_loss_%s' % (name, k)])
            assert abs(v.item() - ref) <= 1e-5 * abs(ref), (name, k, v.item(), ref)
        assert set(grads) == {k[len(name + '_gnorm_'):] for k in g.files if k.startswith(name + '_gnorm_')}, name
        for pname, gr in grads.items():
            ref_norm = float(g['%s_gnorm_%s' % (name, pname)])
            assert abs(gr.double().norm().item() - ref_norm) <= 1e-4 * ref_norm + 1e-12, (name, pname)
            head = g['%s_ghead_%s' % (name, pname)]
            np.testing.assert_allclose(gr.flatten()[:16].numpy(), head, rtol=1e-3, atol=1e-3 * float(np.abs(head).max()) + 1e-12, err_msg=pname)
            key = '%s_gfull_%s' % (name, pname)
            if key in g.files:
                assert np.linalg.norm(gr.numpy() - g[key]) <= 1e-4 * np.linalg.norm(g[key]) + 1e-12, (name, pname)
        assert len(stats) == len([k for k in g.files if k.startswith(name + '_buf_') and k.endswith('running_mean')]), name
        for prefix, (mean, var) in stats.items():
            exp_mean, exp_var = RT.expected_running(sd0, prefix, mean, var, counts[prefix])
            np.testing.assert_allclose(exp_mean.numpy(), g['%s_buf_%s.running_mean' % (name, prefix)], rtol=1e-4, atol=1e-6, err_msg=prefix)
            np.testing.assert_allclose(exp_var.numpy(), g['%s_buf_%s.running_var' % (name, prefix)], rtol=1e-4, atol=1e-6, err_msg=prefix)


@pytest.mark.parametrize('name', ['resnet18', 'resnet34', 'resnet50'])
def test_resnet_trainer_grad_order(name):
    """The trainer lists every parameter exactly once, in the order its backward produces them (the gradient arena's layout and the
    data-parallel buckets follow it).  Building the trainer needs no GPU."""
    from b200 import train_engine
    net = make_net(name)
    order = train_engine.ResNetTrainer(net).grad_order()
    assert len(order) == len(set(order))
    assert set(order) == {n for n, _ in net.named_parameters()}
    assert order[:2] == ['conv.bias', 'conv.weight'] and order[-3:] == ['bn1.weight', 'bn1.bias', 'conv1.weight']
    assert net.trainer.grad_order() == order


def test_resnet_stride2_backward_is_transpose_of_subsample():
    """What the trainer relies on, in fp64: a stride-2 "same" conv is S o (stride-1 conv) (S keeps the even pixels), so its weight and data
    gradients are the stride-1 conv's gradients of the zero-inserted dz -- for the 3x3 convs and the 1x1 downsample (input subsampled first)."""
    gen = torch.Generator().manual_seed(5)
    for k, pad in ((3, 1), (1, 0)):
        x = torch.randn(2, 8, 10, 12, generator=gen, dtype=torch.float64)
        w = torch.randn(6, 8, k, k, generator=gen, dtype=torch.float64)
        dz = torch.randn(2, 6, 5, 6, generator=gen, dtype=torch.float64)
        xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        F.conv2d(xr, wr, None, 2, pad).backward(dz)
        if k == 3:
            dzf = torch.zeros(2, 6, 10, 12, dtype=torch.float64)
            dzf[:, :, ::2, ::2] = dz
            xs, ws = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
            F.conv2d(xs, ws, None, 1, pad).backward(dzf)
            dx = xs.grad
        else:
            xsub = x[:, :, ::2, ::2].clone().requires_grad_(True)
            ws = w.clone().requires_grad_(True)
            F.conv2d(xsub, ws, None, 1, 0).backward(dz)
            dx = torch.zeros_like(x)
            dx[:, :, ::2, ::2] = xsub.grad
        assert torch.allclose(ws.grad, wr.grad, rtol=1e-12, atol=1e-12), k
        assert torch.allclose(dx, xr.grad, rtol=1e-12, atol=1e-12), k


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _nhwc16(t):
    return t.permute(0, 2, 3, 1).contiguous().half().to(DEV)


@pytest.mark.gpu
def test_resnet_training_kernels_vs_torch():
    """The five ResNet training kernels against torch on fp16-representable data: stem raw forward and weight gradient, max-pool backward
    (with deliberate ties: a tied gradient lands on the element torch's CPU kernel picks), the zero-insert (bit-exact) and the block-boundary
    gradient (one rounding, with and without mask and skip stride)."""
    from b200 import ops
    gen = torch.Generator().manual_seed(11)
    # stem: raw forward and weight gradient
    for (b, h, w) in ((2, 32, 48), (1, 64, 32)):
        x = torch.rand(b, 3, h, w, generator=gen)
        w7 = torch.randn(64, 3, 7, 7, generator=gen) * 0.1
        z = torch.empty(b, h // 2, w // 2, 64, dtype=torch.float16, device=DEV)
        ops.call('yb_stem7x7_raw_fwd', x.to(DEV), w7.to(DEV), z, b, h, w)
        assert rel_err(z.permute(0, 3, 1, 2), F.conv2d(x, w7, None, 2, 3)) <= 1e-3, (b, h, w)
        dz = torch.randn(b, 64, h // 2, w // 2, generator=gen).half().float()
        wr = w7.clone().requires_grad_(True)
        F.conv2d(x, wr, None, 2, 3).backward(dz)
        dw = torch.full((64, 3, 7, 7), 3.0, dtype=torch.float32, device=DEV)
        ops.call('yb_stem7x7_wgrad', x.to(DEV), _nhwc16(dz), dw, b, h, w)
        assert rel_err(dw, wr.grad) <= 1e-4, (b, h, w)
    # max-pool backward: a ReLU output (many exact zeros -> all-zero windows) plus repeated values
    for (b, h, w, c) in ((2, 16, 16, 64), (1, 13, 10, 16)):
        a = torch.relu(torch.randn(b, c, h, w, generator=gen)).half().float()
        a[:, :, ::3, :] = 0.5                          # ties between non-zero values too
        ar = a.clone().requires_grad_(True)
        y = F.max_pool2d(ar, 3, 2, 1)
        dy = torch.randn(y.shape, generator=gen).half().float()
        y.backward(dy)
        dx = torch.empty(b, h, w, c, dtype=torch.float16, device=DEV)
        ops.call('yb_maxpool3x3_s2_bwd_f16', _nhwc16(a), _nhwc16(dy), dx, b, h, w, c)
        got = dx.permute(0, 3, 1, 2).float().cpu()
        assert rel_err(got, ar.grad) <= 2e-3, (b, h, w, c)
        assert torch.equal(got != 0, ar.grad != 0), 'a tied gradient went to another element than torch picks'
        # also the forward of the plugin agrees with the pooled values
        yp = torch.empty(b, (h + 1) // 2, (w + 1) // 2, c, dtype=torch.float16, device=DEV)
        ops.call('yb_maxpool3x3_s2_f16', _nhwc16(a), yp, b, h, w, c)
        assert torch.equal(yp.permute(0, 3, 1, 2).float().cpu(), y.detach())
    # zero insertion: bit-exact
    for (b, h, w, c) in ((2, 14, 10, 64), (1, 7, 9, 8)):
        xs = torch.randn(b, (h + 1) // 2, (w + 1) // 2, c, generator=gen).half()
        ref = torch.zeros(b, h, w, c, dtype=torch.float16)
        ref[:, ::2, ::2] = xs
        out = torch.full((b, h, w, c), 9.0, dtype=torch.float16, device=DEV)
        ops.call('yb_upsample2_zero_f16', xs.to(DEV), out, b, h, w, c)
        assert torch.equal(out.cpu(), ref)
    # block-boundary gradient: out = (y > 0) ? g_a + S^T g_b : 0, fp32 sum rounded once
    b, h, w, c = 2, 10, 12, 32
    y = torch.relu(torch.randn(b, h, w, c, generator=gen)).half()
    ga = torch.randn(b, h, w, c, generator=gen).half()
    for stride, with_b, with_mask in ((1, True, True), (2, True, True), (1, False, True), (2, True, False), (1, True, False)):
        gb = torch.randn(b, h // stride, w // stride, c, generator=gen).half() if with_b else None
        ref = ga.float()
        if gb is not None:
            up = torch.zeros(b, h, w, c)
            up[:, ::stride, ::stride] = gb.float()
            ref = ref + up
        if with_mask:
            ref = torch.where(y.float() > 0, ref, torch.zeros(()))
        out = torch.empty(b, h, w, c, dtype=torch.float16, device=DEV)
        ops.call('yb_residual_bwd_f16', y.to(DEV) if with_mask else None, ga.to(DEV), None if gb is None else gb.to(DEV), stride, out, b, h, w, c)
        assert torch.equal(out.cpu(), ref.half()), (stride, with_b, with_mask)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['resnet18', 'resnet50'])
def test_resnet_training_step_vs_oracle_and_descent(name):
    """model.resnet in train() mode: one step (batch-statistics BatchNorm at momentum 0.1, region loss, the full backward) against the
    train-mode restatement with CPU autograd, 15 SGD steps on one batch reduce the loss, and eval() afterwards runs on the trained weights and
    running statistics (the cached folded BatchNorm and packed weights are dropped on the mode switch)."""
    import model
    import train as yb_train
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    sd0 = O.make_resnet_state_dict(name, 0)
    b, size = 8, 160
    s = size // 32
    x = O.synth_images(b, size, size, seed=90)
    tgt = O.synth_targets(b, size, size, slots=5, seed=91)
    data = O.norm_data(tgt, size, size, s, s)
    f_ref, l_ref, g_ref, stats, _ = oracle_step(name, sd0, x, data)
    net = make_net(name, sd0).to(DEV).train()
    inference = model.Inference(cfg, net, anchors).train()
    pred = model._inference(inference, x.to(DEV))
    losses, _ = model.loss(anchors, {k: v.to(DEV) for k, v in data.items()}, pred, 0.6)
    sum(losses[k] * O.HPARAM_DEFAULT[k] for k in losses).backward()
    e_f = rel_err(pred['feature'], f_ref)
    e_loss = {k: abs(losses[k].item() - l_ref[k].item()) / abs(l_ref[k].item()) for k in losses}
    last = 'layer4.%d' % (len(net.layer4) - 1)
    worst_cos, worst_rel, late_cos = (1.0, None), (0.0, None), (1.0, None)
    for pname, p in net.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), pname
        gg, r = p.grad.detach().float().cpu().flatten(), g_ref[pname].flatten()
        cos = (torch.dot(gg, r) / (gg.norm() * r.norm() + 1e-30)).item()
        rel = ((gg - r).norm() / (r.norm() + 1e-30)).item()
        if cos < worst_cos[0]:
            worst_cos = (cos, pname)
        if rel > worst_rel[0]:
            worst_rel = (rel, pname)
        if (pname.startswith('conv.') or pname.startswith(last + '.')) and cos < late_cos[0]:
            late_cos = (cos, pname)
    e_run = 0.0
    bufs = dict(net.named_buffers())
    for prefix, (mean, _) in stats.items():
        exp = (1 - RT.MOMENTUM) * sd0[prefix + '.running_mean'] + RT.MOMENTUM * mean.detach()
        e_run = max(e_run, rel_err(bufs[prefix + '.running_mean'].cpu(), exp))
    assert all(int(bufs[k]) == 1 for k in bufs if k.endswith('num_batches_tracked'))
    record('%s_train_step' % name, dict(feature=e_f, losses=e_loss, worst_grad_cosine=worst_cos, late_grad_cosine=late_cos, worst_grad_rel_l2=worst_rel,
                                        running_mean=e_run))
    assert e_f <= 0.15, e_f
    for k, v in e_loss.items():
        assert v <= 0.15, (k, v)
    # resnet50's 53 train-mode BatchNorm layers amplify the fp16 roundings: fp32 arithmetic with only the GPU path's roundings
    # (tools/resnet_train_error_budget.py resnet50 8 160) gives feature 0.120, worst cosine 0.573 and a last-block cosine of 0.877, where
    # the GPU measures 0.106 / 0.605 / 0.872; resnet18 (21 BatchNorm layers) keeps 0.986 / 0.995 in both
    assert late_cos[0] >= {'resnet18': 0.9, 'resnet50': 0.8}[name], late_cos
    assert worst_cos[0] >= 0.5, worst_cos
    assert e_run <= 1e-2, e_run
    opt = torch.optim.SGD(net.parameters(), 1e-3, momentum=0.9)
    batch = dict(tensor=x, yx_min=tgt['yx_min'], yx_max=tgt['yx_max'], cls=tgt['cls'])
    hist = [float(yb_train.iterate(inference, opt, anchors, cfg, batch)['loss_total'].item()) for _ in range(15)]
    record('%s_train_descent' % name, hist)
    assert hist[-1] < 0.9 * hist[0], hist
    # eval() on the trained state: same as the eval-mode oracle on the trained state_dict
    net.eval()
    xe = x[:2]
    f = net(xe.to(DEV))
    sd_t = {k: v.detach().float().cpu() for k, v in net.state_dict().items() if not k.endswith('num_batches_tracked')}
    with torch.no_grad():
        f_o = O.resnet_forward(sd_t, xe, name)
        f_stale = O.resnet_forward(sd0, xe, name)
    e_eval, e_stale = rel_err(f, f_o), rel_err(f_stale, f_o)
    record('%s_eval_after_training' % name, dict(vs_trained_state=e_eval, stale_state_would_be=e_stale))
    # operands cached from before training (folded running statistics, packed weights) would sit at the distance of the initial state
    # (measured 1.8 for resnet18, 11.4 for resnet50); the fp16 eval path on the trained state measured 4.2e-3 (resnet18) and 3.2e-2
    # (resnet50, whose 15 steps moved the loss from 0.32 to 0.06)
    assert e_eval <= {'resnet18': 1e-2, 'resnet50': 5e-2}[name], e_eval
    assert e_eval <= 0.2 * e_stale, (e_eval, e_stale)


@pytest.mark.gpu
def test_resnet_graphed_training_step_matches_eager():
    """train.GraphedStep on resnet18 (the whole iteration replayed as one CUDA graph) against eager train.iterate from the same state: the
    same first-step loss, and after three SGD steps the parameters moved the same way and the running statistics agree."""
    import model
    import train as yb_train
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    sd0 = O.make_resnet_state_dict('resnet18', 0)
    b, size = 4, 128
    batches = []
    for i in range(2):
        t = O.synth_targets(b, size, size, slots=6, seed=61 + i)
        batches.append(dict(tensor=O.synth_images(b, size, size, seed=71 + i).to(DEV), yx_min=t['yx_min'].to(DEV), yx_max=t['yx_max'].to(DEV),
                            cls=t['cls'].to(DEV)))

    def run(graphed):
        net = make_net('resnet18', sd0).to(DEV).train()
        inference = model.Inference(cfg, net, anchors).train()
        opt = torch.optim.SGD(net.parameters(), 1e-3, momentum=0.9)
        step = yb_train.GraphedStep(inference, opt, anchors, cfg) if graphed else (lambda d: yb_train.iterate(inference, opt, anchors, cfg, d))
        losses = [float(step(batches[i % 2])['loss_total'].item()) for i in range(3)]
        if graphed:
            assert step.launches > 0 and len(step.graphs) == 1
        return losses, {k: v.detach().float().cpu().clone() for k, v in net.state_dict().items()}

    l_e, sd_e = run(False)
    l_g, sd_g = run(True)
    record('resnet18_graphed_vs_eager_losses', dict(eager=l_e, graphed=l_g))
    assert abs(l_e[0] - l_g[0]) <= 1e-3 * abs(l_e[0]), (l_e, l_g)
    for a, g in zip(l_e, l_g):
        assert abs(a - g) <= 0.1 * abs(a), (l_e, l_g)
    for k in sd_e:
        if k.endswith('num_batches_tracked'):
            assert int(sd_e[k]) == int(sd_g[k]) == 3, k
            continue
        de, dg = (sd_e[k] - sd0[k].float()).flatten(), (sd_g[k] - sd0[k].float()).flatten()
        if 'running' in k:
            assert (sd_e[k] - sd_g[k]).norm().item() <= 0.05 * sd_e[k].norm().item() + 1e-6, k
        elif de.norm().item() > 0:
            cos = (torch.dot(de, dg) / (de.norm() * dg.norm() + 1e-30)).item()
            assert cos >= 0.8, '%s: update cosine %.3f' % (k, cos)
            assert 0.5 <= (dg.norm() / de.norm()).item() <= 2.0, k
