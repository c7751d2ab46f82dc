"""VGG training step (model.vgg in train() mode over b200.train_engine.VGGTrainer).

CPU: the train-mode restatement (vgg_oracle.train_step, CPU autograd) against one step of the executed reference (vgg.npz: loss, every
gradient's norm and first elements, running statistics); grad_order() lists every parameter once.

GPU: the first layer's weight gradient (yb_conv0_c64_wgrad) against fp64; the has_bn = 0 ReLU (+ 2x2 max-pool) backward of the plain units
against torch autograd; one step of vgg11, vgg11_bn and vgg16_bn against the restatement (loss, every gradient, running statistics); loss
descent over a few SGD steps and eval() inference on the trained state; the GraphedStep step against the eager step."""
import configparser
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgg_oracle as V
from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu
MEASURED = {}


def record(name, value):
    """Measured figures of this run -> $YB_PARITY_OUT/vgg_train_measured.json when that directory is given."""
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'vgg_train_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                      'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    return config


def make_net(name, sd):
    import model
    import model.vgg
    net = getattr(model.vgg, name)(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    return net


TRAIN = (2, 64, 96, 9)      # the golden's train step: batch, H, W, image seed (state dict seed 4)


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_train_restatement_vs_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'vgg.npz'))
    b, h, w, seed = TRAIN
    x = O.synth_images(b, h, w, seed=seed)
    for name in ('vgg11', 'vgg11_bn'):
        sd = V.make_state_dict(name, seed=4)
        loss, grads, stats = V.train_step(sd, x, name, dtype=torch.float32)
        assert abs(loss.item() - float(g['train_%s_loss' % name])) <= 1e-5 * abs(loss.item()), name
        assert set(grads) == {k for k in sd if 'running' not in k}
        for k, gr in grads.items():
            ref_norm = float(g['train_%s_gnorm_%s' % (name, k)])
            if ref_norm < 1e-6:                        # conv biases before a BatchNorm: zero up to rounding
                assert gr.norm().item() < 1e-5, (name, k)
                continue
            assert abs(gr.norm().item() / ref_norm - 1) < 1e-4, (name, k)
            head = torch.from_numpy(g['train_%s_ghead_%s' % (name, k)])
            assert (gr.flatten()[:16] - head).abs().max().item() <= 1e-4 * gr.abs().max().item(), (name, k)
        for k, v in stats.items():
            ref = torch.from_numpy(g['train_%s_%s' % (name, k)])
            assert (v - ref).abs().max().item() <= 1e-5 * max(ref.abs().max().item(), 1.0), (name, k)


@pytest.mark.parametrize('name', V.NAMES)
def test_grad_order_lists_every_parameter_once(name):
    import model
    import model.vgg
    net = getattr(model.vgg, name)(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    order = net.trainer.grad_order()
    assert len(order) == len(set(order)) and set(order) == {n for n, _ in net.named_parameters()}
    assert order[:2] == ['conv.bias', 'conv.weight'] and order[-1] == 'features.0.weight'


def test_training_width_errors():
    import model
    import model.vgg
    net = model.vgg.vgg11(model.ConfigChannels(make_config(), V.make_state_dict('vgg11', pruned={'features.3.weight': 80})),
                          O.anchors_yolo_voc(), 20)
    with pytest.raises(ValueError, match='multiples of 32'):
        net.trainer._check()
    net = model.vgg.vgg11(model.ConfigChannels(make_config(), V.make_state_dict('vgg11', pruned={'features.0.weight': 32})),
                          O.anchors_yolo_voc(), 20)
    with pytest.raises(ValueError, match='64 filters'):
        net.trainer._check()
    with pytest.raises(RuntimeError):
        net.train()(torch.zeros(1, 3, 64, 64))           # CPU tensor: no CPU fallback


# ------------------------------------------------------------------------------------------------
# GPU: kernels
# ------------------------------------------------------------------------------------------------
@gpu
def test_first_layer_weight_gradient_vs_fp64():
    from b200 import ops
    g = torch.Generator().manual_seed(21)
    rec = {}
    for b, h, w in ((1, 8, 32), (2, 64, 96), (3, 96, 160), (8, 416, 416)):
        x = torch.rand(b, 3, h, w, generator=g) * 2 - 0.5
        dz = (torch.randn(b, h, w, 64, generator=g) * 4).half()
        dw = torch.empty(64, 3, 3, 3, device=DEV)
        ops.call('yb_conv0_c64_wgrad', x.to(DEV), dz.to(DEV), dw, b, h, w)
        ref = torch.nn.grad.conv2d_weight(x.double(), (64, 3, 3, 3), dz.double().permute(0, 3, 1, 2), padding=1)
        rec['%dx%dx%d' % (b, h, w)] = rel_err(dw, ref)
    record('first_layer_wgrad', rec)
    # fp32 products of exact operands, fp32 sums over up to 1.4 M pixels per filter tap; measured <= 9.5e-7, bound twice that
    assert all(v <= 2e-6 for v in rec.values()), rec


@gpu
@pytest.mark.parametrize('pool', [False, True])
def test_plain_unit_relu_pool_backward_vs_autograd(pool):
    """yb_bn_act_bwd with has_bn = 0 and slope 0 on a stored ReLU output a (and a 2x2 max-pool after it): dz = dL/d(conv output) and the
    reduce pass's per-channel sum = the bias gradient, against torch autograd of relu (+ max_pool2d) from the same pre-activation."""
    from b200 import ops
    g = torch.Generator().manual_seed(22 + pool)
    b, h, w, c = 2, 16, 24, 64
    zpre = (torch.randn(b, c, h, w, generator=g)).half().double().requires_grad_()
    out = F.relu(zpre)
    if pool:
        out = F.max_pool2d(out, 2, 2)
    gout = torch.randn(out.shape, generator=g).half().double()
    out.backward(gout)
    a = F.relu(zpre.detach()).permute(0, 2, 3, 1).contiguous().half().to(DEV)
    gd = gout.permute(0, 2, 3, 1).contiguous().half().to(DEV)
    da, dap = (None, gd) if pool else (gd, None)
    sums = torch.zeros(2 * c, dtype=torch.float64, device=DEV)
    dz = torch.empty(b, h, w, c, dtype=torch.float16, device=DEV)
    args = (a, c, None, None, None, None, 0.0, da, 0 if da is None else c, 0, dap, 0 if dap is None else c, 0, b, h, w, c, int(pool), sums)
    ops.call('yb_bn_act_bwd', 0, *args, None, 0, 0)
    ops.call('yb_bn_act_bwd', 1, *args, dz, c, 0)
    ref = zpre.grad.permute(0, 2, 3, 1)
    assert torch.equal(dz.double().cpu(), ref), float((dz.double().cpu() - ref).abs().max())     # a product with 1 or 0: exact
    # per-block fp32 partial sums of fp16 values, added in double
    assert torch.allclose(sums[:c].cpu(), ref.sum((0, 1, 2)), rtol=1e-5, atol=1e-4)


# ------------------------------------------------------------------------------------------------
# GPU: training step
# ------------------------------------------------------------------------------------------------
# fp16 activations and gradients against an fp64 CPU step: gradients compared by relative L2 error and cosine, as the ResNet step test does.
# Measured on an H100 80GB HBM3 (700 W), worst of vgg11 / vgg11_bn / vgg16_bn: feature 1.14e-2, running statistics 4.4e-4, gradient
# relative L2 0.265 and cosine 0.966 (vgg16_bn, the BatchNorm biases of the first blocks); the bounds are twice those deviations
TOL_STEP = dict(feature=2.5e-2, running=1e-3, grad_rel_l2=0.55, grad_cosine=0.93)


@gpu
@pytest.mark.parametrize('name', ['vgg11', 'vgg11_bn', 'vgg16_bn'])
def test_training_step_vs_oracle(name):
    b, h, w = 4, 128, 160
    sd = V.make_state_dict(name, seed=5)
    x = O.synth_images(b, h, w, seed=10)
    params = {k: v.double().clone().requires_grad_('running' not in k) for k, v in sd.items()}
    f_ref = V.vgg_forward(params, x.double(), name, train=True)
    (f_ref * V.loss_weights(tuple(f_ref.shape)).double()).sum().backward()
    net = make_net(name, sd).to(DEV).train()
    f = net(x.to(DEV))
    (f * V.loss_weights(tuple(f.shape)).to(DEV)).sum().backward()
    torch.cuda.synchronize()
    gmax = max(p.grad.abs().max().item() for p in params.values() if p.grad is not None)
    rec = dict(feature=rel_err(f, f_ref), running=0.0, grad_rel_l2=(0.0, None), grad_cosine=(1.0, None))
    for k, p in net.named_parameters():
        r = params[k].grad.flatten()
        gg = p.grad.double().cpu().flatten()
        if name.endswith('_bn') and k.startswith('features.') and k.endswith('.bias') and k.replace('.bias', '.weight') in sd and \
                sd[k.replace('.bias', '.weight')].dim() == 4:
            assert r.abs().max().item() < 1e-9 * gmax and bool((gg == 0).all()), k     # conv bias before a BatchNorm: exactly zero
            continue
        rel = ((gg - r).norm() / (r.norm() + 1e-30)).item()
        cos = (torch.dot(gg, r) / (gg.norm() * r.norm() + 1e-30)).item()
        if rel > rec['grad_rel_l2'][0]:
            rec['grad_rel_l2'] = (rel, k)
        if cos < rec['grad_cosine'][0]:
            rec['grad_cosine'] = (cos, k)
    for k, v in net.state_dict().items():
        if 'running' in k:
            rec['running'] = max(rec['running'], rel_err(v, params[k]))
        if k.endswith('num_batches_tracked'):
            assert int(v) == 1, k
    record('step_' + name, rec)
    assert rec['feature'] <= TOL_STEP['feature'] and rec['running'] <= TOL_STEP['running'], rec
    assert rec['grad_rel_l2'][0] <= TOL_STEP['grad_rel_l2'] and rec['grad_cosine'][0] >= TOL_STEP['grad_cosine'], rec


@gpu
@pytest.mark.parametrize('name', ['vgg11', 'vgg16_bn'])
def test_loss_descent_and_eval_after_training(name):
    sd = V.make_state_dict(name, seed=6)
    net = make_net(name, sd).to(DEV).train()
    x = O.synth_images(4, 96, 128, seed=11).to(DEV)
    target = V.loss_weights((4, 125, 3, 4), seed=1).to(DEV) * 30
    opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9)
    losses = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        loss = ((net(x) - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    record('descent_' + name, losses)
    assert all(np.isfinite(losses)) and losses[-1] < 0.9 * losses[0], losses
    net.eval()
    with torch.no_grad():
        y = net(x)
    trained = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    ref = V.vgg_forward(trained, x.cpu(), name)
    e = rel_err(y, ref)
    record('eval_after_train_' + name, e)
    assert e <= 5e-3, e          # measured 1.8e-3 (vgg11) and 2.5e-3 (vgg16_bn); the inference bound of test_vgg.py


@gpu
def test_graphed_training_step_matches_eager():
    """train.GraphedStep on vgg11_bn against eager train.iterate from the same state: the same first-step loss, and after three SGD steps
    the parameters moved the same way and the running statistics agree."""
    import model
    import train as yb_train
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    sd0 = V.make_state_dict('vgg11_bn', 7)
    b, size = 4, 128
    batches = []
    for i in range(2):
        t = O.synth_targets(b, size, size, slots=6, seed=61 + i)
        batches.append(dict(tensor=O.synth_images(b, size, size, seed=71 + i).to(DEV), yx_min=t['yx_min'].to(DEV), yx_max=t['yx_max'].to(DEV),
                            cls=t['cls'].to(DEV)))

    def run(graphed):
        net = make_net('vgg11_bn', sd0).to(DEV).train()
        inference = model.Inference(cfg, net, anchors).train()
        opt = torch.optim.SGD(net.parameters(), 1e-3, momentum=0.9)
        step = yb_train.GraphedStep(inference, opt, anchors, cfg) if graphed else (lambda d: yb_train.iterate(inference, opt, anchors, cfg, d))
        losses = [float(step(batches[i % 2])['loss_total'].item()) for i in range(3)]
        if graphed:
            assert step.launches > 0 and len(step.graphs) == 1
        return losses, {k: v.detach().float().cpu().clone() for k, v in net.state_dict().items()}

    l_e, sd_e = run(False)
    l_g, sd_g = run(True)
    record('graphed_vs_eager_losses', dict(eager=l_e, graphed=l_g))
    assert abs(l_e[0] - l_g[0]) <= 1e-3 * abs(l_e[0]), (l_e, l_g)
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
