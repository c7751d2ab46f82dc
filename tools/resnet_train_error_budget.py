"""Error budget of one ResNet TRAINING step under fp16 storage, in pure CPU fp32 arithmetic with only the roundings of the GPU path added:
conv weights -> fp16 (not the stem's, which is read as fp32), raw conv output z -> fp16, every stored activation -> fp16, and in the backward
every stored gradient -> fp16 at the trainer's static loss scale (b200.train_engine.ResNetTrainer.default_grad_scale: 16384 for resnet18 / 34
/ 50, 4096 for resnet101, 1024 for resnet152) -- through a rounding op whose backward rounds the scaled gradient.  The step
(train-mode forward, region loss, autograd backward) is compared with the exact fp32 step on the same batch as
tests/test_resnet_train.py::test_resnet_training_step_vs_oracle_and_descent: head feature, gradient cosine per parameter (worst overall and
worst of the head + last block).  If these figures match what the GPU run measures, the discrepancy is the roundings amplified by the
train-mode BatchNorm chain (DESIGN §2), not a kernel.

    python tools/resnet_train_error_budget.py resnet50 8 160     # net (resnet18 / 34 / 50 / 101 / 152), batch, size
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'yolo2-pytorch_b200')]
from oracle import yolo2_oracle as O  # noqa: E402
import resnet_deep_oracle  # noqa: E402,F401  (resnet101 / 152 in the oracle's ResNet table)

SCALE = 16384.0


class _R16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale=SCALE):
        ctx.scale = scale
        return x.half().float()

    @staticmethod
    def backward(ctx, g):
        return (g * ctx.scale).half().float() / ctx.scale, None


def grad_scale(name):
    """The static loss scale the trainer uses for this net."""
    from b200 import train_engine
    return train_engine.ResNetTrainer.default_grad_scale(len(O.resnet_blocks(name)))


def step(sd0, x, data, name, rounded, scale=SCALE):
    r = (lambda t: _R16.apply(t, scale)) if rounded else (lambda t: t)
    sd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v.clone()) for k, v in sd0.items()}

    def w(key):
        return r(sd[key]) if key != 'conv1.weight' else sd[key]

    def bn(y, prefix):
        return F.batch_norm(r(y), None, None, sd[prefix + '.weight'], sd[prefix + '.bias'], True, 0.0, 1e-5)

    h = r(F.relu(bn(F.conv2d(x, w('conv1.weight'), None, 2, 3), 'bn1')))
    h = F.max_pool2d(h, 3, 2, 1)
    for b in O.resnet_blocks(name):
        p = b['prefix']
        residual = h
        if b['kind'] == 'basic':
            out = r(F.relu(bn(F.conv2d(h, w(p + '.conv1.weight'), None, b['stride'], 1), p + '.bn1')))
            out = r(bn(F.conv2d(out, w(p + '.conv2.weight'), None, 1, 1), p + '.bn2'))
        else:
            out = r(F.relu(bn(F.conv2d(h, w(p + '.conv1.weight')), p + '.bn1')))
            out = r(F.relu(bn(F.conv2d(out, w(p + '.conv2.weight'), None, b['stride'], 1), p + '.bn2')))
            out = r(bn(F.conv2d(out, w(p + '.conv3.weight')), p + '.bn3'))
        if b['downsample']:
            residual = r(bn(F.conv2d(h, w(p + '.downsample.0.weight'), None, b['stride']), p + '.downsample.1'))
        h = r(F.relu(out + residual))
    feature = F.conv2d(h, w('conv.weight'), sd['conv.bias'])
    anchors = O.anchors_yolo_voc()
    pred = O.decode(feature, anchors)
    pred['feature'] = feature
    losses, _ = O.loss(anchors, data, pred, 0.6)
    O.loss_total(losses).backward()
    return feature.detach(), {k: v.grad for k, v in sd.items() if v.requires_grad}


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else 'resnet50'
    b = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    size = int(sys.argv[3]) if len(sys.argv) > 3 else 160
    torch.set_num_threads(8)
    sd0 = O.make_resnet_state_dict(name, 0)
    s = size // 32
    x = O.synth_images(b, size, size, seed=90)
    data = O.norm_data(O.synth_targets(b, size, size, slots=5, seed=91), size, size, s, s)
    f_ref, g_ref = step(sd0, x, data, name, False)
    f_16, g_16 = step(sd0, x, data, name, True, grad_scale(name))
    last = [blk['prefix'] for blk in O.resnet_blocks(name)][-1]
    worst, late = (1.0, None), (1.0, None)
    for k, g in g_ref.items():
        a, c = g_16[k].flatten(), g.flatten()
        cos = (torch.dot(a, c) / (a.norm() * c.norm() + 1e-30)).item()
        worst = min(worst, (cos, k))
        if k.startswith('conv.') or k.startswith(last + '.'):
            late = min(late, (cos, k))
    print('%s B=%d %d^2, fp32 + fp16 roundings vs fp32: feature rel %.3e, worst gradient cosine %.3f (%s), head + %s worst %.3f (%s)'
          % (name, b, size, ((f_16 - f_ref).abs().max() / f_ref.abs().max()).item(), worst[0], worst[1], last, late[0], late[1]))


if __name__ == '__main__':
    main()
