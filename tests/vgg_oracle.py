"""torch-functional restatement of the reference's VGG backbone (model/vgg.py: make_layers, VGG.forward) in eval mode, and deterministic
synthetic state dicts for the eight constructors with any channel widths.  Pinned to the executed reference by tests/golden/vgg.npz
(tests/golden/make_golden_vgg.py); the GPU tests compare the plugin against it, in eval and train mode (train_step: CPU autograd of one
step).  Runs in the dtype of its inputs (fp32 or fp64)."""
from collections import OrderedDict

import torch
import torch.nn.functional as F

BN_EPS = 1e-5
CFGS = {
    'A': [64, 'M', 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'B': [64, 64, 'M', 128, 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'D': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M'],
    'E': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512, 'M'],
}
NAMES = ('vgg11', 'vgg11_bn', 'vgg13', 'vgg13_bn', 'vgg16', 'vgg16_bn', 'vgg19', 'vgg19_bn')
ARCH = {'vgg11': 'A', 'vgg13': 'B', 'vgg16': 'D', 'vgg19': 'E'}


def layers(name, pruned=None):
    """[(kind, feature index, width)] of `features` as make_layers builds it: kind 'conv' (width = its filters, `pruned['features.i.weight']`
    when given), 'bn', 'relu' or 'pool'."""
    bn = name.endswith('_bn')
    out = []
    for v in CFGS[ARCH[name[:5]]]:
        i = len(out)
        if v == 'M':
            out.append(('pool', i, None))
            continue
        key = 'features.%d.weight' % i
        c = pruned[key] if pruned and key in pruned else v
        out.append(('conv', i, c))
        if bn:
            out.append(('bn', i + 1, c))
        out.append(('relu', len(out), c))
    return out


def pruned_widths():
    """A channel-pruned vgg11_bn checkpoint's widths: none a multiple of 32, features.0 below 64."""
    return {'features.0.weight': 48, 'features.4.weight': 80, 'features.8.weight': 200, 'features.11.weight': 136, 'features.15.weight': 300,
            'features.18.weight': 260, 'features.22.weight': 100, 'features.25.weight': 72}


def make_state_dict(name, seed=0, pruned=None, num_anchors=5, num_cls=20):
    """Deterministic parameters (and BatchNorm running statistics) with the reference's keys, in its order.  Conv weights are He-scaled
    (variance 2 / fan_in) so activations stay O(1) through 16 ReLU convs; biases, BatchNorm affine parameters and running statistics are
    non-trivial."""
    g = torch.Generator().manual_seed(1000 + seed)
    sd = OrderedDict()
    cin = 3
    for kind, i, c in layers(name, pruned):
        if kind == 'conv':
            sd['features.%d.weight' % i] = torch.randn(c, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
            sd['features.%d.bias' % i] = torch.randn(c, generator=g) * 0.05
            cin = c
        elif kind == 'bn':
            p = 'features.%d.' % i
            sd[p + 'weight'] = 1 + 0.2 * (torch.rand(c, generator=g) - 0.5)
            sd[p + 'bias'] = 0.1 * torch.randn(c, generator=g)
            sd[p + 'running_mean'] = 0.1 * torch.randn(c, generator=g)
            sd[p + 'running_var'] = 0.5 + torch.rand(c, generator=g)
    cout = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    sd['conv.weight'] = torch.randn(cout, cin, 1, 1, generator=g) * (1.0 / cin) ** 0.5
    sd['conv.bias'] = torch.randn(cout, generator=g) * 0.1
    return sd


def vgg_forward(sd, x, name, pruned=None, collect=None, train=False):
    """conv(features(x)); `collect` receives each MaxPool2d's output under its feature index.  `train`: BatchNorm on batch statistics,
    updating sd's running_mean / running_var in place (momentum 0.1), as nn.BatchNorm2d in train() mode; parameters keep their autograd
    identity, so sd may hold leaf tensors that require gradients."""
    dt = x.dtype
    p = {k: (v if v.dtype == dt else v.to(dt)) for k, v in sd.items()}
    for kind, i, _ in layers(name, pruned):
        if kind == 'conv':
            x = F.conv2d(x, p['features.%d.weight' % i], p['features.%d.bias' % i], padding=1)
        elif kind == 'bn':
            k = 'features.%d.' % i
            x = F.batch_norm(x, sd[k + 'running_mean'] if train else p[k + 'running_mean'], sd[k + 'running_var'] if train else p[k + 'running_var'],
                             p[k + 'weight'], p[k + 'bias'], train, 0.1, BN_EPS)
        elif kind == 'relu':
            x = F.relu(x)
        else:
            x = F.max_pool2d(x, 2, 2)
            if collect is not None:
                collect[i] = x
    return F.conv2d(x, p['conv.weight'], p['conv.bias'])


def loss_weights(shape, seed=0):
    """The fixed weights R of the synthetic training loss sum(feature * R) (a smooth stand-in for the region loss: every head output gets a
    non-zero gradient)."""
    g = torch.Generator().manual_seed(500 + seed)
    return torch.randn(*shape, generator=g) / float(torch.tensor(shape).prod()) ** 0.5


def train_step(sd, x, name, seed=0, dtype=torch.float64):
    """One train-mode forward + backward of sum(feature * R) with CPU autograd.  Returns (loss, {parameter: gradient}, {running stat: value
    after the step}); sd is not modified."""
    params = {k: v.detach().to(dtype).clone() for k, v in sd.items()}
    for k, v in params.items():
        v.requires_grad_('running' not in k)
    f = vgg_forward(params, x.to(dtype), name, train=True)
    loss = (f * loss_weights(tuple(f.shape), seed).to(dtype)).sum()
    loss.backward()
    grads = {k: v.grad.detach() for k, v in params.items() if v.grad is not None}
    stats = {k: v.detach() for k, v in params.items() if 'running' in k}
    return loss.detach(), grads, stats
