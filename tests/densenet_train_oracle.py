"""fp64 restatement of one train-mode step of the reference's DenseNet backbone (model/densenet.py over torchvision's _DenseLayer /
_Transition, drop_rate 0): batch-statistics BatchNorm with the running-statistics update, the loss sum(feature * R) and torch autograd for
every parameter gradient.  Pinned to the executed reference by tests/golden/densenet_train.npz (tests/golden/make_golden_densenet_train.py);
it is the teacher of tests/test_densenet_train.py.

`rnd` (inception_train_oracle.Rounding) adds the fp16 roundings of the GPU path (b200.train_engine.DenseNetTrainer) and nothing else: conv
weights read as fp16 (not conv0's, read as fp32); stored as fp16 with their loss-scaled gradients: the stem's z and activation, every
pre-activation a = act(norm(x)) the 1x1 convs read, conv1's z1, a2 = relu(norm2(z1)), every conv2 and transition-conv output (the block
buffers; the gradient of each 32-channel slice is rounded once, when it is final), the transition's pooled activation; the head's output
gradient.  With roundings the transition pools before its conv, as the GPU path does (equal in exact arithmetic)."""
import torch
import torch.nn.functional as F

import densenet_oracle as D
from inception_train_oracle import EXACT, Rounding, loss_weights, step_errors  # noqa: F401  (re-exported for the tests and tools)

MOMENTUM, EPS = 0.1, 1e-5


def _bn(p, run, x, key):
    return F.batch_norm(x, run[key + '.running_mean'], run[key + '.running_var'], p[key + '.weight'], p[key + '.bias'], True, MOMENTUM, EPS)


def stem(p, run, x, rnd=EXACT):
    z = rnd.a(F.conv2d(x, p['features.conv0.weight'], None, 2, 3))
    return rnd.a(F.max_pool2d(rnd.a(F.relu(_bn(p, run, z, 'features.norm0'))), 3, 2, 1))


def dense_layer(p, run, x, key, rnd=EXACT):
    """One _DenseLayer on the concatenation x: its 32 new channels."""
    a1 = rnd.a(F.relu(_bn(p, run, x, key + '.norm1')))
    z1 = rnd.a(F.conv2d(a1, rnd.w(p[key + '.conv1.weight'])))
    a2 = rnd.a(F.relu(_bn(p, run, z1, key + '.norm2')))
    return rnd.a(F.conv2d(a2, rnd.w(p[key + '.conv2.weight']), None, 1, 1))


def transition(p, run, x, t, rnd=EXACT):
    a = F.relu(_bn(p, run, x, t + '.norm'))
    if rnd is EXACT:
        return F.avg_pool2d(F.conv2d(a, p[t + '.conv.weight']), 2, 2)
    return rnd.a(F.conv2d(rnd.a(F.avg_pool2d(a, 2, 2)), rnd.w(p[t + '.conv.weight'])))


def head(p, run, x, rnd=EXACT):
    a5 = rnd.a(_bn(p, run, x, 'features.norm5'))
    return rnd.g(F.conv2d(a5, rnd.w(p['features.conv.weight']), p['features.conv.bias']))


def forward(p, run, x, name='densenet121', collect=None, rnd=EXACT):
    """Train-mode forward on leaves `p` (parameters) and `run` (running statistics, updated in place)."""
    _, config, _ = D.CONFIGS[name]
    x = stem(p, run, x, rnd)
    bl, _ = D.blocks(name)
    for bi, n, _ in bl:
        feats = [x]
        for j in range(n):
            feats.append(dense_layer(p, run, torch.cat(feats, 1), 'features.denseblock%d.denselayer%d' % (bi, j + 1), rnd))
        x = torch.cat(feats, 1)
        if collect is not None:
            collect['denseblock%d' % bi] = x
        if bi < len(config):
            x = transition(p, run, x, 'features.transition%d' % bi, rnd)
    return head(p, run, x, rnd)


def step(sd, x, r=None, name='densenet121', rnd=EXACT, device='cpu', dtype=torch.float64):
    """One step from the state_dict `sd` on images x with the loss sum(feature * r) (default: loss_weights of the feature's shape).  Returns
    (loss, feature, {parameter: gradient}, {running-statistic key: value after the step})."""
    p = {k: v.to(device, dtype).clone().requires_grad_(True) for k, v in sd.items()
         if not k.endswith(('running_mean', 'running_var', 'num_batches_tracked'))}
    run = {k: v.to(device, dtype).clone() for k, v in sd.items() if k.endswith(('running_mean', 'running_var'))}
    feature = forward(p, run, x.to(device, dtype), name, rnd=rnd)
    if r is None:
        r = loss_weights(tuple(feature.shape))
    loss = (feature * r.to(device, dtype)).sum()
    loss.backward()
    return loss.detach(), feature.detach(), {k: v.grad for k, v in p.items()}, run
