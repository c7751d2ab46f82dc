"""Train-mode restatement of the reference's Inception-v3 backbone (model/inception3.py:29-118 over torchvision's BasicConv2d / InceptionA-E
in train() mode): every BatchNorm normalises with the batch statistics and updates its running statistics (momentum 0.1, eps 1e-3).
One step is that forward plus CPU autograd of the synthetic loss sum(feature * R).  Pinned to the executed reference by
tests/golden/inception_train.npz (tests/golden/make_golden_inception_train.py); the GPU tests run it in float64 as the teacher of the
training step, block by block and whole."""
import torch
import torch.nn.functional as F

import inception_oracle as I

MOMENTUM = 0.1


class _Exact(object):
    """No rounding: the restatement itself."""
    def a(self, t):
        return t

    def w(self, t):
        return t

    def g(self, t):
        return t


class _Store16(torch.autograd.Function):
    """fp16 storage of a tensor, and of the loss-scaled gradient that reaches it."""
    @staticmethod
    def forward(ctx, x, scale):
        ctx.scale = scale
        return x.half().to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return (g * ctx.scale).half().to(g.dtype) / ctx.scale, None


class _Grad16(torch.autograd.Function):
    """The loss-scaled gradient stored in fp16; the value passes unchanged."""
    @staticmethod
    def forward(ctx, x, scale):
        ctx.scale = scale
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return (g * ctx.scale).half().to(g.dtype) / ctx.scale, None


class Rounding(object):
    """The fp16 roundings of the GPU training path (b200.train_engine.InceptionTrainer) and nothing else: conv weights read as fp16 (not
    the stem conv's, read as fp32), every raw conv output z, activation and average-pooled tensor stored as fp16, and every stored gradient
    (at z, at an activation, at the head's output) fp16 at the static loss scale.  For tools/inception_train_error_budget.py and the
    whole-step test: what those roundings alone do to the step."""
    def __init__(self, scale):
        self.scale = float(scale)

    def a(self, t):
        return _Store16.apply(t, self.scale)

    def w(self, t):
        return t.detach().half().to(t.dtype) + (t - t.detach())     # value rounded, gradient straight through (fp32 weight gradients)

    def g(self, t):
        return _Grad16.apply(t, self.scale)


EXACT = _Exact()


def basic_conv(p, x, key, collect=None, rnd=EXACT):
    """BasicConv2d in train mode: relu(batch_norm(conv(x))) with the batch statistics; p[key + '.bn.running_*'] are updated in place.
    `collect` receives z (the conv output) and a (the activation) under key; `rnd` adds the GPU path's fp16 roundings (Rounding)."""
    _, _, kh, kw, stride, ph, pw = I.units()[key]
    w = p[key + '.conv.weight']
    z = rnd.a(F.conv2d(x, w if key == 'Conv2d_1a_3x3' else rnd.w(w), None, stride, (ph, pw)))
    y = F.batch_norm(z, p[key + '.bn.running_mean'], p[key + '.bn.running_var'], p[key + '.bn.weight'], p[key + '.bn.bias'], True, MOMENTUM,
                     I.BN_EPS)
    a = rnd.a(F.relu(y))
    if collect is not None:
        collect[key] = (z, a)
    return a


def block_forward(p, x, name, collect=None, rnd=EXACT):
    """torchvision's InceptionA..E forward of block `name` in train mode (x fp NCHW)."""
    kind = {b[0]: b[1] for b in I.BLOCKS}[name]

    def u(branch, t):
        return basic_conv(p, t, name + '.' + branch, collect, rnd)

    def pool(t):
        return rnd.a(F.avg_pool2d(t, 3, 1, 1))
    if kind == 'A':
        outs = [u('branch1x1', x), u('branch5x5_2', u('branch5x5_1', x)), u('branch3x3dbl_3', u('branch3x3dbl_2', u('branch3x3dbl_1', x))),
                u('branch_pool', pool(x))]
    elif kind == 'B':
        outs = [u('branch3x3', x), u('branch3x3dbl_3', u('branch3x3dbl_2', u('branch3x3dbl_1', x))), F.max_pool2d(x, 3, 2)]
    elif kind == 'C':
        d = u('branch7x7dbl_1', x)
        for b in ('branch7x7dbl_2', 'branch7x7dbl_3', 'branch7x7dbl_4', 'branch7x7dbl_5'):
            d = u(b, d)
        outs = [u('branch1x1', x), u('branch7x7_3', u('branch7x7_2', u('branch7x7_1', x))), d, u('branch_pool', pool(x))]
    elif kind == 'D':
        d = u('branch7x7x3_1', x)
        for b in ('branch7x7x3_2', 'branch7x7x3_3', 'branch7x7x3_4'):
            d = u(b, d)
        outs = [u('branch3x3_2', u('branch3x3_1', x)), d, F.max_pool2d(x, 3, 2)]
    else:
        a = u('branch3x3_1', x)
        d = u('branch3x3dbl_2', u('branch3x3dbl_1', x))
        outs = [u('branch1x1', x), u('branch3x3_2a', a), u('branch3x3_2b', a), u('branch3x3dbl_3a', d), u('branch3x3dbl_3b', d),
                u('branch_pool', pool(x))]
    return torch.cat(outs, 1)


def stem_forward(p, x, collect=None, rnd=EXACT):
    """Conv2d_1a_3x3 .. the second max-pool in train mode: Mixed_5b's input."""
    for key in ('Conv2d_1a_3x3', 'Conv2d_2a_3x3', 'Conv2d_2b_3x3'):
        x = basic_conv(p, x, key, collect, rnd)
    x = F.max_pool2d(x, 3, 2)
    for key in ('Conv2d_3b_1x1', 'Conv2d_4a_3x3'):
        x = basic_conv(p, x, key, collect, rnd)
    return F.max_pool2d(x, 3, 2)


def inception_forward(p, x, collect=None, rnd=EXACT):
    """model/inception3.py:73-118 in train mode (transform_input=False); p's running statistics are updated."""
    x = stem_forward(p, x, collect, rnd)
    for name, _, _, _ in I.BLOCKS:
        x = block_forward(p, x, name, collect, rnd)
        if collect is not None:
            collect[name] = x
    return rnd.g(F.conv2d(x, rnd.w(p['conv.weight']), p['conv.bias']))


def loss_weights(shape, seed=0):
    """The fixed weights R of the synthetic training loss sum(feature * R) (a smooth stand-in for the region loss: every head output gets a
    non-zero gradient)."""
    g = torch.Generator().manual_seed(700 + seed)
    return torch.randn(*shape, generator=g) / float(torch.tensor(shape).prod()) ** 0.5


def params_of(sd, dtype):
    """Leaf copies of a state_dict in `dtype`: parameters require grad, running statistics do not."""
    p = {k: v.detach().to(dtype).clone() for k, v in sd.items() if not k.endswith('num_batches_tracked')}
    for k, v in p.items():
        v.requires_grad_('running' not in k)
    return p


def train_step(sd, x, seed=0, dtype=torch.float64, rnd=EXACT, device='cpu'):
    """One train-mode forward + backward of sum(feature * R) with autograd.  Returns (feature, loss, {parameter: gradient}, {running stat:
    value after the step}); sd is not modified."""
    p = {k: v.to(device).detach().requires_grad_(v.requires_grad) for k, v in params_of(sd, dtype).items()}
    f = inception_forward(p, x.to(device, dtype), rnd=rnd)
    loss = (f * loss_weights(tuple(f.shape), seed).to(device, dtype)).sum()
    loss.backward()
    grads = {k: v.grad.detach() for k, v in p.items() if v.grad is not None}
    stats = {k: v.detach() for k, v in p.items() if 'running' in k}
    return f.detach(), loss.detach(), grads, stats


def step_errors(f, grads, stats, f_ref, g_ref, s_ref, names):
    """How far a step (f, grads, stats) is from the reference step: feature relative L2, the median and the worst gradient relative L2 and
    cosine over the parameters `names`, and the worst running statistic (relative L2)."""
    def rel(a, b):
        a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
        return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()

    def cos(a, b):
        a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
        return (torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-300)).item()
    errs = sorted(rel(grads[n], g_ref[n]) for n in names)
    coss = sorted(cos(grads[n], g_ref[n]) for n in names)
    return dict(feature=rel(f, f_ref), grad_rel_l2=[errs[len(errs) // 2], errs[-1]], grad_cosine=[coss[len(coss) // 2], coss[0]],
                running=max(rel(stats[k], s_ref[k]) for k in s_ref))
