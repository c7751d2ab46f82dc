"""Train-mode restatement of the reference's Inception-v4 backbone (model/inception4.py in train() mode): with BatchNorm every unit
normalises with the batch statistics and updates its running statistics (momentum 0.1, eps 1e-3); with `[batch_norm] enable = 0` every unit
is conv with bias -> ReLU.  One step is that forward plus CPU autograd of the synthetic loss sum(feature * R).  Pinned to the executed
reference by tests/golden/inception4_train.npz (tests/golden/make_golden_inception4_train.py); the GPU tests run it in float64 as the teacher
of the training step, block by block and whole.  The geometry and the synthetic state_dict are inception4_oracle's; the rounding model, the
loss weights and the step comparison are inception_train_oracle's."""
import torch
import torch.nn.functional as F

import inception4_oracle as I
import inception_train_oracle as T

MOMENTUM = 0.1
EXACT = T.EXACT
Rounding = T.Rounding
loss_weights = T.loss_weights
step_errors = T.step_errors


def conv_unit(p, x, key, collect=None, rnd=EXACT):
    """The reference's Conv2d in train mode: relu(batch_norm(conv(x))) with the batch statistics (p[key + '.bn.running_*'] updated in
    place), or relu(conv(x) + bias) when p has no BatchNorm for the unit.  `collect` receives (z, a) under key, z the conv output (with the
    bias when there is no BatchNorm); `rnd` adds the GPU path's fp16 roundings (inception_train_oracle.Rounding): fp16 weights except
    features.0's, fp16 z / activations, fp16 gradients at z and at the activation."""
    kh, kw, stride, ph, pw, _ = I.GEOM[key]
    w = p[key + '.conv.weight']
    w = w if key == 'features.0' else rnd.w(w)
    if key + '.bn.weight' in p:
        z = rnd.a(F.conv2d(x, w, None, stride, (ph, pw)))
        y = F.batch_norm(z, p[key + '.bn.running_mean'], p[key + '.bn.running_var'], p[key + '.bn.weight'], p[key + '.bn.bias'], True, MOMENTUM,
                         I.BN_EPS)
    else:
        z = y = rnd.g(F.conv2d(x, w, p[key + '.conv.bias'], stride, (ph, pw)))
    a = rnd.a(F.relu(y))
    if collect is not None:
        collect[key] = (z, a)
    return a


def block_forward(p, x, index, collect=None, rnd=EXACT):
    """Block features.`index` (3 .. 21) in train mode on x (NCHW): the concatenated output.  Every unit runs once (Inception_C's branch1_0
    and branch2_2 feed two convs each).  The count-exclusive pool's output is stored as fp16 and so is the gradient it hands back."""
    kind = I.KINDS[index - 3]
    pre = 'features.%d' % index
    out = {}

    def get(key):
        if key not in out:
            src = I.GEOM[key][5]
            t = x if src is None else rnd.a(I.avg_pool(rnd.g(x))) if src == 'avg' else get(src)
            out[key] = conv_unit(p, t, key, collect, rnd)
        return out[key]
    return torch.cat([F.max_pool2d(x, 3, 2) if n == 'max' else get('%s.%s' % (pre, n)) for n in I.TABLE[kind][1]], 1)


def inception4_forward(p, x, collect=None, rnd=EXACT):
    """The reference's Inception4.forward in train mode; p's running statistics are updated.  `collect` receives every unit's (z, a), the
    stem output ('stem') and every block output under its index."""
    for key, *_ in I.STEM:
        x = conv_unit(p, x, key, collect, rnd)
    if collect is not None:
        collect['stem'] = x
    for i in range(3, 3 + len(I.KINDS)):
        x = block_forward(p, x, i, collect, rnd)
        if collect is not None:
            collect[i] = x
    return rnd.g(F.conv2d(x, rnd.w(p[I.HEAD + '.weight']), p[I.HEAD + '.bias']))


def train_step(sd, x, seed=0, dtype=torch.float64, rnd=EXACT, device='cpu'):
    """One train-mode forward + backward of sum(feature * R) with autograd.  Returns (feature, loss, {parameter: gradient}, {running stat:
    value after the step}); sd is not modified."""
    p = {k: v.to(device).detach().requires_grad_(v.requires_grad) for k, v in T.params_of(sd, dtype).items()}
    f = inception4_forward(p, x.to(device, dtype), rnd=rnd)
    loss = (f * loss_weights(tuple(f.shape), seed).to(device, dtype)).sum()
    loss.backward()
    grads = {k: v.grad.detach() for k, v in p.items() if v.grad is not None}
    stats = {k: v.detach() for k, v in p.items() if 'running' in k}
    return f.detach(), loss.detach(), grads, stats
