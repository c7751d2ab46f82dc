"""fp32 torch-functional restatement of the reference's Inception-v3 backbone (model/inception3.py:29-118 over torchvision's BasicConv2d /
InceptionA-E) and a deterministic synthetic state_dict with its key names.  Pinned to the executed reference by tests/golden/inception.npz
(tests/golden/make_golden_inception.py); the GPU tests compare the plugin against it."""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

BN_EPS = 1e-3
STEM = (('Conv2d_1a_3x3', 3, 32, 3, 3, 2, 0, 0), ('Conv2d_2a_3x3', 32, 32, 3, 3, 1, 0, 0), ('Conv2d_2b_3x3', 32, 64, 3, 3, 1, 1, 1),
        ('Conv2d_3b_1x1', 64, 80, 1, 1, 1, 0, 0), ('Conv2d_4a_3x3', 80, 192, 3, 3, 1, 0, 0))
BLOCKS = (('Mixed_5b', 'A', 192, 32), ('Mixed_5c', 'A', 256, 64), ('Mixed_5d', 'A', 288, 64), ('Mixed_6a', 'B', 288, None),
          ('Mixed_6b', 'C', 768, 128), ('Mixed_6c', 'C', 768, 160), ('Mixed_6d', 'C', 768, 160), ('Mixed_6e', 'C', 768, 192),
          ('Mixed_7a', 'D', 768, None), ('Mixed_7b', 'E', 1280, None), ('Mixed_7c', 'E', 2048, None))


def block_units(kind, cin, arg):
    """torchvision's InceptionA..E: [(branch name, cin, cout, kh, kw, stride, pad_h, pad_w)] in registration order."""
    if kind == 'A':
        return [('branch1x1', cin, 64, 1, 1, 1, 0, 0), ('branch5x5_1', cin, 48, 1, 1, 1, 0, 0), ('branch5x5_2', 48, 64, 5, 5, 1, 2, 2),
                ('branch3x3dbl_1', cin, 64, 1, 1, 1, 0, 0), ('branch3x3dbl_2', 64, 96, 3, 3, 1, 1, 1), ('branch3x3dbl_3', 96, 96, 3, 3, 1, 1, 1),
                ('branch_pool', cin, arg, 1, 1, 1, 0, 0)]
    if kind == 'B':
        return [('branch3x3', cin, 384, 3, 3, 2, 0, 0), ('branch3x3dbl_1', cin, 64, 1, 1, 1, 0, 0), ('branch3x3dbl_2', 64, 96, 3, 3, 1, 1, 1),
                ('branch3x3dbl_3', 96, 96, 3, 3, 2, 0, 0)]
    if kind == 'C':
        c7 = arg
        return [('branch1x1', cin, 192, 1, 1, 1, 0, 0), ('branch7x7_1', cin, c7, 1, 1, 1, 0, 0), ('branch7x7_2', c7, c7, 1, 7, 1, 0, 3),
                ('branch7x7_3', c7, 192, 7, 1, 1, 3, 0), ('branch7x7dbl_1', cin, c7, 1, 1, 1, 0, 0), ('branch7x7dbl_2', c7, c7, 7, 1, 1, 3, 0),
                ('branch7x7dbl_3', c7, c7, 1, 7, 1, 0, 3), ('branch7x7dbl_4', c7, c7, 7, 1, 1, 3, 0), ('branch7x7dbl_5', c7, 192, 1, 7, 1, 0, 3),
                ('branch_pool', cin, 192, 1, 1, 1, 0, 0)]
    if kind == 'D':
        return [('branch3x3_1', cin, 192, 1, 1, 1, 0, 0), ('branch3x3_2', 192, 320, 3, 3, 2, 0, 0), ('branch7x7x3_1', cin, 192, 1, 1, 1, 0, 0),
                ('branch7x7x3_2', 192, 192, 1, 7, 1, 0, 3), ('branch7x7x3_3', 192, 192, 7, 1, 1, 3, 0), ('branch7x7x3_4', 192, 192, 3, 3, 2, 0, 0)]
    return [('branch1x1', cin, 320, 1, 1, 1, 0, 0), ('branch3x3_1', cin, 384, 1, 1, 1, 0, 0), ('branch3x3_2a', 384, 384, 1, 3, 1, 0, 1),
            ('branch3x3_2b', 384, 384, 3, 1, 1, 1, 0), ('branch3x3dbl_1', cin, 448, 1, 1, 1, 0, 0), ('branch3x3dbl_2', 448, 384, 3, 3, 1, 1, 1),
            ('branch3x3dbl_3a', 384, 384, 1, 3, 1, 0, 1), ('branch3x3dbl_3b', 384, 384, 3, 1, 1, 1, 0), ('branch_pool', cin, 192, 1, 1, 1, 0, 0)]


def units():
    """Every BasicConv2d of the backbone: name -> (cin, cout, kh, kw, stride, pad_h, pad_w), in the reference's registration order."""
    out = OrderedDict((u[0], u[1:]) for u in STEM)
    for name, kind, cin, arg in BLOCKS:
        for u in block_units(kind, cin, arg):
            out[name + '.' + u[0]] = u[1:]
    return out


def make_inception_state_dict(seed=0, num_anchors=5, num_cls=20):
    """He-scaled normal convs and random, non-trivial BatchNorm parameters and running statistics, so every fold of the plugin is exercised.
    Keys as the module tree the reference builds (`Mixed_5b.branch1x1.conv.weight`, `...bn.running_var`, ..., `conv.weight`, `conv.bias`)."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for key, (cin, cout, kh, kw, _, _, _) in units().items():
        sd[key + '.conv.weight'] = torch.randn(cout, cin, kh, kw, generator=g) * math.sqrt(2.0 / (cin * kh * kw))
        sd[key + '.bn.weight'] = torch.rand(cout, generator=g) + 0.5
        sd[key + '.bn.bias'] = torch.randn(cout, generator=g) * 0.1
        sd[key + '.bn.running_mean'] = torch.randn(cout, generator=g) * 0.1
        sd[key + '.bn.running_var'] = torch.rand(cout, generator=g) + 0.5
    ch = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    sd['conv.weight'] = torch.randn(ch, 2048, 1, 1, generator=g) * math.sqrt(1.0 / 2048)
    sd['conv.bias'] = torch.randn(ch, generator=g) * 0.1
    return sd


def basic_conv(sd, x, key):
    """BasicConv2d (eval): relu(bn(conv(x))), BatchNorm eps 1e-3."""
    _, _, kh, kw, stride, ph, pw = units()[key]
    y = F.conv2d(x, sd[key + '.conv.weight'], None, stride, (ph, pw))
    y = F.batch_norm(y, sd[key + '.bn.running_mean'], sd[key + '.bn.running_var'], sd[key + '.bn.weight'], sd[key + '.bn.bias'], False, 0.0, BN_EPS)
    return F.relu(y)


def block_forward(sd, x, name):
    """torchvision's InceptionA..E forward (eval) of block `name` on x (fp32 NCHW)."""
    kind = {b[0]: b[1] for b in BLOCKS}[name]

    def u(branch, t):
        return basic_conv(sd, t, name + '.' + branch)

    def pool(t):
        return F.avg_pool2d(t, 3, 1, 1)
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


def inception_forward(sd, x, collect=None):
    """model/inception3.py:73-118, eval mode, transform_input=False.  `collect` receives both stem pools ('pool1', 'pool2') and every Mixed_*
    output."""
    x = basic_conv(sd, x, 'Conv2d_1a_3x3')
    x = basic_conv(sd, x, 'Conv2d_2a_3x3')
    x = basic_conv(sd, x, 'Conv2d_2b_3x3')
    x = F.max_pool2d(x, 3, 2)
    if collect is not None:
        collect['pool1'] = x
    x = basic_conv(sd, x, 'Conv2d_3b_1x1')
    x = basic_conv(sd, x, 'Conv2d_4a_3x3')
    x = F.max_pool2d(x, 3, 2)
    if collect is not None:
        collect['pool2'] = x
    for name, _, _, _ in BLOCKS:
        x = block_forward(sd, x, name)
        if collect is not None:
            collect[name] = x
    return F.conv2d(x, sd['conv.weight'], sd['conv.bias'])
