"""fp32 torch-functional restatement of the reference's Inception-v4 backbone (model/inception4.py: Conv2d, Mixed_3a/4a/5a, Inception_A/B/C,
Reduction_A/B, Inception4) in eval mode, and a deterministic synthetic state_dict for any channel widths (`ratio`, a pruned width table) with
BatchNorm on or off.  Pinned to the executed reference by tests/golden/inception4.npz (tests/golden/make_golden_inception4.py); the GPU tests
compare the plugin against it."""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

BN_EPS = 1e-3
STEM = (('features.0', 32, 3, 3, 2, 0, 0), ('features.1', 32, 3, 3, 1, 0, 0), ('features.2', 64, 3, 3, 1, 1, 1))
KINDS = ('Mixed_3a', 'Mixed_4a', 'Mixed_5a') + ('Inception_A',) * 4 + ('Reduction_A',) + ('Inception_B',) * 7 + ('Reduction_B',) + \
        ('Inception_C',) * 3                   # features.3 .. features.21
HEAD = 'features.22'

# per block kind: units (name, width at ratio 1, kh, kw, stride, pad_h, pad_w, source) in registration order -- source None = the block
# input, 'avg' = the block input after AvgPool2d(3, 1, 1, count_include_pad=False), else the producing unit -- and the concatenation order
# ('max' = MaxPool2d(3, stride=2) of the block input)
TABLE = {
    'Mixed_3a': ((('conv', 96, 3, 3, 2, 0, 0, None),), ('max', 'conv')),
    'Mixed_4a': ((('branch0.0', 64, 1, 1, 1, 0, 0, None), ('branch0.1', 96, 3, 3, 1, 0, 0, 'branch0.0'), ('branch1.0', 64, 1, 1, 1, 0, 0, None),
                  ('branch1.1', 64, 1, 7, 1, 0, 3, 'branch1.0'), ('branch1.2', 64, 7, 1, 1, 3, 0, 'branch1.1'),
                  ('branch1.3', 96, 3, 3, 1, 0, 0, 'branch1.2')), ('branch0.1', 'branch1.3')),
    'Mixed_5a': ((('conv', 192, 3, 3, 2, 0, 0, None),), ('conv', 'max')),
    'Inception_A': ((('branch0', 96, 1, 1, 1, 0, 0, None), ('branch1.0', 64, 1, 1, 1, 0, 0, None), ('branch1.1', 96, 3, 3, 1, 1, 1, 'branch1.0'),
                     ('branch2.0', 64, 1, 1, 1, 0, 0, None), ('branch2.1', 96, 3, 3, 1, 1, 1, 'branch2.0'),
                     ('branch2.2', 96, 3, 3, 1, 1, 1, 'branch2.1'), ('branch3.1', 96, 1, 1, 1, 0, 0, 'avg')),
                    ('branch0', 'branch1.1', 'branch2.2', 'branch3.1')),
    'Reduction_A': ((('branch0', 384, 3, 3, 2, 0, 0, None), ('branch1.0', 192, 1, 1, 1, 0, 0, None), ('branch1.1', 224, 3, 3, 1, 1, 1, 'branch1.0'),
                     ('branch1.2', 256, 3, 3, 2, 0, 0, 'branch1.1')), ('branch0', 'branch1.2', 'max')),
    'Inception_B': ((('branch0', 384, 1, 1, 1, 0, 0, None), ('branch1.0', 192, 1, 1, 1, 0, 0, None), ('branch1.1', 224, 1, 7, 1, 0, 3, 'branch1.0'),
                     ('branch1.2', 256, 7, 1, 1, 3, 0, 'branch1.1'), ('branch2.0', 192, 1, 1, 1, 0, 0, None),
                     ('branch2.1', 192, 7, 1, 1, 3, 0, 'branch2.0'), ('branch2.2', 224, 1, 7, 1, 0, 3, 'branch2.1'),
                     ('branch2.3', 224, 7, 1, 1, 3, 0, 'branch2.2'), ('branch2.4', 256, 1, 7, 1, 0, 3, 'branch2.3'),
                     ('branch3.1', 128, 1, 1, 1, 0, 0, 'avg')), ('branch0', 'branch1.2', 'branch2.4', 'branch3.1')),
    'Reduction_B': ((('branch0.0', 192, 1, 1, 1, 0, 0, None), ('branch0.1', 192, 3, 3, 2, 0, 0, 'branch0.0'), ('branch1.0', 256, 1, 1, 1, 0, 0, None),
                     ('branch1.1', 256, 1, 7, 1, 0, 3, 'branch1.0'), ('branch1.2', 320, 7, 1, 1, 3, 0, 'branch1.1'),
                     ('branch1.3', 320, 3, 3, 2, 0, 0, 'branch1.2')), ('branch0.1', 'branch1.3', 'max')),
    'Inception_C': ((('branch0', 256, 1, 1, 1, 0, 0, None), ('branch1_0', 384, 1, 1, 1, 0, 0, None), ('branch1_1a', 256, 1, 3, 1, 0, 1, 'branch1_0'),
                     ('branch1_1b', 256, 3, 1, 1, 1, 0, 'branch1_0'), ('branch2_0', 384, 1, 1, 1, 0, 0, None),
                     ('branch2_1', 448, 3, 1, 1, 1, 0, 'branch2_0'), ('branch2_2', 512, 1, 3, 1, 0, 1, 'branch2_1'),
                     ('branch2_3a', 256, 1, 3, 1, 0, 1, 'branch2_2'), ('branch2_3b', 256, 3, 1, 1, 1, 0, 'branch2_2'),
                     ('branch3.1', 256, 1, 1, 1, 0, 0, 'avg')),
                    ('branch0', 'branch1_1a', 'branch1_1b', 'branch2_3a', 'branch2_3b', 'branch3.1')),
}
# the reference builds Inception_C's branch3 conv with int(256 * ratio) filters without looking its width up in a checkpoint
FIXED = {'Inception_C': ('branch3.1',)}


def geometry():
    """key prefix -> (kh, kw, stride, pad_h, pad_w, source key or None / 'avg') of every conv unit of the backbone."""
    out = OrderedDict((k, (kh, kw, s, ph, pw, None)) for k, _, kh, kw, s, ph, pw in STEM)
    for i, kind in enumerate(KINDS):
        p = 'features.%d' % (i + 3)
        for name, _, kh, kw, s, ph, pw, src in TABLE[kind][0]:
            out['%s.%s' % (p, name)] = (kh, kw, s, ph, pw, src if src in (None, 'avg') else '%s.%s' % (p, src))
    return out


GEOM = geometry()


def widths(ratio=1, pruned=None):
    """key prefix -> output channels, as the reference's constructor resolves them: int(width * ratio) for the blocks (the stem is not scaled),
    or `pruned[key]` where a checkpoint is given (ConfigChannels(config, state_dict)); Inception_C's branch3 conv stays int(256 * ratio)."""
    out = OrderedDict()
    for k, c, *_ in STEM:
        out[k] = c
    for i, kind in enumerate(KINDS):
        for name, c, *_ in TABLE[kind][0]:
            out['features.%d.%s' % (i + 3, name)] = int(c * ratio)
    if pruned:
        for k in out:
            kind = KINDS[int(k.split('.')[1]) - 3] if int(k.split('.')[1]) >= 3 else None
            if k in pruned and k.split('.', 2)[-1] not in FIXED.get(kind, ()):
                out[k] = pruned[k]
    return out


def pruned_widths(seed=0):
    """A channel-pruned width table: every prunable unit loses 1 .. 29 filters and no width is a multiple of 8; features.0 keeps 29 filters."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for k, c in widths().items():
        w = c - 1 - int(torch.randint(0, 29, (1,), generator=g))
        out[k] = w - 3 if w % 8 == 0 else w
    out['features.0'] = 29
    return out


def in_channels(w):
    """key prefix -> input channels for the width table w, and the channel count of the head's input."""
    geom = GEOM
    cin = {}
    c = 3
    for k, *_ in STEM:
        cin[k] = c
        c = w[k]
    for i, kind in enumerate(KINDS):
        p = 'features.%d' % (i + 3)
        for name, *_, src in TABLE[kind][0]:
            key = '%s.%s' % (p, name)
            cin[key] = c if geom[key][5] in (None, 'avg') else w[geom[key][5]]
        c = sum(c if n == 'max' else w['%s.%s' % (p, n)] for n in TABLE[kind][1])
    return cin, c


def make_state_dict(seed=0, ratio=1, bn=True, pruned=None, num_anchors=5, num_cls=20):
    """He-scaled normal convs and, with BatchNorm, random non-trivial BatchNorm parameters and running statistics (without it, a random conv
    bias), so every fold of the plugin is exercised.  Keys as the module tree the reference builds (`features.6.branch3.1.conv.weight`,
    `features.19.branch2_3a.bn.running_var`, ..., `features.22.weight`, `features.22.bias`)."""
    g = torch.Generator().manual_seed(seed)
    w = widths(ratio, pruned)
    cin, c_last = in_channels(w)
    sd = OrderedDict()
    for key, (kh, kw, *_) in geometry().items():
        ci, co = cin[key], w[key]
        sd[key + '.conv.weight'] = torch.randn(co, ci, kh, kw, generator=g) * math.sqrt(2.0 / (ci * kh * kw))
        if bn:
            sd[key + '.bn.weight'] = torch.rand(co, generator=g) + 0.5
            sd[key + '.bn.bias'] = torch.randn(co, generator=g) * 0.1
            sd[key + '.bn.running_mean'] = torch.randn(co, generator=g) * 0.1
            sd[key + '.bn.running_var'] = torch.rand(co, generator=g) + 0.5
        else:
            sd[key + '.conv.bias'] = torch.randn(co, generator=g) * 0.1
    ch = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    sd[HEAD + '.weight'] = torch.randn(ch, c_last, 1, 1, generator=g) * math.sqrt(1.0 / c_last)
    sd[HEAD + '.bias'] = torch.randn(ch, generator=g) * 0.1
    return sd


def avg_pool(x):
    return F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)


def conv_unit(sd, x, key):
    """The reference's Conv2d (eval): relu(bn(conv(x))), BatchNorm eps 1e-3, or relu(conv(x) + bias) when the state_dict has no BatchNorm."""
    kh, kw, stride, ph, pw, _ = GEOM[key]
    y = F.conv2d(x, sd[key + '.conv.weight'], sd.get(key + '.conv.bias'), stride, (ph, pw))
    if key + '.bn.weight' in sd:
        y = F.batch_norm(y, sd[key + '.bn.running_mean'], sd[key + '.bn.running_var'], sd[key + '.bn.weight'], sd[key + '.bn.bias'], False, 0.0,
                         BN_EPS)
    return F.relu(y)


def block_forward(sd, x, index, units=None):
    """Block features.`index` (3 .. 21) in eval mode on x (fp32 NCHW): the concatenated output.  `units` (a dict) receives every conv unit's
    input and output under its key prefix, as (input, output)."""
    kind = KINDS[index - 3]
    p = 'features.%d' % index
    geom = GEOM
    out = {}

    def get(key):
        if key not in out:
            src = geom[key][5]
            t = x if src is None else avg_pool(x) if src == 'avg' else get(src)
            out[key] = conv_unit(sd, t, key)
            if units is not None:
                units[key] = (t, out[key])
        return out[key]
    parts = [F.max_pool2d(x, 3, 2) if n == 'max' else get('%s.%s' % (p, n)) for n in TABLE[kind][1]]
    return torch.cat(parts, 1)


def inception4_forward(sd, x, collect=None, units=None):
    """The reference's Inception4.forward (eval).  `collect` receives the stem output ('stem') and every block's output under its index;
    `units` every conv unit's (input, output) and the head's under HEAD."""
    for k, *_ in STEM:
        y = conv_unit(sd, x, k)
        if units is not None:
            units[k] = (x, y)
        x = y
    if collect is not None:
        collect['stem'] = x
    for i in range(3, 3 + len(KINDS)):
        x = block_forward(sd, x, i, units)
        if collect is not None:
            collect[i] = x
    y = F.conv2d(x, sd[HEAD + '.weight'], sd[HEAD + '.bias'])
    if units is not None:
        units[HEAD] = (x, y)
    return y
