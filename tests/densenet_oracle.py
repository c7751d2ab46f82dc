"""fp32 torch-functional restatement of the reference's DenseNet backbone (model/densenet.py:29-65 over torchvision's _DenseLayer /
_Transition) and a deterministic synthetic state_dict with its key names.  Pinned to the executed reference by tests/golden/densenet.npz
(tests/golden/make_golden_densenet.py); the GPU tests compare the plugin against it."""
import math

import torch
import torch.nn.functional as F

CONFIGS = {
    # name: (growth_rate, block_config, num_init_features), model/densenet.py:68-117
    'densenet121': (32, (6, 12, 24, 16), 64),
    'densenet169': (32, (6, 12, 32, 32), 64),
    'densenet201': (32, (6, 12, 48, 32), 64),
    'densenet161': (48, (6, 12, 36, 24), 96),
}
BN_SIZE = 4


def blocks(name):
    """[(block index, number of layers, input channels)] and the final channel count."""
    growth, config, c = CONFIGS[name]
    out = []
    for i, n in enumerate(config):
        out.append((i + 1, n, c))
        c += n * growth
        if i + 1 < len(config):
            c //= 2
    return out, c


def make_densenet_state_dict(name='densenet121', seed=0, num_anchors=5, num_cls=20):
    """Kaiming-normal convs (model/densenet.py:57-59) and random, non-trivial BatchNorm parameters and running statistics, so every fold of
    the plugin is exercised.  Keys as the module tree the reference builds (`features.denseblock1.denselayer1.norm1.weight`, ...)."""
    growth, config, c0 = CONFIGS[name]
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def conv(key, cout, cin, k):
        sd[key + '.weight'] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cin * k * k))

    def bn(key, c):
        sd[key + '.weight'] = torch.rand(c, generator=g) + 0.5
        sd[key + '.bias'] = torch.randn(c, generator=g) * 0.1
        sd[key + '.running_mean'] = torch.randn(c, generator=g) * 0.1
        sd[key + '.running_var'] = torch.rand(c, generator=g) + 0.5

    conv('features.conv0', c0, 3, 7)
    bn('features.norm0', c0)
    bl, cfinal = blocks(name)
    for bi, n, cin in bl:
        for j in range(n):
            p = 'features.denseblock%d.denselayer%d' % (bi, j + 1)
            c = cin + j * growth
            bn(p + '.norm1', c)
            conv(p + '.conv1', BN_SIZE * growth, c, 1)
            bn(p + '.norm2', BN_SIZE * growth)
            conv(p + '.conv2', growth, BN_SIZE * growth, 3)
        if bi < len(config):
            c = cin + n * growth
            bn('features.transition%d.norm' % bi, c)
            conv('features.transition%d.conv' % bi, c // 2, c, 1)
    bn('features.norm5', cfinal)
    ch = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    sd['features.conv.weight'] = torch.randn(ch, cfinal, 1, 1, generator=g) * math.sqrt(1.0 / cfinal)
    sd['features.conv.bias'] = torch.randn(ch, generator=g) * 0.1
    return sd


def _bn(sd, x, key):
    return F.batch_norm(x, sd[key + '.running_mean'], sd[key + '.running_var'], sd[key + '.weight'], sd[key + '.bias'], False, 0.0, 1e-5)


def dense_layer(sd, x, key):
    """torchvision _DenseLayer (eval, drop_rate 0): conv2(relu2(norm2(conv1(relu1(norm1(x))))))."""
    y = F.conv2d(F.relu(_bn(sd, x, key + '.norm1')), sd[key + '.conv1.weight'])
    return F.conv2d(F.relu(_bn(sd, y, key + '.norm2')), sd[key + '.conv2.weight'], None, 1, 1)


def densenet_forward(sd, x, name='densenet121', collect=None):
    """model/densenet.py:64-65 (self.features(x)), eval mode.  `collect` receives every dense block's output (the concatenation), every
    transition's output and the stem pool output."""
    growth, config, _ = CONFIGS[name]
    x = F.relu(_bn(sd, F.conv2d(x, sd['features.conv0.weight'], None, 2, 3), 'features.norm0'))
    x = F.max_pool2d(x, 3, 2, 1)
    if collect is not None:
        collect['pool0'] = x
    bl, _ = blocks(name)
    for bi, n, _ in bl:
        feats = [x]
        for j in range(n):
            feats.append(dense_layer(sd, torch.cat(feats, 1), 'features.denseblock%d.denselayer%d' % (bi, j + 1)))
        x = torch.cat(feats, 1)
        if collect is not None:
            collect['denseblock%d' % bi] = x
        if bi < len(config):
            p = 'features.transition%d' % bi
            x = F.avg_pool2d(F.conv2d(F.relu(_bn(sd, x, p + '.norm')), sd[p + '.conv.weight']), 2, 2)
            if collect is not None:
                collect['transition%d' % bi] = x
    x = _bn(sd, x, 'features.norm5')
    return F.conv2d(x, sd['features.conv.weight'], sd['features.conv.bias'])
