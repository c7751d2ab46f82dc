"""model.inception4 -- Inception-v4 backbone plugin on the CUDA kernels (inference and training).

Drop-in for the reference's `model/inception4.py`: `Inception4(config_channels, anchors, num_cls, ratio=1)`, selectable with
`[model] dnn = model.inception4.Inception4`, with the reference's module tree and state_dict keys: `features.0 .. features.2` the stem convs,
`features.3 .. features.21` Mixed_3a, Mixed_4a, Mixed_5a, 4x Inception_A, Reduction_A, 7x Inception_B, Reduction_B, 3x Inception_C, and
`features.22` the 1x1 detection head with bias.  Every conv unit is `Conv2d`: conv -> BatchNorm2d(eps 1e-3) -> ReLU, or, with
`[batch_norm] enable = 0`, conv with bias -> ReLU.  Channel widths go through `config_channels(int(c * ratio), key)`, so a channel-pruned
checkpoint (`ConfigChannels(config, state_dict)`) or ratio != 1 gives widths that are not multiples of 32.
Forward x[B,3,H,W] fp32 -> [B, A*(5+C), OH, OW] fp32 with OH, OW following the valid convs (416 -> 11, 320 -> 8, 608 -> 17, 75 -> 1; below 75
a stage is empty).  Modules only hold parameters; the forward pass runs in fp16 NHWC:
  features.0 (3 -> 32, 3x3, s2, no pad)     -> yb_stem3x3_s2_bn_relu_fwd (a pruned features.0 with fewer filters runs with zero filters)
  every other Conv2d                        -> yb_conv2d_bn_act_fwd with the module's kh x kw, stride and padding, ReLU, the BatchNorm folded
                                               into the epilogue (or scale 1, shift = bias); each branch writes its own channel range of the
                                               block buffer (no torch.cat)
  MaxPool2d(3, stride=2) branches           -> yb_maxpool3x3_s2_valid_f16 straight into the block buffer
  branch3 = AvgPool2d(3, 1, 1, count_include_pad=False) + 1x1 conv -> yb_avgpool3x3_s1_excl_f16, then the conv
  features.22 (+ bias)                      -> yb_conv2d_bn_act_fwd, fp32 NCHW out.
Padded channel layout: the tensor-core conv needs Cin % 32 == 0, so every conv's output occupies round32(width) channels (the extra filters
are zero with scale 1, shift 0: exact zeros after the ReLU), a block buffer is its branches' padded segments in the reference's concatenation
order, and a max-pool branch carries its input's layout through.  Each tensor has a `Layout` (reference channel j -> buffer channel pos[j]);
a consumer's weight is scattered onto its input's layout, zero elsewhere, before the pack.  With ratio 1 and an unpruned model every width is a
multiple of 32 and every layout is the identity.  The scattered weights, folded BatchNorms and packs are cached per parameter version;
switching train() / eval() drops the cache.
In train() mode on a CUDA tensor the forward is one autograd node (model._TrainFunction) over
b200.train_engine.Inception4Trainer: batch-statistics BatchNorm (eps 1e-3, momentum 0.1) with the running-statistics update, or conv + bias
+ ReLU with BatchNorm disabled, and an explicit backward chain that gives every parameter its fp32 gradient.  Training needs the full-width
model: a channel-pruned or ratio != 1 model raises ValueError on a train-mode forward (its eval mode is unchanged).  There is no CPU path:
a train-mode forward on a CPU tensor raises NotImplementedError, an eval-mode one RuntimeError.
"""
import configparser

import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train

MIN_SIZE = 75      # the smallest input side whose every stage is non-empty (Reduction_B's output is 1 x 1)
STEM_FILTERS = 32  # yb_stem3x3_s2_bn_relu_fwd computes exactly 32 filters


def _round32(c):
    return (c + 31) // 32 * 32


class Layout(object):
    """Where each of the reference's channels sits in an fp16 NHWC buffer of `width` channels: reference channel j is buffer channel pos[j]."""

    def __init__(self, pos, width):
        self.pos = pos
        self.width = width

    @staticmethod
    def dense(channels):
        """A conv's own output: channels [0, C) of a round32(C)-wide buffer."""
        return Layout(torch.arange(channels), _round32(channels))

    @staticmethod
    def concat(parts):
        """The layouts side by side, each starting where the previous one's buffer ends."""
        pos, off = [], 0
        for p in parts:
            pos.append(p.pos + off)
            off += p.width
        return Layout(torch.cat(pos), off)


def scatter_weight(w, layout, cout_pad=None):
    """fp32 weight [Cout, Cin, kh, kw] -> [cout_pad, layout.width, kh, kw]: input channel j at layout.pos[j], zero in every other input channel
    and in the filters past Cout."""
    cout, cin, kh, kw = w.shape
    if cin != layout.pos.numel():
        raise ValueError('weight has %d input channels, its input layout %d' % (cin, layout.pos.numel()))
    full = torch.zeros(cout if cout_pad is None else cout_pad, layout.width, kh, kw, dtype=torch.float32, device=w.device)
    full[:cout].index_copy_(1, layout.pos.to(w.device), w.detach().float())
    return full


class Conv2d(nn.Module):
    """The reference's conv unit: nn.Conv2d -> BatchNorm2d(eps=0.001) -> ReLU, or nn.Conv2d with bias -> ReLU when BatchNorm is disabled."""

    def __init__(self, in_channels, out_channels, kernel_size, padding=0, stride=1, bn=True):
        nn.Module.__init__(self)
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding=padding, bias=not bn)
        self.bn = nn.BatchNorm2d(out_channels, eps=0.001) if bn else None


class Block(nn.Module):
    """One Inception-v4 block built from its class's table.  UNITS: (path, width, kernel, stride, padding, source) in the reference's registration
    order; `path` 'branchK.i' is element i of the nn.Sequential `branchK`; `source` None is the block input, 'avg' the block input after the
    count-exclusive 3x3 average pool (element 0 of the same Sequential), any other value the path of the producing unit.  POOLS: the attribute
    names of the MaxPool2d(3, stride=2) branches.  CAT: the concatenation order, unit paths and max-pool names.  FIXED: unit
    paths whose width the reference does not look up in the checkpoint (Inception_C's branch3 conv)."""
    UNITS = ()
    POOLS = ()
    CAT = ()
    FIXED = ()

    def __init__(self, config_channels, prefix, bn=True, ratio=1):
        nn.Module.__init__(self)
        cin = config_channels.channels
        # registration order as the reference's: a pool listed first in CAT (Mixed_3a) comes before the convs, the others after them
        first = [c for c in self.CAT[:1] if c in self.POOLS]
        for name in first:
            setattr(self, name, nn.MaxPool2d(3, stride=2))
        width = {}
        for path, w, k, s, p, src in self.UNITS:
            c_in = cin if src in (None, 'avg') else width[src]
            key = '%s.%s.conv.weight' % (prefix, path)
            c_out = int(w * ratio) if path in self.FIXED else config_channels(int(w * ratio), key)
            width[path] = c_out
            unit = Conv2d(c_in, c_out, k, padding=p, stride=s, bn=bn)
            head, _, idx = path.partition('.')
            if not idx:
                setattr(self, path, unit)
                continue
            if not hasattr(self, head):
                setattr(self, head, nn.Sequential())
                if src == 'avg':
                    getattr(self, head).append(nn.AvgPool2d(3, stride=1, padding=1, count_include_pad=False))
            getattr(self, head).append(unit)
        for name in self.POOLS:
            if name not in first:
                setattr(self, name, nn.MaxPool2d(3, stride=2))
        config_channels.channels = sum(cin if c in self.POOLS else width[c] for c in self.CAT)

    def chain(self, path):
        """(source kind 'conv' / 'avg', [units from the block input to `path`]) of one concatenated branch."""
        src = {u[0]: u[5] for u in self.UNITS}
        paths = [path]
        while src[paths[0]] not in (None, 'avg'):
            paths.insert(0, src[paths[0]])
        return ('avg' if src[paths[0]] == 'avg' else 'conv'), [self.get_submodule(p) for p in paths]


def _units(*rows):
    """Rows (path, width, kh, kw, stride, pad_h, pad_w, source) -> Block.UNITS."""
    return tuple((r[0], r[1], (r[2], r[3]), r[4], (r[5], r[6]), r[7]) for r in rows)


class Mixed_3a(Block):
    UNITS = _units(('conv', 96, 3, 3, 2, 0, 0, None))
    POOLS = ('maxpool',)
    CAT = ('maxpool', 'conv')


class Mixed_4a(Block):
    UNITS = _units(('branch0.0', 64, 1, 1, 1, 0, 0, None), ('branch0.1', 96, 3, 3, 1, 0, 0, 'branch0.0'),
                   ('branch1.0', 64, 1, 1, 1, 0, 0, None), ('branch1.1', 64, 1, 7, 1, 0, 3, 'branch1.0'), ('branch1.2', 64, 7, 1, 1, 3, 0, 'branch1.1'),
                   ('branch1.3', 96, 3, 3, 1, 0, 0, 'branch1.2'))
    CAT = ('branch0.1', 'branch1.3')


class Mixed_5a(Block):
    UNITS = _units(('conv', 192, 3, 3, 2, 0, 0, None))
    POOLS = ('maxpool',)
    CAT = ('conv', 'maxpool')


class Inception_A(Block):
    UNITS = _units(('branch0', 96, 1, 1, 1, 0, 0, None),
                   ('branch1.0', 64, 1, 1, 1, 0, 0, None), ('branch1.1', 96, 3, 3, 1, 1, 1, 'branch1.0'),
                   ('branch2.0', 64, 1, 1, 1, 0, 0, None), ('branch2.1', 96, 3, 3, 1, 1, 1, 'branch2.0'), ('branch2.2', 96, 3, 3, 1, 1, 1, 'branch2.1'),
                   ('branch3.1', 96, 1, 1, 1, 0, 0, 'avg'))
    CAT = ('branch0', 'branch1.1', 'branch2.2', 'branch3.1')


class Reduction_A(Block):
    UNITS = _units(('branch0', 384, 3, 3, 2, 0, 0, None),
                   ('branch1.0', 192, 1, 1, 1, 0, 0, None), ('branch1.1', 224, 3, 3, 1, 1, 1, 'branch1.0'),
                   ('branch1.2', 256, 3, 3, 2, 0, 0, 'branch1.1'))
    POOLS = ('branch2',)
    CAT = ('branch0', 'branch1.2', 'branch2')


class Inception_B(Block):
    UNITS = _units(('branch0', 384, 1, 1, 1, 0, 0, None),
                   ('branch1.0', 192, 1, 1, 1, 0, 0, None), ('branch1.1', 224, 1, 7, 1, 0, 3, 'branch1.0'),
                   ('branch1.2', 256, 7, 1, 1, 3, 0, 'branch1.1'),
                   ('branch2.0', 192, 1, 1, 1, 0, 0, None), ('branch2.1', 192, 7, 1, 1, 3, 0, 'branch2.0'),
                   ('branch2.2', 224, 1, 7, 1, 0, 3, 'branch2.1'), ('branch2.3', 224, 7, 1, 1, 3, 0, 'branch2.2'),
                   ('branch2.4', 256, 1, 7, 1, 0, 3, 'branch2.3'),
                   ('branch3.1', 128, 1, 1, 1, 0, 0, 'avg'))
    CAT = ('branch0', 'branch1.2', 'branch2.4', 'branch3.1')


class Reduction_B(Block):
    UNITS = _units(('branch0.0', 192, 1, 1, 1, 0, 0, None), ('branch0.1', 192, 3, 3, 2, 0, 0, 'branch0.0'),
                   ('branch1.0', 256, 1, 1, 1, 0, 0, None), ('branch1.1', 256, 1, 7, 1, 0, 3, 'branch1.0'),
                   ('branch1.2', 320, 7, 1, 1, 3, 0, 'branch1.1'), ('branch1.3', 320, 3, 3, 2, 0, 0, 'branch1.2'))
    POOLS = ('branch2',)
    CAT = ('branch0.1', 'branch1.3', 'branch2')


class Inception_C(Block):
    UNITS = _units(('branch0', 256, 1, 1, 1, 0, 0, None),
                   ('branch1_0', 384, 1, 1, 1, 0, 0, None), ('branch1_1a', 256, 1, 3, 1, 0, 1, 'branch1_0'),
                   ('branch1_1b', 256, 3, 1, 1, 1, 0, 'branch1_0'),
                   ('branch2_0', 384, 1, 1, 1, 0, 0, None), ('branch2_1', 448, 3, 1, 1, 1, 0, 'branch2_0'),
                   ('branch2_2', 512, 1, 3, 1, 0, 1, 'branch2_1'), ('branch2_3a', 256, 1, 3, 1, 0, 1, 'branch2_2'),
                   ('branch2_3b', 256, 3, 1, 1, 1, 0, 'branch2_2'),
                   ('branch3.1', 256, 1, 1, 1, 0, 0, 'avg'))
    CAT = ('branch0', 'branch1_1a', 'branch1_1b', 'branch2_3a', 'branch2_3b', 'branch3.1')
    FIXED = ('branch3.1',)


BLOCKS = (Mixed_3a, Mixed_4a, Mixed_5a) + (Inception_A,) * 4 + (Reduction_A,) + (Inception_B,) * 7 + (Reduction_B,) + (Inception_C,) * 3
STEM = ((32, 3, 2, 0), (32, 3, 1, 0), (64, 3, 1, 1))      # (filters, kernel, stride, padding) of features.0 .. features.2


class Inception4(model.Backbone):
    TRAINER = _train.Inception4Trainer

    def __init__(self, config_channels, anchors, num_cls, ratio=1):
        model.Backbone.__init__(self)
        config = config_channels.config
        bn = config.getboolean('batch_norm', 'enable')
        features = []
        for filters, k, s, p in STEM:
            cin = config_channels.channels
            features.append(Conv2d(cin, config_channels(filters, 'features.%d.conv.weight' % len(features)), k, padding=p, stride=s, bn=bn))
        if features[0].conv.out_channels > STEM_FILTERS:
            raise ValueError('Inception4: features.0 has %d filters; the stem kernel computes at most %d'
                             % (features[0].conv.out_channels, STEM_FILTERS))
        for cls in BLOCKS:
            features.append(cls(config_channels, 'features.%d' % len(features), bn=bn, ratio=ratio))
        features.append(nn.Conv2d(config_channels.channels, model.output_channels(len(anchors), num_cls), 1))
        self.features = nn.Sequential(*features)
        self._init(config)
        self._plan()
        _pretrained(self, config)

    def _init(self, config):
        """He-normal conv weights (kaiming_normal, fan_in, gain sqrt 2); BatchNorm weight 1, bias 0, trainable as `[batch_norm] gamma / beta`."""
        gamma = config.getboolean('batch_norm', 'gamma', fallback=True)
        beta = config.getboolean('batch_norm', 'beta', fallback=True)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)
            elif isinstance(m, nn.BatchNorm2d):
                with torch.no_grad():
                    m.weight.fill_(1)
                    m.bias.zero_()
                m.weight.requires_grad = gamma
                m.bias.requires_grad = beta

    def _plan(self):
        """The padded channel layout of every tensor: `layouts[unit]` is the layout its input arrives in; `blocks[i]` = (module, segments, output
        layout) with segments (kind, units, channel offset), kind 'conv' / 'avg' / 'max', in concatenation order."""
        f = self.features
        self.layouts = {f[0]: None, f[1]: Layout(torch.arange(f[0].conv.out_channels), STEM_FILTERS), f[2]: Layout.dense(f[1].conv.out_channels)}
        lay = Layout.dense(f[2].conv.out_channels)
        self.blocks = []
        for m in f[3:-1]:
            segs, parts, off = [], [], 0
            for name in m.CAT:
                if name in m.POOLS:
                    kind, units, part = 'max', [], lay
                else:
                    kind, units = m.chain(name)
                    self.layouts[units[0]] = lay
                    for a, b in zip(units[:-1], units[1:]):
                        self.layouts[b] = Layout.dense(a.conv.out_channels)
                    part = Layout.dense(units[-1].conv.out_channels)
                segs.append((kind, tuple(units), off))
                parts.append(part)
                off += part.width
            lay = Layout.concat(parts)
            self.blocks.append((m, tuple(segs), lay))
        self.layouts[f[-1]] = lay

    def scope(self, name):
        return '.'.join(name.split('.')[:-2])

    # ---- operand preparation (cached per parameter version) ------------------------------------------
    def scattered(self, unit):
        """The fp32 weight handed to the pack: [round32(Cout), input width, kh, kw], the module's weight scattered onto its input's layout."""
        w = unit.conv.weight
        return scatter_weight(w, self.layouts[unit], _round32(w.shape[0]))

    def _operands(self, unit):
        """(weight, scale, shift) of one Conv2d: features.0's fp32 weight with zero filters up to 32, else the packed scattered weight; the
        epilogue padded to the weight's filter count."""
        def build():
            if unit is self.features[0]:
                w = unit.conv.weight.detach().float()
                w32 = torch.zeros(STEM_FILTERS, 3, 3, 3, dtype=torch.float32, device=w.device)
                w32[:w.shape[0]] = w
                return (w32,) + _engine.fold_epilogue(unit.bn, unit.conv.bias, STEM_FILTERS)
            full = self.scattered(unit)
            return (_ops.pack_weight_khw_f16(full.contiguous()),) + _engine.fold_epilogue(unit.bn, unit.conv.bias, full.shape[0])
        return self._cache.fetch(unit, (unit.conv.weight,) + _engine.epilogue_tensors(unit.bn, unit.conv.bias), build)

    def scattered_head(self):
        """The head's fp32 weight handed to the pack: [Cout, input width, 1, 1], scattered onto the last block's layout."""
        head = self.features[-1]
        return scatter_weight(head.weight, self.layouts[head])

    def _head(self):
        w, b = self.features[-1].weight, self.features[-1].bias
        return self._cache.fetch('head', (w, b), lambda: (_ops.pack_weight_khw_f16(self.scattered_head().contiguous()),
                                                          torch.ones(w.shape[0], dtype=torch.float32, device=w.device), b.detach().float().contiguous()))

    # ---- units -----------------------------------------------------------------------------------------
    def unit(self, unit, x, out=None, y_ch_off=0):
        """One Conv2d on x (fp16 NHWC in its input layout): into channels [y_ch_off, y_ch_off + round32(Cout)) of `out`, or a new tensor."""
        conv = unit.conv
        w16, s, t = self._operands(unit)
        return _ops.conv2d_bn_act(x, w16, s, t, 0.0, stride=conv.stride[0], pad=conv.padding, out=out, y_ch_off=y_ch_off)

    def block(self, index, x):
        """Block features.`index` (3 .. 21) on x (fp16 NHWC in its input layout): its output buffer (fp16 NHWC, the block's output layout)."""
        m, segs, lay = self.blocks[index - 3]
        b, h, w, _ = x.shape
        if m.POOLS:      # Mixed_3a / 5a, Reduction_A / B: every branch ends in a 3x3 valid stride-2 conv or pool
            oh, ow = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        elif isinstance(m, Mixed_4a):
            oh, ow = h - 2, w - 2
        else:
            oh, ow = h, w
        out = torch.empty(b, oh, ow, lay.width, dtype=torch.float16, device=x.device)
        memo = {}
        for kind, units, off in segs:
            if kind == 'max':
                _ops.maxpool3x3_s2_valid(x, out, off)
                continue
            t = x if kind == 'conv' else _ops.avgpool3x3_s1_excl(x)
            for j in range(len(units) - 1):       # Inception_C's branch1_0 and branch2_0 .. 2_2 feed two branches: run once
                key = units[:j + 1]
                if key not in memo:
                    memo[key] = self.unit(units[j], t)
                t = memo[key]
            self.unit(units[-1], t, out, off)
        return out

    def stem(self, x):
        """features.0 .. features.2: x fp32 NCHW -> Mixed_3a's input, fp16 NHWC."""
        f = self.features
        w32, s, t = self._operands(f[0])
        a = _ops.stem3x3_s2(x, w32, s, t, pad=0)
        return self.unit(f[2], self.unit(f[1], a))

    def run(self, x, collect=None):
        """Forward on the kernels; `collect` (a dict) receives the stem output ('stem') and every block's buffer under its index (fp16 NHWC,
        padded layout: see `blocks`)."""
        b, c, h, w = x.shape
        if c != 3:
            raise ValueError('Inception4 expects [B,3,H,W]')
        if h < MIN_SIZE or w < MIN_SIZE:
            raise ValueError('Inception4: a %d x %d input leaves a stage empty (H and W must be >= %d)' % (h, w, MIN_SIZE))
        if not x.is_cuda:
            raise RuntimeError('Inception4: input must be a CUDA tensor; there is no CPU fallback')
        a = self.stem(x.contiguous().float())
        if collect is not None:
            collect['stem'] = a
        for i in range(3, 3 + len(self.blocks)):
            a = self.block(i, a)
            if collect is not None:
                collect[i] = a
        w16, one, bias = self._head()
        return _ops.conv2d_bn_act(a, w16, one, bias, 1.0, out_mode=_ops.OUT_F32_NCHW)

    def forward(self, x):
        if self.training:
            if not x.is_cuda:
                raise NotImplementedError('Inception4: training runs on the CUDA kernels only; the input is a CPU tensor')
            return self.train_forward(x)
        return self.run(x)


def _pretrained(net, config):
    """`[model] pretrained`: copy the ImageNet weights of `pretrainedmodels`' inceptionv4 (setting `[inception4] pretrained`) whose keys exist
    in this model.  Needs that package and the network."""
    try:
        if not config.getboolean('model', 'pretrained'):
            return net
    except (configparser.NoSectionError, configparser.NoOptionError):
        return net
    from pretrainedmodels.models.inceptionv4 import pretrained_settings
    settings = pretrained_settings['inceptionv4'][config.get('inception4', 'pretrained')]
    loaded = torch.hub.load_state_dict_from_url(settings['url'], progress=False)
    state_dict = net.state_dict()
    for key, value in loaded.items():
        if key in state_dict:
            state_dict[key] = value
    net.load_state_dict(state_dict)
    return net
