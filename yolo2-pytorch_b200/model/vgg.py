"""model.vgg -- VGG backbone plugin on the CUDA kernels (inference and training).

Drop-in for the reference's `model/vgg.py`: the constructors `vgg11, vgg11_bn, vgg13, vgg13_bn, vgg16, vgg16_bn, vgg19, vgg19_bn
(config_channels, anchors, num_cls)` (:57-150), selectable with `[model] dnn = model.vgg.vgg16`, with the reference's module tree and
state_dict keys: `features` an nn.Sequential of Conv2d(3x3, padding 1, bias) [-> BatchNorm2d] -> ReLU units and MaxPool2d(2, 2), built from
torchvision's configurations 'A', 'B', 'D', 'E' (:41-50); `conv` the 1x1 detection head with bias (:32).  The `_bn` in the name decides
BatchNorm (`[batch_norm] enable` is not read).  Widths go through `config_channels(v, 'features.%d.weight')`, so a channel-pruned checkpoint
(`ConfigChannels(config, state_dict)`) sets any width.  Initialisation is the reference's `_initialize_weights` (torchvision 0.2): conv
weights N(0, 2 / (kh * kw * out_channels)), conv biases 0, BatchNorm weight 1 and bias 0.
Forward x[B,3,H,W] fp32, H and W multiples of 32 -> [B, A*(5+C), H/32, W/32] fp32.  Modules only hold parameters; the forward pass runs in
fp16 NHWC:
  features.0 (3 -> <= 64 filters)     -> yb_conv0_c64_bn_act_fwd: the fp32 image in, the BatchNorm folded (or scale 1, shift = bias), ReLU,
                                         and the 2x2 max-pool fused when a MaxPool2d follows (vgg11); a pruned layer runs with zero filters
  every other conv unit               -> yb_conv_bn_act_fwd (3x3), the same epilogue
  MaxPool2d(2, 2) after those         -> yb_maxpool2x2_f16 (the implicit-GEMM conv fuses the pool only for Cin = 32)
  conv (+ bias)                       -> yb_conv_bn_act_fwd (1x1), fp32 NCHW out.
Padded channel layout: the tensor-core conv needs Cin % 32 == 0, so a conv with C filters writes round32(C) channels (features.0: 64), the
extra filters zero with scale 1, shift 0 (exact zeros after the ReLU), and the consumer's packed weight is zero on those input channels
(pack_weight_khw_f16 with cout_pad / cin_pad).  Folded BatchNorms and packed weights are cached per parameter version; switching train() /
eval() drops the cache, so inference after training uses the trained state.
In train() mode the forward is one autograd node (model._TrainFunction) over b200.train_engine.VGGTrainer: batch-statistics
BatchNorm (momentum and eps read from the modules), the explicit backward chain, the first layer's weight gradient from the fp32 image
(yb_conv0_c64_wgrad).  Training needs features.0 with 64 filters and every other width a multiple of 32.  There is no CPU path.
"""
import math

import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train

# torchvision's VGG configurations (`cfgs`; `cfg` in torchvision 0.2): output widths of the 3x3 convs, 'M' = MaxPool2d(2, 2)
CFGS = {
    'A': [64, 'M', 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'B': [64, 64, 'M', 128, 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'D': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M'],
    'E': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512, 'M'],
}
ARCH = {'vgg11': 'A', 'vgg13': 'B', 'vgg16': 'D', 'vgg19': 'E'}
FIRST_FILTERS = 64   # yb_conv0_c64_bn_act_fwd computes exactly 64 filters


def _round32(c):
    return (c + 31) // 32 * 32


def _features(config_channels, arch, batch_norm):
    """`features` of configuration `arch`: per width a 3x3 padding-1 conv with bias, a BatchNorm2d when `batch_norm`, and a ReLU; per 'M' a
    2x2 stride-2 max-pool.  A conv's width is looked up under its own state_dict key, `features.<its index>.weight`."""
    seq = nn.Sequential()
    for item in CFGS[arch]:
        if item == 'M':
            seq.append(nn.MaxPool2d(kernel_size=2, stride=2))
            continue
        cin = config_channels.channels
        cout = config_channels(item, 'features.%d.weight' % len(seq))
        seq.append(nn.Conv2d(cin, cout, kernel_size=3, padding=1))
        if batch_norm:
            seq.append(nn.BatchNorm2d(cout))
        seq.append(nn.ReLU(inplace=True))
    return seq


class _Unit(object):
    """One conv unit of `features`: the conv, its BatchNorm (or None), whether a MaxPool2d follows, and the feature index of that pool."""

    def __init__(self, conv, bn, pool_index):
        self.conv, self.bn, self.pool_index = conv, bn, pool_index

    @property
    def pool(self):
        return self.pool_index is not None


class VGG(model.Backbone):
    TRAINER = _train.VGGTrainer

    def __init__(self, config_channels, anchors, num_cls, features):
        model.Backbone.__init__(self)
        self.features = features
        self.conv = nn.Conv2d(config_channels.channels, model.output_channels(len(anchors), num_cls), 1)
        self._initialize_weights()
        self.units = self._plan()
        if self.units[0].conv.out_channels > FIRST_FILTERS:
            raise ValueError('VGG: features.0 has %d filters; the first-layer kernel computes at most %d'
                             % (self.units[0].conv.out_channels, FIRST_FILTERS))

    def _initialize_weights(self):
        """torchvision 0.2's VGG._initialize_weights, which the reference calls (model/vgg.py:33)."""
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                with torch.no_grad():
                    m.weight.normal_(0, math.sqrt(2. / n))
                    if m.bias is not None:
                        m.bias.zero_()
            elif isinstance(m, nn.BatchNorm2d):
                with torch.no_grad():
                    m.weight.fill_(1)
                    m.bias.zero_()

    def _plan(self):
        """The conv units in order, each with its BatchNorm and the index of the MaxPool2d that follows it."""
        f = list(self.features)
        units = []
        for i, m in enumerate(f):
            if not isinstance(m, nn.Conv2d):
                continue
            j = i + 1
            bn = f[j] if isinstance(f[j], nn.BatchNorm2d) else None
            j += 2 if bn is not None else 1           # past the ReLU
            units.append(_Unit(m, bn, j if j < len(f) and isinstance(f[j], nn.MaxPool2d) else None))
        return units

    # ---- operand preparation (cached per parameter version) ------------------------------------------
    def in_width(self, index):
        """Channels of the fp16 buffer unit `index` reads: 64 after features.0, else round32 of the producer's filters."""
        if index == 0:
            return 3
        return FIRST_FILTERS if index == 1 else _round32(self.units[index - 1].conv.out_channels)

    def out_width(self, index):
        return FIRST_FILTERS if index == 0 else _round32(self.units[index].conv.out_channels)

    def _operands(self, index):
        """(weight, scale, shift) of unit `index`: features.0's fp32 weight with zero filters up to 64, else the packed fp16 weight on the
        padded layout; the epilogue padded to the unit's output width."""
        u = self.units[index]

        def build():
            w = u.conv.weight.detach().float().contiguous()
            if index == 0:
                wp = torch.zeros(FIRST_FILTERS, 3, 3, 3, dtype=torch.float32, device=w.device)
                wp[:w.shape[0]] = w
            else:
                wp = _ops.pack_weight_khw_f16(w, self.out_width(index), self.in_width(index))
            return (wp,) + _engine.fold_epilogue(u.bn, u.conv.bias, self.out_width(index))
        return self._cache.fetch(index, (u.conv.weight,) + _engine.epilogue_tensors(u.bn, u.conv.bias), build)

    def _head(self):
        w, b = self.conv.weight, self.conv.bias
        cin_pad = self.out_width(len(self.units) - 1)
        return self._cache.fetch('head', (w, b), lambda: (_ops.pack_weight_khw_f16(w.detach().float().contiguous(), None, cin_pad),
                                                          torch.ones(w.shape[0], dtype=torch.float32, device=w.device), b.detach().float().contiguous()))

    # ---- forward ---------------------------------------------------------------------------------------
    def run(self, x, collect=None):
        """Forward on the kernels; `collect` (a dict) receives every MaxPool2d's output under its feature index (fp16 NHWC, padded layout)."""
        if x.dim() != 4:
            raise ValueError('VGG expects [B,3,H,W]')
        x, lut, (b, c, h, w) = self.eval_input(x)
        if c != 3:
            raise ValueError('VGG expects [B,3,H,W]')
        if h % 32 or w % 32 or h == 0 or w == 0:
            raise ValueError('VGG: H and W must be positive multiples of 32 (got %d x %d)' % (h, w))
        if not x.is_cuda:
            raise RuntimeError('VGG: input must be a CUDA tensor; there is no CPU fallback')
        u0 = self.units[0]
        w0, s, t = self._operands(0)
        a = _ops.conv0_c64_bn_act(x, w0, s, t, 0.0, pool=u0.pool, lut=lut)
        if collect is not None and u0.pool:
            collect[u0.pool_index] = a
        for i in range(1, len(self.units)):
            u = self.units[i]
            w16, s, t = self._operands(i)
            a = _ops.conv_bn_act(a, w16, s, t, 0.0)
            if u.pool:
                a = _ops.maxpool2x2(a)
                if collect is not None:
                    collect[u.pool_index] = a
        w16, one, bias = self._head()
        return _ops.conv_bn_act(a, w16, one, bias, 1.0, out_mode=_ops.OUT_F32_NCHW)

    def forward(self, x):
        if self.training:
            if not x.is_cuda:
                raise RuntimeError('VGG training: input must be a CUDA tensor; there is no CPU fallback')
            return self.train_forward(x)
        return self.run(x)


def _pretrained(net, config_channels, name):
    """`[model] pretrained` (model/vgg.py:59-67): copy the torchvision ImageNet weights whose keys exist in this model (the `features.*`
    convs and BatchNorms; the classifier has no counterpart).  Needs the network, so it is not exercised by the tests."""
    config = getattr(config_channels, 'config', None)
    if config is None or not config.getboolean('model', 'pretrained', fallback=False):
        return net
    import torchvision.models as tvm
    weights = getattr(tvm, name.upper() + '_Weights').IMAGENET1K_V1
    state_dict = net.state_dict()
    for key, value in weights.get_state_dict(progress=False).items():
        if key in state_dict:
            state_dict[key] = value
    net.load_state_dict(state_dict)
    return net


def _build(name, config_channels, anchors, num_cls):
    arch = ARCH[name[:5]]
    net = VGG(config_channels, anchors, num_cls, _features(config_channels, arch, name.endswith('_bn')))
    return _pretrained(net, config_channels, name)


def vgg11(config_channels, anchors, num_cls):
    return _build('vgg11', config_channels, anchors, num_cls)


def vgg11_bn(config_channels, anchors, num_cls):
    return _build('vgg11_bn', config_channels, anchors, num_cls)


def vgg13(config_channels, anchors, num_cls):
    return _build('vgg13', config_channels, anchors, num_cls)


def vgg13_bn(config_channels, anchors, num_cls):
    return _build('vgg13_bn', config_channels, anchors, num_cls)


def vgg16(config_channels, anchors, num_cls):
    return _build('vgg16', config_channels, anchors, num_cls)


def vgg16_bn(config_channels, anchors, num_cls):
    return _build('vgg16_bn', config_channels, anchors, num_cls)


def vgg19(config_channels, anchors, num_cls):
    return _build('vgg19', config_channels, anchors, num_cls)


def vgg19_bn(config_channels, anchors, num_cls):
    return _build('vgg19_bn', config_channels, anchors, num_cls)
