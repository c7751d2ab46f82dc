"""model.densenet -- DenseNet backbone plugin on the CUDA kernels (inference and training).

Drop-in for the reference's `model/densenet.py`: same constructors `densenet121 / densenet169 / densenet201 / densenet161
(config_channels, anchors, num_cls)` (:68-117), same module tree and state_dict keys as torchvision's DenseNet under `features`
(`conv0, norm0, relu0, pool0, denseblockN.denselayerM.{norm1, conv1, norm2, conv2}, transitionN.{norm, conv}, norm5`) plus the 1x1
detection head `features.conv` (:53-54), same forward contract x[B,3,H,W] fp32 -> [B, A*(5+C), H/32, W/32] fp32 (:64-65: `norm5` feeds the
head directly, with no ReLU).  Modules only hold parameters; the forward pass runs in fp16 NHWC with one buffer per dense block, as wide as
the block's final channel count, so the concatenations of the reference are never copied:
  conv0 7x7 s2 + norm0 + relu0       -> yb_stem7x7_bn_relu_fwd (the ResNet stem)
  pool0 3x3 s2 p1                    -> yb_maxpool3x3_s2_ld_f16 into channels [0, 64) of block 1's buffer
  dense layer over channels [0, Ci)  -> yb_conv1x1_preact_fwd (norm1 + relu1 applied to the conv's input, norm2 + relu2 folded into its
                                        epilogue) into a 128-channel temporary, then the 3x3 conv2 (yb_conv_bn_act_fwd, identity epilogue)
                                        writing its 32 channels at channel Ci of the block buffer
  transition                         -> yb_bn_relu_avgpool2x2_f16 (norm + relu + AvgPool2d(2)), then the 1x1 conv on the pooled tensor
                                        into channels [0, C/2) of the next block's buffer.  Pooling before a 1x1 conv equals pooling after it
                                        in exact arithmetic and cuts that conv's work 4x; only the fp32 rounding order differs from the reference.
  norm5 + head conv (+ bias)         -> yb_conv1x1_preact_fwd with norm5 as the (identity-activation) pre-transform, fp32 NCHW out.
The folded BatchNorms and packed weights are cached per parameter version; switching train() / eval() drops the cache.  There is no CPU
path.

train() mode on a CUDA tensor runs one autograd node over b200.train_engine.DenseNetTrainer (batch-statistics BatchNorm shared by every
norm that reads a block channel, running-statistics update, the explicit backward chain), so train.iterate and train.GraphedStep work as
for the other backbones.  A CPU tensor, densenet161 and drop_rate > 0 raise NotImplementedError in train mode.
"""
import re
from collections import OrderedDict

import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train

# torchvision 0.2 (the reference's) named a dense layer's parameters `norm.1`, `conv.2`, ...; torchvision's own loader renames them
_OLD_KEY = re.compile(r'^(.*denselayer\d+\.(?:norm|relu|conv))\.((?:[12])\.(?:weight|bias|running_mean|running_var|num_batches_tracked))$')


def remap_legacy_keys(state_dict, prefix=''):
    """Rename torchvision-0.2 dense-layer keys (`...denselayer1.norm.1.weight`) to the current ones (`...denselayer1.norm1.weight`) in place."""
    for key in list(state_dict.keys()):
        if not key.startswith(prefix):
            continue
        m = _OLD_KEY.match(key[len(prefix):])
        if m is not None:
            state_dict[prefix + m.group(1) + m.group(2)] = state_dict.pop(key)
    return state_dict


class _DenseLayer(nn.Module):
    def __init__(self, num_input_features, growth_rate, bn_size):
        nn.Module.__init__(self)
        self.norm1 = nn.BatchNorm2d(num_input_features)
        self.relu1 = nn.ReLU(inplace=True)
        self.conv1 = nn.Conv2d(num_input_features, bn_size * growth_rate, kernel_size=1, stride=1, bias=False)
        self.norm2 = nn.BatchNorm2d(bn_size * growth_rate)
        self.relu2 = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(bn_size * growth_rate, growth_rate, kernel_size=3, stride=1, padding=1, bias=False)


class _DenseBlock(nn.Module):
    def __init__(self, num_layers, num_input_features, bn_size, growth_rate):
        nn.Module.__init__(self)
        for i in range(num_layers):
            self.add_module('denselayer%d' % (i + 1), _DenseLayer(num_input_features + i * growth_rate, growth_rate, bn_size))


class _Transition(nn.Sequential):
    def __init__(self, num_input_features, num_output_features):
        nn.Sequential.__init__(self)
        self.add_module('norm', nn.BatchNorm2d(num_input_features))
        self.add_module('relu', nn.ReLU(inplace=True))
        self.add_module('conv', nn.Conv2d(num_input_features, num_output_features, kernel_size=1, stride=1, bias=False))
        self.add_module('pool', nn.AvgPool2d(kernel_size=2, stride=2))


class DenseNet(model.Backbone):
    TRAINER = _train.DenseNetTrainer

    def __init__(self, config_channels, anchors, num_cls, growth_rate=32, block_config=(6, 12, 24, 16), num_init_features=64, bn_size=4, drop_rate=0):
        model.Backbone.__init__(self)
        # drop_rate (model/densenet.py:30): torchvision's dense-layer dropout acts in training only, so the eval-mode forward is the same for any rate
        self.drop_rate = float(drop_rate)
        self.growth_rate, self.block_config, self.num_init_features, self.bn_size = growth_rate, tuple(block_config), num_init_features, bn_size
        self.features = nn.Sequential(OrderedDict([
            ('conv0', nn.Conv2d(3, num_init_features, kernel_size=7, stride=2, padding=3, bias=False)),
            ('norm0', nn.BatchNorm2d(num_init_features)),
            ('relu0', nn.ReLU(inplace=True)),
            ('pool0', nn.MaxPool2d(kernel_size=3, stride=2, padding=1)),
        ]))
        num_features = num_init_features
        self.block_channels = []               # (input, output) channels of each dense block
        for i, num_layers in enumerate(block_config):
            self.features.add_module('denseblock%d' % (i + 1), _DenseBlock(num_layers, num_features, bn_size, growth_rate))
            self.block_channels.append((num_features, num_features + num_layers * growth_rate))
            num_features = num_features + num_layers * growth_rate
            if i != len(block_config) - 1:
                self.features.add_module('transition%d' % (i + 1), _Transition(num_features, num_features // 2))
                num_features = num_features // 2
        self.features.add_module('norm5', nn.BatchNorm2d(num_features))
        self.features.add_module('conv', nn.Conv2d(num_features, model.output_channels(len(anchors), num_cls), 1))
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        self._register_load_state_dict_pre_hook(self._remap_hook)

    @staticmethod
    def _remap_hook(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        remap_legacy_keys(state_dict, prefix)

    def unsupported(self):
        """Why this configuration has no kernel path (None when it has one)."""
        reasons = []
        if self.num_init_features != 64:
            reasons.append('a %d-channel stem (the stem kernel computes 64 channels)' % self.num_init_features)
        if self.growth_rate % 32 or (self.bn_size * self.growth_rate) % 32 or any(c % 32 for c, _ in self.block_channels):
            reasons.append('growth rate %d (block widths must stay multiples of 32 for the tensor-core conv)' % self.growth_rate)
        return '; '.join(reasons) or None

    # ---- operand preparation (cached per parameter version) ------------------------------------------
    def _fold(self, key, bn):
        return self._cache.fetch(key, _engine.epilogue_tensors(bn), lambda: _engine.fold_epilogue(bn, None))

    def _packed(self, key, w):
        return self._cache.fetch(key, (w,), lambda: _ops.pack_weight_f16(w.detach().float().contiguous(), 0))

    def _const(self, value, n, device):
        return self._cache.fetch(('const', value, n, str(device)), (), lambda: torch.full((n,), float(value), dtype=torch.float32, device=device))

    # ---- units -----------------------------------------------------------------------------------------
    def dense_layer(self, key, layer, buf, cin, tmp):
        """One _DenseLayer on channels [0, cin) of the block buffer: its `growth_rate` new channels land at channel cin of `buf`."""
        ps, pb = self._fold(key + '.norm1', layer.norm1)
        s2, b2 = self._fold(key + '.norm2', layer.norm2)
        _ops.conv1x1_preact(buf, self._packed(key + '.conv1', layer.conv1.weight), ps, pb, True, s2, b2, 0.0, out=tmp, cin=cin)
        g = layer.conv2.weight.shape[0]
        _ops.conv_bn_act(tmp, self._packed(key + '.conv2', layer.conv2.weight), self._const(1, g, buf.device), self._const(0, g, buf.device), 1.0,
                         out=buf, y_ch_off=cin)

    def transition(self, key, trans, buf, out):
        """norm + relu + AvgPool2d(2) on all channels of `buf`, then the 1x1 conv into channels [0, C/2) of `out`."""
        b, h, w, c = buf.shape
        s, t = self._fold(key + '.norm', trans.norm)
        pooled = torch.empty(b, h // 2, w // 2, c, dtype=torch.float16, device=buf.device)
        _ops.call('yb_bn_relu_avgpool2x2_f16', buf, c, s, t, pooled, b, h, w, c)
        co = trans.conv.weight.shape[0]
        _ops.conv_bn_act(pooled, self._packed(key + '.conv', trans.conv.weight), self._const(1, co, buf.device), self._const(0, co, buf.device),
                         1.0, out=out, y_ch_off=0)

    def stem(self, x, buf):
        """conv0 + norm0 + relu0 + pool0 into channels [0, 64) of block 1's buffer."""
        b, _, h, w = x.shape
        f = self.features
        s, t = self._fold('norm0', f.norm0)
        stem = torch.empty(b, h // 2, w // 2, 64, dtype=torch.float16, device=x.device)
        _ops.call('yb_stem7x7_bn_relu_fwd', x, f.conv0.weight.detach().float().contiguous(), s, t, stem, b, h, w)
        _ops.call('yb_maxpool3x3_s2_ld_f16', stem, buf, buf.shape[-1], 0, b, h // 2, w // 2, 64)

    def run(self, x, collect=None):
        """Forward on the kernels; `collect` (a dict) receives every dense block's and transition's output buffer (fp16 NHWC)."""
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('DenseNet expects [B,3,H,W] with H, W multiples of 32')
        why = self.unsupported()
        if why is not None:
            raise NotImplementedError('DenseNet: no kernel path for %s' % why)
        if not x.is_cuda:
            raise RuntimeError('DenseNet: input must be a CUDA tensor; there is no CPU fallback')
        x = x.contiguous().float()
        f = self.features
        hh, ww = h // 4, w // 4
        buf = torch.empty(b, hh, ww, self.block_channels[0][1], dtype=torch.float16, device=x.device)
        self.stem(x, buf)
        for i, n in enumerate(self.block_config):
            name = 'denseblock%d' % (i + 1)
            block = getattr(f, name)
            cin0 = self.block_channels[i][0]
            tmp = torch.empty(b, hh, ww, self.bn_size * self.growth_rate, dtype=torch.float16, device=x.device)
            for j in range(n):
                self.dense_layer('%s.denselayer%d' % (name, j + 1), getattr(block, 'denselayer%d' % (j + 1)), buf, cin0 + j * self.growth_rate, tmp)
            if collect is not None:
                collect[name] = buf
            if i + 1 < len(self.block_config):
                tname = 'transition%d' % (i + 1)
                hh, ww = hh // 2, ww // 2
                nbuf = torch.empty(b, hh, ww, self.block_channels[i + 1][1], dtype=torch.float16, device=x.device)
                self.transition(tname, getattr(f, tname), buf, nbuf)
                if collect is not None:
                    collect[tname] = nbuf[..., :self.block_channels[i + 1][0]]
                buf = nbuf
        s5, t5 = self._fold('norm5', f.norm5)
        cout = f.conv.weight.shape[0]
        return _ops.conv1x1_preact(buf, self._packed('head', f.conv.weight), s5, t5, False, self._const(1, cout, x.device),
                                   f.conv.bias.detach().float().contiguous(), 1.0, out_mode=_ops.OUT_F32_NCHW)

    def forward(self, x):
        if self.training:
            if not x.is_cuda:
                raise NotImplementedError('DenseNet: training runs on the CUDA kernels only; the input is a CPU tensor')
            why = self.unsupported()
            if why is not None:
                raise NotImplementedError('DenseNet: no kernel path for %s' % why)
            if self.drop_rate > 0:
                raise NotImplementedError('DenseNet: drop_rate=%g: dense-layer dropout is not implemented in training' % self.drop_rate)
            return self.train_forward(x)
        return self.run(x)


def _pretrained(net, config_channels, name):
    """`[model] pretrained` (model/densenet.py:70-77): copy the torchvision ImageNet weights whose keys exist in this model (legacy
    torchvision-0.2 key names are renamed by the load hook)."""
    config = getattr(config_channels, 'config', None)
    if config is None or not config.getboolean('model', 'pretrained', fallback=False):
        return net
    import torchvision.models as tvm
    weights = getattr(tvm, 'DenseNet%s_Weights' % name[len('densenet'):]).IMAGENET1K_V1
    loaded = remap_legacy_keys(dict(weights.get_state_dict(progress=False)))
    state_dict = net.state_dict()
    for key, value in loaded.items():
        if key in state_dict:
            state_dict[key] = value
    net.load_state_dict(state_dict)
    return net


def densenet121(config_channels, anchors, num_cls, **kwargs):
    return _pretrained(DenseNet(config_channels, anchors, num_cls, 32, (6, 12, 24, 16), 64, **kwargs), config_channels, 'densenet121')


def densenet169(config_channels, anchors, num_cls, **kwargs):
    return _pretrained(DenseNet(config_channels, anchors, num_cls, 32, (6, 12, 32, 32), 64, **kwargs), config_channels, 'densenet169')


def densenet201(config_channels, anchors, num_cls, **kwargs):
    return _pretrained(DenseNet(config_channels, anchors, num_cls, 32, (6, 12, 48, 32), 64, **kwargs), config_channels, 'densenet201')


def densenet161(config_channels, anchors, num_cls, **kwargs):
    """Constructs with the reference's state_dict; its forward raises NotImplementedError (96-channel stem, 48-channel growth)."""
    return _pretrained(DenseNet(config_channels, anchors, num_cls, 48, (6, 12, 36, 24), 96, **kwargs), config_channels, 'densenet161')
