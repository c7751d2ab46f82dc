"""model.resnet -- ResNet backbone plugin on the CUDA kernels (inference and training).

Drop-in for the reference's `model/resnet.py` (file:line cited per item): same constructors `resnet18 / resnet34 / resnet50
(config_channels, anchors, num_cls)` (:161-197), same state_dict keys as torchvision's ResNet (`conv1.weight`, `bn1.*`,
`layerL.B.conv1.weight`, `layerL.B.downsample.0.weight`, ...) plus the 1x1 detection head `conv.weight / conv.bias` (:115), same
`scope(name)` (:144-158), same forward contract x[B,3,H,W] fp32 -> [B, A*(5+C), H/32, W/32] fp32 (:131-142).  Modules only hold
parameters; the forward pass is:
  conv1 7x7 s2 + bn1 + relu      -> yb_stem7x7_bn_relu_fwd   (fp32 NCHW image in, fp16 NHWC out)
  maxpool 3x3 s2 p1              -> yb_maxpool3x3_s2_f16
  3x3 / 1x1 conv + bn (+ relu)   -> wgmma implicit-GEMM conv with the folded BatchNorm in its epilogue (slope 0 = ReLU, 1 = none)
  stride-2 3x3 conv              -> the same kernel at stride 1, then yb_subsample2_f16 (a padded stride-2 conv IS its stride-1
                                    form at the even pixels); stride-2 1x1 downsample -> yb_subsample2_f16, then the 1x1 conv
  out += residual; relu          -> yb_add_relu_f16
  nn.Conv2d(C, A*(5+C), 1) + bias-> wgmma 1x1 conv writing fp32 NCHW.
In train() mode the forward is one autograd node (model._TrainFunction) over b200.train_engine.ResNetTrainer: batch-statistics
BatchNorm (momentum 0.1, read from the modules) on the raw conv outputs, the explicit backward chain (stride-2 convs as the stride-1 gradients of the
zero-inserted dz, max-pool backward to the first maximum of each window, the stem's weight gradient on the fp32 image).  There is no CPU path.
Switching back to eval() drops the cached folded BatchNorm and packed weights, so inference uses the trained state.
"""
import re

import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train


def conv3x3(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


def _downsample(channels_in, channels_out, stride):
    return nn.Sequential(nn.Conv2d(channels_in, channels_out, kernel_size=1, stride=stride, bias=False), nn.BatchNorm2d(channels_out))


class BasicBlock(nn.Module):
    """Two 3x3 convs (model/resnet.py:28-61).  Parameter container; `units()` lists (conv, bn, relu?) in execution order."""
    def __init__(self, config_channels, prefix, channels, stride=1):
        nn.Module.__init__(self)
        cc = config_channels
        channels_in = cc.channels
        self.conv1 = conv3x3(cc.channels, cc(channels, '%s.conv1.weight' % prefix), stride)
        self.bn1 = nn.BatchNorm2d(cc.channels)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(cc.channels, cc(channels, '%s.conv2.weight' % prefix))
        self.bn2 = nn.BatchNorm2d(cc.channels)
        self.downsample = _downsample(channels_in, cc.channels, stride) if (stride > 1 or channels_in != cc.channels) else None

    def units(self):
        return [('conv1', self.conv1, self.bn1, True), ('conv2', self.conv2, self.bn2, False)]


class Bottleneck(nn.Module):
    """1x1 -> 3x3 (strided) -> 1x1 x4 (model/resnet.py:64-103)."""
    def __init__(self, config_channels, prefix, channels, stride=1):
        nn.Module.__init__(self)
        cc = config_channels
        channels_in = cc.channels
        self.conv1 = nn.Conv2d(cc.channels, cc(channels, '%s.conv1.weight' % prefix), kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(cc.channels)
        self.conv2 = nn.Conv2d(cc.channels, cc(channels, '%s.conv2.weight' % prefix), kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(cc.channels)
        self.conv3 = nn.Conv2d(cc.channels, cc(channels * 4, '%s.conv3.weight' % prefix), kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(cc.channels)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = _downsample(channels_in, cc.channels, stride) if (stride > 1 or channels_in != cc.channels) else None

    def units(self):
        return [('conv1', self.conv1, self.bn1, True), ('conv2', self.conv2, self.bn2, True), ('conv3', self.conv3, self.bn3, False)]


class ResNet(model.Backbone):
    TRAINER = _train.ResNetTrainer

    def __init__(self, config_channels, anchors, num_cls, block, layers):
        model.Backbone.__init__(self)
        cc = config_channels
        self.conv1 = nn.Conv2d(cc.channels, cc(64, 'conv1.weight'), kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(cc.channels)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(cc, 'layer1', block, 64, layers[0])
        self.layer2 = self._make_layer(cc, 'layer2', block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(cc, 'layer3', block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(cc, 'layer4', block, 512, layers[3], stride=2)
        self.conv = nn.Conv2d(cc.channels, model.output_channels(len(anchors), num_cls), 1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def _make_layer(self, config_channels, prefix, block, channels, blocks, stride=1):
        seq = [block(config_channels, '%s.0' % prefix, channels, stride)]
        for i in range(1, blocks):
            seq.append(block(config_channels, '%s.%d' % (prefix, i), channels))
        return nn.Sequential(*seq)

    def scope(self, name):
        """Parameter name -> the unit it belongs to ('layer1.0.conv1.weight' -> 'layer1.0.1'), as model/resnet.py:144-158."""
        comp = name.split('.')[:-1]
        m = re.search(r'[(conv)|(bn)](\d+)', comp[-1])
        if m is not None:
            comp[-1] = m.group(1)
        elif len(comp) > 1:
            assert comp[-2] == 'downsample', name
            comp = comp[:-1]
        else:
            assert comp[-1] == 'conv', name
        return '.'.join(comp)

    # ---- operand preparation (cached per parameter version) ------------------------------------------
    def _fold(self, key, bn):
        return self._cache.fetch(key, _engine.epilogue_tensors(bn), lambda: _engine.fold_epilogue(bn, None))

    def _packed(self, key, w):
        return self._cache.fetch(key, (w,), lambda: _ops.pack_weight_f16(w.detach().contiguous(), 0))

    @staticmethod
    def _subsample(x):
        b, h, w, c = x.shape
        out = torch.empty(b, (h + 1) // 2, (w + 1) // 2, c, dtype=torch.float16, device=x.device)
        _ops.call('yb_subsample2_f16', x, out, b, h, w, c)
        return out

    def _unit(self, key, x, conv, bn, relu):
        """conv (stride 1 or 2) + folded bn + optional relu on fp16 NHWC."""
        stride, k = conv.stride[0], conv.kernel_size[0]
        if stride == 2 and k == 1:
            x = self._subsample(x)
        scale, shift = self._fold(key + '.bn', bn)
        y = _ops.conv_bn_act(x, self._packed(key + '.w', conv.weight), scale, shift, 0.0 if relu else 1.0)
        if stride == 2 and k == 3:
            y = self._subsample(y)
        return y

    def _block(self, prefix, blk, x):
        out = x
        for name, conv, bn, relu in blk.units():
            out = self._unit('%s.%s' % (prefix, name), out, conv, bn, relu)
        residual = x if blk.downsample is None else self._unit(prefix + '.downsample', x, blk.downsample[0], blk.downsample[1], False)
        _ops.call('yb_add_relu_f16', out, residual, out, out.numel())
        return out

    def forward(self, x):
        if self.training:
            if not x.is_cuda:
                raise NotImplementedError('ResNet training: no CPU path, input must be a CUDA tensor')
            return self.train_forward(x)
        if not x.is_cuda:
            raise RuntimeError('ResNet: input must be a CUDA tensor; there is no CPU fallback')
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('ResNet expects [B,3,H,W] with H, W multiples of 32')
        if self.conv1.weight.shape[0] != 64:
            raise ValueError('ResNet: the stem must have 64 output channels')
        x = x.contiguous().float()
        scale, shift = self._fold('bn1', self.bn1)
        stem = torch.empty(b, h // 2, w // 2, 64, dtype=torch.float16, device=x.device)
        _ops.call('yb_stem7x7_bn_relu_fwd', x, self.conv1.weight.detach().contiguous(), scale, shift, stem, b, h, w)
        cur = torch.empty(b, h // 4, w // 4, 64, dtype=torch.float16, device=x.device)
        _ops.call('yb_maxpool3x3_s2_f16', stem, cur, b, h // 2, w // 2, 64)
        for lname in ('layer1', 'layer2', 'layer3', 'layer4'):
            for bname, blk in getattr(self, lname).named_children():
                cur = self._block('%s.%s' % (lname, bname), blk, cur)
        cout = self.conv.weight.shape[0]
        ones = self._cache.fetch('ones', (), lambda: torch.ones(cout, dtype=torch.float32, device=x.device), extra=(cout, x.device))
        return _ops.conv_bn_act(cur, self._packed('head', self.conv.weight), ones, self.conv.bias.detach().float().contiguous(), 1.0,
                                out_mode=_ops.OUT_F32_NCHW)


def _pretrained(net, config_channels, name):
    """`[model] pretrained` (model/resnet.py:163-171): copy the torchvision ImageNet weights whose keys exist in this model."""
    config = getattr(config_channels, 'config', None)
    if config is None or not config.getboolean('model', 'pretrained', fallback=False):
        return net
    import torchvision.models as tvm
    weights = getattr(tvm, 'ResNet%s_Weights' % name[len('resnet'):]).IMAGENET1K_V1
    state_dict = net.state_dict()
    for key, value in weights.get_state_dict(progress=False).items():
        if key in state_dict:
            state_dict[key] = value
    net.load_state_dict(state_dict)
    return net


def resnet18(config_channels, anchors, num_cls, **kwargs):
    return _pretrained(ResNet(config_channels, anchors, num_cls, BasicBlock, [2, 2, 2, 2], **kwargs), config_channels, 'resnet18')


def resnet34(config_channels, anchors, num_cls, **kwargs):
    return _pretrained(ResNet(config_channels, anchors, num_cls, BasicBlock, [3, 4, 6, 3], **kwargs), config_channels, 'resnet34')


def resnet50(config_channels, anchors, num_cls, **kwargs):
    return _pretrained(ResNet(config_channels, anchors, num_cls, Bottleneck, [3, 4, 6, 3], **kwargs), config_channels, 'resnet50')
