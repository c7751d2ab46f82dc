"""model.mobilenet -- MobileNet backbone plugin on the CUDA kernels (inference and training).

Drop-in for the reference's `model/mobilenet.py` (file:line cited per item): same constructor contract
`MobileNet(config_channels, anchors, num_cls)` (:56-77), same state_dict keys (`layers.0.conv.weight`,
`layers.N.dw.conv.weight`, `layers.N.pw.bn.running_var`, `layers.14.weight`, `layers.14.bias`), same forward
contract x[B,3,H,W] fp32 -> [B, A*(5+C), H/32, W/32] fp32 (:84-85).  Modules only hold parameters; the forward pass is:
  conv_bn(3,32,s2)   -> yb_mb_conv0_bn_relu_fwd  (fp32 NCHW image in, fp16 NHWC out)
  13 x conv_unit      -> yb_dwconv3x3_bn_relu_fwd (depthwise, HBM-bound) + wgmma 1x1 conv with fused BN + ReLU
  nn.Conv2d(1024, A*(5+C), 1) with bias -> wgmma 1x1 conv writing fp32 NCHW.
BatchNorm uses the PyTorch-default momentum 0.1 (unlike model.yolo2's 0.01) and the activation is ReLU (:28-29).

Two inference precisions, as for Darknet (`set_precision`, `[b200] precision` in the INI, YB_PRECISION): `fast` (fp16 operands, 1.4e-3 from
the fp32 reference after 27 layers) and `strict`: activations travel as [hi | lo] fp16 pairs, the pointwise convs and the head run the
split-precision wgmma kernel (operands [a_hi | a_lo | a_hi] x [w_hi | w_hi | w_lo] in one fp32 accumulator), the first conv and the depthwise
convs compute in fp32 on hi + lo -- within 1e-3 of the reference.
"""
import os
import collections

import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train


def conv_bn(in_channels, out_channels, stride):
    return nn.Sequential(collections.OrderedDict([
        ('conv', nn.Conv2d(in_channels, out_channels, 3, stride, 1, bias=False)),
        ('bn', nn.BatchNorm2d(out_channels)),
        ('act', nn.ReLU(inplace=True)),
    ]))


def conv_dw(in_channels, stride):
    return nn.Sequential(collections.OrderedDict([
        ('conv', nn.Conv2d(in_channels, in_channels, 3, stride, 1, groups=in_channels, bias=False)),
        ('bn', nn.BatchNorm2d(in_channels)),
        ('act', nn.ReLU(inplace=True)),
    ]))


def conv_pw(in_channels, out_channels):
    return nn.Sequential(collections.OrderedDict([
        ('conv', nn.Conv2d(in_channels, out_channels, 1, 1, 0, bias=False)),
        ('bn', nn.BatchNorm2d(out_channels)),
        ('act', nn.ReLU(inplace=True)),
    ]))


def conv_unit(in_channels, out_channels, stride):
    return nn.Sequential(collections.OrderedDict([
        ('dw', conv_dw(in_channels, stride)),
        ('pw', conv_pw(in_channels, out_channels)),
    ]))


UNITS = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1), (1024, 2), (1024, 1)]


class MobileNet(model.Backbone):
    TRAINER = _train.MobileNetTrainer

    def __init__(self, config_channels, anchors, num_cls):
        model.Backbone.__init__(self)
        cc = config_channels
        layers = [conv_bn(cc.channels, cc(32, 'layers.0.conv.weight'), 2)]
        for width, stride in UNITS:
            layers.append(conv_unit(cc.channels, cc(width, 'layers.%d.pw.conv.weight' % len(layers)), stride))
        layers.append(nn.Conv2d(cc.channels, model.output_channels(len(anchors), num_cls), 1))
        self.layers = nn.Sequential(*layers)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        config = getattr(config_channels, 'config', None)
        precision = os.environ.get('YB_PRECISION')
        if precision is None and config is not None and config.has_option('b200', 'precision'):
            precision = config.get('b200', 'precision')
        self.precision = 'fast'
        self.set_precision(precision or 'fast')

    def set_precision(self, precision):
        if precision not in ('fast', 'strict'):
            raise ValueError("precision must be 'fast' or 'strict', got %r" % (precision,))
        if precision != self.precision:
            self.drop_operands()
        self.precision = precision
        return self

    # ---- operand preparation (cached per parameter version) ------------------------------------------
    def _fold(self, key, bn):
        return self._cache.fetch(key, _engine.epilogue_tensors(bn), lambda: _engine.fold_epilogue(bn, None))

    def _packed(self, key, w):
        return self._cache.fetch(key, (w,), lambda: _ops.pack_weight_f16(w.detach().contiguous(), 0))

    def _packed_split(self, key, w):
        return self._cache.fetch(key, (w,), lambda: _ops.pack_weight_split_f16(w.detach().contiguous(), True, True))

    def _forward_strict(self, x, lut, shape):
        b, c, h, w = shape
        dev = x.device
        first = self.layers[0]
        scale, shift = self._fold('bn0', first.bn)
        ch = first.conv.weight.shape[0]
        cur = torch.empty(b, h // 2, w // 2, 2 * ch, dtype=torch.float16, device=dev)            # [hi | lo]
        if lut is None:
            _ops.call('yb_mb_conv0_split_fwd', x, first.conv.weight.detach().contiguous(), scale, shift, cur, b, h, w)
        else:
            _ops.call('yb_mb_conv0_split_lut_fwd', x, lut, first.conv.weight.detach().contiguous(), scale, shift, cur, b, h, w)
        hh, ww = h // 2, w // 2
        for i, unit in enumerate(list(self.layers)[1:-1], 1):
            dw, pw = unit.dw, unit.pw
            stride = dw.conv.stride[0]
            scale, shift = self._fold('dw%d' % i, dw.bn)
            out = torch.empty(b, hh // stride, ww // stride, 2 * ch, dtype=torch.float16, device=dev)
            _ops.call('yb_dwconv3x3_split_fwd', cur, dw.conv.weight.detach().contiguous().view(ch, 9), scale, shift, out, b, hh, ww, ch, stride)
            hh, ww = hh // stride, ww // stride
            scale, shift = self._fold('pw%d' % i, pw.bn)
            cout = pw.conv.weight.shape[0]
            cur = torch.empty(b, hh, ww, 2 * cout, dtype=torch.float16, device=dev)
            _ops.conv_bn_act_split(out, self._packed_split('pws%d' % i, pw.conv.weight), scale, shift, 0.0, cur, a_channels=2 * ch, lo_ch_off=cout)
            ch = cout
        head = self.layers[-1]
        cout = head.weight.shape[0]
        ones = torch.ones(cout, dtype=torch.float32, device=dev)
        feature = torch.empty(b, cout, hh, ww, dtype=torch.float32, device=dev)
        _ops.conv_bn_act_split(cur, self._packed_split('heads', head.weight), ones, head.bias.detach().float().contiguous(), 1.0, feature,
                               a_channels=2 * ch, out_mode=_ops.OUT_F32_NCHW)
        return feature

    def forward(self, x):
        if self.training:
            return self.train_forward(x)
        if not x.is_cuda:
            raise RuntimeError('MobileNet: input must be a CUDA tensor; there is no CPU fallback')
        x, lut, shape = self.eval_input(x)
        b, c, h, w = shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('MobileNet expects [B,3,H,W] with H, W multiples of 32')
        first = self.layers[0]
        if first.conv.weight.shape[0] != 32:
            raise ValueError('MobileNet: the first layer must have 32 output channels')
        if self.precision == 'strict':
            return self._forward_strict(x, lut, shape)
        scale, shift = self._fold('bn0', first.bn)
        cur = torch.empty(b, h // 2, w // 2, first.conv.weight.shape[0], dtype=torch.float16, device=x.device)
        if lut is None:
            _ops.call('yb_mb_conv0_bn_relu_fwd', x, first.conv.weight.detach().contiguous(), scale, shift, cur, b, h, w)
        else:
            _ops.call('yb_mb_conv0_bn_relu_lut_fwd', x, lut, first.conv.weight.detach().contiguous(), scale, shift, cur, b, h, w)
        hh, ww = h // 2, w // 2
        for i, unit in enumerate(list(self.layers)[1:-1], 1):
            dw, pw = unit.dw, unit.pw
            ch = dw.conv.weight.shape[0]
            stride = dw.conv.stride[0]
            scale, shift = self._fold('dw%d' % i, dw.bn)
            out = torch.empty(b, hh // stride, ww // stride, ch, dtype=torch.float16, device=x.device)
            _ops.call('yb_dwconv3x3_bn_relu_fwd', cur, dw.conv.weight.detach().contiguous().view(ch, 9), scale, shift, out, b, hh, ww, ch, stride)
            hh, ww = hh // stride, ww // stride
            scale, shift = self._fold('pw%d' % i, pw.bn)
            cur = _ops.conv_bn_act(out, self._packed('pww%d' % i, pw.conv.weight), scale, shift, 0.0)      # slope 0 == ReLU
        head = self.layers[-1]
        cout = head.weight.shape[0]
        ones = self._cache.fetch('ones', (), lambda: torch.ones(cout, dtype=torch.float32, device=x.device), extra=(cout, x.device))
        return _ops.conv_bn_act(cur, self._packed('head', head.weight), ones, head.bias.detach().float().contiguous(), 1.0,
                                out_mode=_ops.OUT_F32_NCHW)
