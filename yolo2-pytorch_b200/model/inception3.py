"""model.inception3 -- Inception-v3 backbone plugin on the CUDA kernels (inference and training).

Drop-in for the reference's `model/inception3.py` (:29-118): `Inception3(config_channels, anchors, num_cls, transform_input=False)`, selectable
with `[model] dnn = model.inception3.Inception3`, with the module tree and state_dict keys of the reference (torchvision's `BasicConv2d` =
conv without bias + BatchNorm (eps 1e-3) + ReLU, and `InceptionA`..`InceptionE`, under `Conv2d_1a_3x3` .. `Mixed_7c`) plus the 1x1 detection
head `conv` (:52).  Forward x[B,3,H,W] fp32 -> [B, A*(5+C), OH, OW] fp32, where OH, OW follow the reference's valid convs and pools
(416 -> 11, 320 -> 8, 608 -> 17, 75 -> 1; below 75 a stage is empty).  Modules only hold parameters; the forward pass runs in fp16 NHWC:
  Conv2d_1a_3x3 (3 -> 32, s2, no pad)   -> yb_stem3x3_s2_bn_relu_fwd
  every other BasicConv2d               -> yb_conv2d_bn_act_fwd (kh x kw, stride 1 / 2, padding as the module's), BatchNorm folded into the
                                           epilogue, ReLU; each branch writes its own channel range of its block's buffer (no torch.cat)
  F.max_pool2d(3, stride=2)             -> yb_maxpool3x3_s2_valid_f16 (the stem pools; the pool branch of Mixed_6a / 7a straight into the
                                           block buffer)
  F.avg_pool2d(3, 1, 1) of branch_pool  -> yb_avgpool3x3_s1_f16 (count_include_pad, divisor 9), then the 1x1 conv
  conv (+ bias)                         -> yb_conv2d_bn_act_fwd, fp32 NCHW out.
The tensor-core conv needs Cin % 32 == 0: Conv2d_3b_1x1 (80 filters) and branch5x5_1 (48) run with 96 / 64 filters whose extra rows are zero
(scale 1, shift 0: ReLU stores exact zeros) and their consumers read those channels with zero weights -- exact, no kernel change.
The folded BatchNorms and packed weights are cached per parameter version; switching train() / eval() drops the cache.
In train() mode on a CUDA tensor the forward is one autograd node (model._TrainFunction) over
b200.train_engine.InceptionTrainer: batch-statistics BatchNorm (eps 1e-3, momentum from the module), the running-statistics update, and an
explicit backward chain that gives every parameter its fp32 gradient.  There is no CPU path: a train-mode forward on a CPU tensor raises
NotImplementedError, an eval-mode one RuntimeError.
"""
import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train

MIN_SIZE = 75      # the smallest input side whose every stage is non-empty (Mixed_7a's output is 1 x 1)


def _round32(c):
    return (c + 31) // 32 * 32


class BasicConv2d(nn.Module):
    """torchvision.models.inception.BasicConv2d: conv (no bias) -> BatchNorm2d(eps=0.001) -> ReLU."""

    def __init__(self, in_channels, out_channels, **kwargs):
        nn.Module.__init__(self)
        self.conv = nn.Conv2d(in_channels, out_channels, bias=False, **kwargs)
        self.bn = nn.BatchNorm2d(out_channels, eps=0.001)


class InceptionA(nn.Module):
    def __init__(self, in_channels, pool_features):
        nn.Module.__init__(self)
        self.branch1x1 = BasicConv2d(in_channels, 64, kernel_size=1)
        self.branch5x5_1 = BasicConv2d(in_channels, 48, kernel_size=1)
        self.branch5x5_2 = BasicConv2d(48, 64, kernel_size=5, padding=2)
        self.branch3x3dbl_1 = BasicConv2d(in_channels, 64, kernel_size=1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, kernel_size=3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, kernel_size=3, padding=1)
        self.branch_pool = BasicConv2d(in_channels, pool_features, kernel_size=1)


class InceptionB(nn.Module):
    def __init__(self, in_channels):
        nn.Module.__init__(self)
        self.branch3x3 = BasicConv2d(in_channels, 384, kernel_size=3, stride=2)
        self.branch3x3dbl_1 = BasicConv2d(in_channels, 64, kernel_size=1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, kernel_size=3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, kernel_size=3, stride=2)


class InceptionC(nn.Module):
    def __init__(self, in_channels, channels_7x7):
        nn.Module.__init__(self)
        c7 = channels_7x7
        self.branch1x1 = BasicConv2d(in_channels, 192, kernel_size=1)
        self.branch7x7_1 = BasicConv2d(in_channels, c7, kernel_size=1)
        self.branch7x7_2 = BasicConv2d(c7, c7, kernel_size=(1, 7), padding=(0, 3))
        self.branch7x7_3 = BasicConv2d(c7, 192, kernel_size=(7, 1), padding=(3, 0))
        self.branch7x7dbl_1 = BasicConv2d(in_channels, c7, kernel_size=1)
        self.branch7x7dbl_2 = BasicConv2d(c7, c7, kernel_size=(7, 1), padding=(3, 0))
        self.branch7x7dbl_3 = BasicConv2d(c7, c7, kernel_size=(1, 7), padding=(0, 3))
        self.branch7x7dbl_4 = BasicConv2d(c7, c7, kernel_size=(7, 1), padding=(3, 0))
        self.branch7x7dbl_5 = BasicConv2d(c7, 192, kernel_size=(1, 7), padding=(0, 3))
        self.branch_pool = BasicConv2d(in_channels, 192, kernel_size=1)


class InceptionD(nn.Module):
    def __init__(self, in_channels):
        nn.Module.__init__(self)
        self.branch3x3_1 = BasicConv2d(in_channels, 192, kernel_size=1)
        self.branch3x3_2 = BasicConv2d(192, 320, kernel_size=3, stride=2)
        self.branch7x7x3_1 = BasicConv2d(in_channels, 192, kernel_size=1)
        self.branch7x7x3_2 = BasicConv2d(192, 192, kernel_size=(1, 7), padding=(0, 3))
        self.branch7x7x3_3 = BasicConv2d(192, 192, kernel_size=(7, 1), padding=(3, 0))
        self.branch7x7x3_4 = BasicConv2d(192, 192, kernel_size=3, stride=2)


class InceptionE(nn.Module):
    def __init__(self, in_channels):
        nn.Module.__init__(self)
        self.branch1x1 = BasicConv2d(in_channels, 320, kernel_size=1)
        self.branch3x3_1 = BasicConv2d(in_channels, 384, kernel_size=1)
        self.branch3x3_2a = BasicConv2d(384, 384, kernel_size=(1, 3), padding=(0, 1))
        self.branch3x3_2b = BasicConv2d(384, 384, kernel_size=(3, 1), padding=(1, 0))
        self.branch3x3dbl_1 = BasicConv2d(in_channels, 448, kernel_size=1)
        self.branch3x3dbl_2 = BasicConv2d(448, 384, kernel_size=3, padding=1)
        self.branch3x3dbl_3a = BasicConv2d(384, 384, kernel_size=(1, 3), padding=(0, 1))
        self.branch3x3dbl_3b = BasicConv2d(384, 384, kernel_size=(3, 1), padding=(1, 0))
        self.branch_pool = BasicConv2d(in_channels, 192, kernel_size=1)


BLOCKS = ('Mixed_5b', 'Mixed_5c', 'Mixed_5d', 'Mixed_6a', 'Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e', 'Mixed_7a', 'Mixed_7b', 'Mixed_7c')


class Inception3(model.Backbone):
    TRAINER = _train.InceptionTrainer

    def __init__(self, config_channels, anchors, num_cls, transform_input=False):
        model.Backbone.__init__(self)
        self.transform_input = transform_input
        self.Conv2d_1a_3x3 = BasicConv2d(3, 32, kernel_size=3, stride=2)
        self.Conv2d_2a_3x3 = BasicConv2d(32, 32, kernel_size=3)
        self.Conv2d_2b_3x3 = BasicConv2d(32, 64, kernel_size=3, padding=1)
        self.Conv2d_3b_1x1 = BasicConv2d(64, 80, kernel_size=1)
        self.Conv2d_4a_3x3 = BasicConv2d(80, 192, kernel_size=3)
        self.Mixed_5b = InceptionA(192, pool_features=32)
        self.Mixed_5c = InceptionA(256, pool_features=64)
        self.Mixed_5d = InceptionA(288, pool_features=64)
        self.Mixed_6a = InceptionB(288)
        self.Mixed_6b = InceptionC(768, channels_7x7=128)
        self.Mixed_6c = InceptionC(768, channels_7x7=160)
        self.Mixed_6d = InceptionC(768, channels_7x7=160)
        self.Mixed_6e = InceptionC(768, channels_7x7=192)
        self.Mixed_7a = InceptionD(768)
        self.Mixed_7b = InceptionE(1280)
        self.Mixed_7c = InceptionE(2048)
        self.conv = nn.Conv2d(2048, model.output_channels(len(anchors), num_cls), 1)
        # model/inception3.py:54-62: truncated normal over +-2 sigma with sigma = 0.1 for every conv, BatchNorm weight 1 and bias 0
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                with torch.no_grad():
                    nn.init.trunc_normal_(m.weight, std=0.1, a=-0.2, b=0.2)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        _pretrained(self, config_channels)

    # ---- operand preparation (cached per parameter version) ------------------------------------------
    def _operands(self, unit, cin_pad):
        """Folded BatchNorm (scale, shift) padded to the 32-rounded filter count with (1, 0), and the packed fp16 weight with zero filters and
        zero input channels up to (cout_pad, cin_pad)."""
        w, bn = unit.conv.weight, unit.bn
        cout_pad = _round32(w.shape[0])

        def build():
            s, t = _engine.fold_epilogue(bn, None, cout_pad)
            return _ops.pack_weight_khw_f16(w.detach().float().contiguous(), cout_pad, cin_pad), s, t
        return self._cache.fetch(unit, (w,) + _engine.epilogue_tensors(bn), build, extra=(cin_pad,))

    def _head(self):
        w, b = self.conv.weight, self.conv.bias
        return self._cache.fetch('head', (w, b), lambda: (_ops.pack_weight_khw_f16(w.detach().float().contiguous()),
                                                          torch.ones(w.shape[0], dtype=torch.float32, device=w.device), b.detach().float().contiguous()))

    # ---- units -----------------------------------------------------------------------------------------
    def unit(self, unit, x, out=None, y_ch_off=0):
        """One BasicConv2d on x (fp16 NHWC, all of its channels; zero weights for any beyond the module's Cin): into channels [y_ch_off,
        y_ch_off + Cout) of `out`, or a new tensor of the 32-rounded width."""
        conv = unit.conv
        w16, s, t = self._operands(unit, x.shape[-1])
        return _ops.conv2d_bn_act(x, w16, s, t, 0.0, stride=conv.stride[0], pad=conv.padding, out=out, y_ch_off=y_ch_off)

    def _new(self, x, h, w, c):
        return torch.empty(x.shape[0], h, w, c, dtype=torch.float16, device=x.device)

    def block_a(self, m, x):
        b, h, w, c = x.shape
        out = self._new(x, h, w, 224 + m.branch_pool.conv.out_channels)
        self.unit(m.branch1x1, x, out, 0)
        self.unit(m.branch5x5_2, self.unit(m.branch5x5_1, x), out, 64)
        self.unit(m.branch3x3dbl_3, self.unit(m.branch3x3dbl_2, self.unit(m.branch3x3dbl_1, x)), out, 128)
        self.unit(m.branch_pool, _ops.avgpool3x3_s1(x), out, 224)
        return out

    def block_b(self, m, x):
        b, h, w, c = x.shape
        oh, ow = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        out = self._new(x, oh, ow, 480 + c)
        self.unit(m.branch3x3, x, out, 0)
        self.unit(m.branch3x3dbl_3, self.unit(m.branch3x3dbl_2, self.unit(m.branch3x3dbl_1, x)), out, 384)
        _ops.maxpool3x3_s2_valid(x, out, 480)
        return out

    def block_c(self, m, x):
        b, h, w, c = x.shape
        out = self._new(x, h, w, 768)
        self.unit(m.branch1x1, x, out, 0)
        self.unit(m.branch7x7_3, self.unit(m.branch7x7_2, self.unit(m.branch7x7_1, x)), out, 192)
        y = self.unit(m.branch7x7dbl_1, x)
        for u in (m.branch7x7dbl_2, m.branch7x7dbl_3, m.branch7x7dbl_4):
            y = self.unit(u, y)
        self.unit(m.branch7x7dbl_5, y, out, 384)
        self.unit(m.branch_pool, _ops.avgpool3x3_s1(x), out, 576)
        return out

    def block_d(self, m, x):
        b, h, w, c = x.shape
        oh, ow = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        out = self._new(x, oh, ow, 512 + c)
        self.unit(m.branch3x3_2, self.unit(m.branch3x3_1, x), out, 0)
        y = self.unit(m.branch7x7x3_3, self.unit(m.branch7x7x3_2, self.unit(m.branch7x7x3_1, x)))
        self.unit(m.branch7x7x3_4, y, out, 320)
        _ops.maxpool3x3_s2_valid(x, out, 512)
        return out

    def block_e(self, m, x):
        b, h, w, c = x.shape
        out = self._new(x, h, w, 2048)
        self.unit(m.branch1x1, x, out, 0)
        y = self.unit(m.branch3x3_1, x)
        self.unit(m.branch3x3_2a, y, out, 320)
        self.unit(m.branch3x3_2b, y, out, 704)
        y = self.unit(m.branch3x3dbl_2, self.unit(m.branch3x3dbl_1, x))
        self.unit(m.branch3x3dbl_3a, y, out, 1088)
        self.unit(m.branch3x3dbl_3b, y, out, 1472)
        self.unit(m.branch_pool, _ops.avgpool3x3_s1(x), out, 1856)
        return out

    def block(self, name, x):
        """Mixed_* block `name` on x (fp16 NHWC): its concatenated output (fp16 NHWC)."""
        kind = {'5': self.block_a, '6a': self.block_b, '6': self.block_c, '7a': self.block_d, '7': self.block_e}
        tag = name[len('Mixed_'):]
        fn = kind.get(tag) or kind[tag[0]]
        return fn(getattr(self, name), x)

    def stem(self, x, collect=None):
        """Conv2d_1a_3x3 .. the second max-pool: x fp32 NCHW -> Mixed_5b's input, fp16 NHWC [B,H5,W5,192]."""
        s, t = self._operands_stem()
        a = _ops.stem3x3_s2(x, self.Conv2d_1a_3x3.conv.weight.detach().float().contiguous(), s, t, pad=0)
        a = self.unit(self.Conv2d_2b_3x3, self.unit(self.Conv2d_2a_3x3, a))
        a = _ops.maxpool3x3_s2_valid(a)
        if collect is not None:
            collect['pool1'] = a
        a = self.unit(self.Conv2d_4a_3x3, self.unit(self.Conv2d_3b_1x1, a))
        a = _ops.maxpool3x3_s2_valid(a)
        if collect is not None:
            collect['pool2'] = a
        return a

    def _operands_stem(self):
        bn = self.Conv2d_1a_3x3.bn
        return self._cache.fetch('stem', _engine.epilogue_tensors(bn), lambda: _engine.fold_epilogue(bn, None))

    def run(self, x, collect=None):
        """Forward on the kernels; `collect` (a dict) receives both stem pools and every Mixed_* output (fp16 NHWC)."""
        b, c, h, w = x.shape
        if c != 3:
            raise ValueError('Inception3 expects [B,3,H,W]')
        if h < MIN_SIZE or w < MIN_SIZE:
            raise ValueError('Inception3: a %d x %d input leaves a stage empty (H and W must be >= %d)' % (h, w, MIN_SIZE))
        if not x.is_cuda:
            raise RuntimeError('Inception3: input must be a CUDA tensor; there is no CPU fallback')
        a = self.stem(x.contiguous().float(), collect)
        for name in BLOCKS:
            a = self.block(name, a)
            if collect is not None:
                collect[name] = a
        w16, one, bias = self._head()
        return _ops.conv2d_bn_act(a, w16, one, bias, 1.0, out_mode=_ops.OUT_F32_NCHW)

    def forward(self, x):
        if self.transform_input:
            raise NotImplementedError('Inception3: transform_input=True has no kernel path (the reference never sets it)')
        if self.training:
            if not x.is_cuda:
                raise NotImplementedError('Inception3: training runs on the CUDA kernels only; the input is a CPU tensor')
            return self.train_forward(x)
        return self.run(x)


def _pretrained(net, config_channels):
    """`[model] pretrained` (model/inception3.py:64-71): copy the torchvision ImageNet weights whose keys exist in this model."""
    config = getattr(config_channels, 'config', None)
    if config is None or not config.getboolean('model', 'pretrained', fallback=False):
        return net
    import torchvision.models as tvm
    loaded = tvm.Inception_V3_Weights.IMAGENET1K_V1.get_state_dict(progress=False)
    state_dict = net.state_dict()
    for key, value in loaded.items():
        if key in state_dict:
            state_dict[key] = value
    net.load_state_dict(state_dict)
    return net
