"""model.yolo2 -- Darknet-19 backbone plugin, H100-native.

Drop-in for the plugin surface of ruiminshen/yolo2-pytorch `model/yolo2.py` (reference file:line
cited per item): same constructor contract `Darknet(config_channels, anchors, num_cls, stride=2,
ratio=1)` (:69), same `forward(x[B,3,H,W] fp32) -> [B, A*(5+C), H/32, W/32] fp32` (:125-130), same
state_dict key names (`layers1.N.conv.weight`, `layers1.N.bn.running_mean`, `passthrough.*`,
`layers3.1.conv.bias`, ...), `init()` (:117-123), `scope()` (:132-133), `get_mapper()` (:135-137) and
the module-level `reorg()` (:33-46).

The modules here only HOLD parameters (so `.cuda()`, `.state_dict()`, `load_state_dict()`,
`.parameters()` and torch.optim work unchanged).  No torch.nn forward is ever executed: the forward
pass is the kernel chain in b200.engine (wgmma implicit-GEMM convs with fused BN + leaky-ReLU,
fp16 NHWC activations, in-place concat).  There is no CPU fallback.
"""
import torch
import torch.nn as nn

import model
from b200 import engine as _engine
from b200 import ops as _ops
from b200 import train_engine as _train

settings = {
    'size': (416, 416),
}


def reorg(x, stride_h=2, stride_w=2):
    """Space-to-depth with offset-major channel order: out[b,(sh*stride_w+sw)*C+c,h',w'] =
    x[b,c,h'*stride_h+sh,w'*stride_w+sw]  (reference model/yolo2.py:33-46), one CUDA kernel."""
    return _ops.reorg_f32_nchw(x.contiguous().float(), stride_h, stride_w)


class MaxPool2d(nn.Module):
    """Placeholder that keeps the reference's nn.Sequential indices (model/yolo2.py:79,86,97); the
    2x2 pooling itself runs inside the engine (fused into the first conv, or yb_maxpool2x2_f16)."""
    is_pool = True

    def __init__(self, kernel_size=2):
        nn.Module.__init__(self)
        if kernel_size != 2:
            raise ValueError('only MaxPool2d(2) is on the Darknet path')
        self.kernel_size = kernel_size

    def forward(self, x):
        y = _ops.maxpool2x2(x.permute(0, 2, 3, 1).contiguous().half())
        return y.permute(0, 3, 1, 2).float()


class Conv2d(nn.Module):
    """Parameter holder for conv(k, stride 1, pad (k-1)//2, bias = not bn) -> BatchNorm2d(momentum
    0.01) -> LeakyReLU(0.1)  (reference model/yolo2.py:49-65)."""
    is_pool = False

    def __init__(self, in_channels, out_channels, kernel_size, padding=0, stride=1, bn=True, act=True):
        nn.Module.__init__(self)
        if isinstance(padding, bool):
            padding = (kernel_size - 1) // 2 if padding else 0
        if stride != 1 or padding != (kernel_size - 1) // 2 or kernel_size not in (1, 3):
            raise ValueError('Conv2d supports k in {1,3}, stride 1, "same" padding (got k=%d stride=%d pad=%d)'
                             % (kernel_size, stride, padding))
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding=padding, bias=not bn)
        self.has_bn, self.has_act = bool(bn), bool(act)
        if bn:
            self.bn = nn.BatchNorm2d(out_channels, momentum=0.01)
        self._unit = None

    def forward(self, x):
        """Stand-alone use of one unit on an fp32 NCHW tensor (tests, pruning tools).  Layout/dtype
        conversion at this boundary is plain data movement; the conv runs on the wgmma kernel."""
        if self.training and self.has_bn:
            raise NotImplementedError('a stand-alone Conv2d unit runs in eval mode only; training goes through Darknet.forward (b200.train_engine)')
        if self._unit is None:
            self._unit = _engine.ConvUnit(self.conv, self.bn if self.has_bn else None, self.has_act)
        u = self._unit
        if u.cin % 32 != 0:
            raise ValueError('stand-alone Conv2d needs Cin %% 32 == 0 (the 3-channel first layer is fused in Darknet.forward)')
        u.refresh()
        y = _ops.conv_bn_act(x.permute(0, 2, 3, 1).contiguous().half(), u.w16, u.scale, u.shift, u.slope, out_mode=_ops.OUT_F32_NCHW)
        return y


class Darknet(model.Backbone):
    TRAINER = _train.DarknetTrainer

    def __init__(self, config_channels, anchors, num_cls, stride=2, ratio=1):
        model.Backbone.__init__(self)
        if stride != 2:
            raise ValueError('Darknet: passthrough stride must be 2')
        self.stride = stride
        bn = config_channels.config.getboolean('batch_norm', 'enable')
        cc = config_channels

        def unit(group, seq, width, k):
            seq.append(Conv2d(cc.channels, cc(width, '%s.%d.conv.weight' % (group, len(seq))), k, bn=bn, padding=True))

        # layers1: C32 P C64 P | C128 c64 C128 P | C256 c128 C256 P | C512 c256 C512 c256 C512
        width = int(32 * ratio)
        seq = []
        for _ in range(2):
            unit('layers1', seq, width, 3)
            seq.append(MaxPool2d(2))
            width *= 2
        for _ in range(2):
            unit('layers1', seq, width, 3)
            unit('layers1', seq, width // 2, 1)
            unit('layers1', seq, width, 3)
            seq.append(MaxPool2d(2))
            width *= 2
        for _ in range(2):
            unit('layers1', seq, width, 3)
            unit('layers1', seq, width // 2, 1)
        unit('layers1', seq, width, 3)
        self.layers1 = nn.Sequential(*seq)
        c_trunk16 = cc.channels

        # layers2: P C1024 c512 C1024 c512 C1024 C1024 C1024
        width *= 2
        seq = [MaxPool2d(2)]
        for _ in range(2):
            unit('layers2', seq, width, 3)
            unit('layers2', seq, width // 2, 1)
        for _ in range(3):
            unit('layers2', seq, width, 3)
        self.layers2 = nn.Sequential(*seq)
        c_trunk32 = cc.channels

        self.passthrough = Conv2d(c_trunk16, cc(int(64 * ratio), 'passthrough.conv.weight'), 1, bn=bn)
        c_cat = cc.channels * stride * stride + c_trunk32

        seq = [Conv2d(c_cat, cc(int(1024 * ratio), 'layers3.0.conv.weight'), 3, bn=bn, padding=True)]
        seq.append(Conv2d(cc.channels, model.output_channels(len(anchors), num_cls), 1, bn=False, act=False))
        self.layers3 = nn.Sequential(*seq)

        self.init()
        self._engine = None
        # optional `[b200] precision = fast | strict` in the INI (not a reference key): see b200.engine.DarknetEngine.set_precision
        cfg = config_channels.config
        self._precision = cfg.get('b200', 'precision') if cfg.has_option('b200', 'precision') else None

    def init(self):
        """kaiming-normal conv weights, BN gamma = 1, beta = 0 (reference model/yolo2.py:117-123)."""
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    @property
    def engine(self):
        if self._engine is None:
            self._engine = _engine.DarknetEngine(self)
            if self._precision is not None:
                self._engine.set_precision(self._precision)
        return self._engine

    @property
    def trainer(self):
        padded = self.engine.padded_unit()
        if padded is not None:
            raise ValueError('Darknet: training needs every width a multiple of 32 and layers1.0 at 32 filters; %s is pruned to another '
                             'width (channel-pruned models run in eval mode)' % padded)
        return model.Backbone.trainer.fget(self)

    def drop_operands(self):
        """The engine's per-unit operands (Darknet caches nothing on the module)."""
        if self._engine is not None:
            self._engine.invalidate()

    def forward(self, x):
        if self.training:
            return self.train_forward(x)
        return self.engine.forward(x).clone()     # the plan-owned buffer is overwritten by the next call; callers own what we return

    def scope(self, name):
        """'layers1.4.conv.weight' -> 'layers1.4' (reference model/yolo2.py:132-133)."""
        return name.rsplit('.', 2)[0]

    def get_mapper(self, index):
        """Channel map of the reorg node for the pruning tools (reference model/yolo2.py:135-137)."""
        if index == 94:
            n = self.stride * self.stride
            return lambda indices, channels: torch.cat([indices + k * channels for k in range(n)])


class ConstantPad2d(nn.Module):
    """Index placeholder for Tiny's nn.ConstantPad2d((0, 1, 0, 1), float32 min) (reference model/yolo2.py:150); the pad
    is folded into the stride-1 pooling kernel (yb_maxpool2x2_s1_f16)."""
    is_pool = True

    def __init__(self, padding=(0, 1, 0, 1)):
        nn.Module.__init__(self)
        if tuple(padding) != (0, 1, 0, 1):
            raise ValueError('only ConstantPad2d((0, 1, 0, 1)) is on the Tiny path')
        self.padding = tuple(padding)


class MaxPool2dStride1(nn.Module):
    """Index placeholder for Tiny's nn.MaxPool2d(kernel_size=2, stride=1) (reference model/yolo2.py:151)."""
    is_pool = True

    def __init__(self):
        nn.Module.__init__(self)
        self.kernel_size, self.stride = 2, 1


class Tiny(model.Backbone):
    """Tiny YOLOv2 backbone plugin (reference model/yolo2.py:140-173; the repo's default `model/dnn`, config.ini:25),
    inference and training on the CUDA kernels.  Same constructor contract `Tiny(config_channels, anchors, num_cls, channels=16)`, same
    state_dict keys (`layers.{0,2,4,6,8,10,13,14,15}.conv.*`, `.bn.*`), `init()` (xavier-normal, :159-165), `scope()`
    (:170-171) and forward contract x[B,3,H,W] fp32 -> [B, A*(5+C), H/32, W/32] fp32.

    Kernel chain: the 3->16 first layer runs on the fused first-layer kernel with its 16 filters zero-padded to 32 (the
    extra channels come out as exact zeros and the next layer's weights are zero-padded on the input side to match), the
    two Cin = 32 layers on the halo-tile wgmma kernel with the 2x2 max-pool fused, the rest on the implicit-GEMM
    kernel; `ConstantPad2d + MaxPool2d(2, stride=1)` is one HBM kernel.

    Channel-pruned checkpoints (model.ConfigChannels) run at their own widths in eval mode: every unit but the head stores
    round_up(Cout, 8) channels (zero filters), the next unit's weight is zero-padded on the input side to that width, and a unit whose
    input width is not a multiple of 32 runs on the channel-tail conv (yb_conv_bn_act_tail_fwd)."""

    TRAINER = _train.TinyTrainer

    def __init__(self, config_channels, anchors, num_cls, channels=16):
        model.Backbone.__init__(self)
        cc = config_channels
        bn = cc.config.getboolean('batch_norm', 'enable')
        layers = []
        for _ in range(5):
            layers.append(Conv2d(cc.channels, cc(channels, 'layers.%d.conv.weight' % len(layers)), 3, bn=bn, padding=True))
            layers.append(MaxPool2d(2))
            channels *= 2
        layers.append(Conv2d(cc.channels, cc(channels, 'layers.%d.conv.weight' % len(layers)), 3, bn=bn, padding=True))
        layers.append(ConstantPad2d((0, 1, 0, 1)))
        layers.append(MaxPool2dStride1())
        channels *= 2
        for _ in range(2):
            layers.append(Conv2d(cc.channels, cc(channels, 'layers.%d.conv.weight' % len(layers)), 3, bn=bn, padding=True))
        layers.append(Conv2d(cc.channels, model.output_channels(len(anchors), num_cls), 1, bn=False, act=False))
        self.layers = nn.Sequential(*layers)
        self.init()
        self._units = None

    def unit_keys(self):
        """[(state_dict prefix 'layers.N', ConvUnit, followed_by)] in network order."""
        keys = ['layers.%d' % i for i, m in enumerate(self.layers) if not m.is_pool]
        return [(k, u, after) for k, (u, after) in zip(keys, self._plan())]

    def padded_unit(self):
        """The prefix of the first unit after layers.0 whose width is not a multiple of 32 (the head aside), or None."""
        for key, u, _ in self.unit_keys()[1:-1]:
            if u.cout % 32:
                return key
        return None

    @property
    def trainer(self):
        padded = self.padded_unit()
        if padded is not None:
            raise ValueError('Tiny: training needs every width after layers.0 a multiple of 32; %s is pruned to another width '
                             '(channel-pruned models run in eval mode)' % padded)
        return model.Backbone.trainer.fget(self)

    def drop_operands(self):
        """The padded operands and the units' own (ConvUnit.refresh)."""
        model.Backbone.drop_operands(self)
        for u, _ in self._units or ():
            u._wver = u._bver = None

    def init(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.xavier_normal_(m.weight)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def scope(self, name):
        return '.'.join(name.split('.')[:-2])

    # ---- operands ----------------------------------------------------------------------------------
    def _plan(self):
        """[(ConvUnit, followed_by: None | 'pool' | 'pool_s1')] in network order."""
        if self._units is None:
            mods = list(self.layers)
            plan = []
            for i, m in enumerate(mods):
                if m.is_pool:
                    continue
                after = None
                if i + 1 < len(mods) and isinstance(mods[i + 1], MaxPool2d):
                    after = 'pool'
                elif i + 1 < len(mods) and isinstance(mods[i + 1], ConstantPad2d):
                    after = 'pool_s1'
                plan.append((_engine.ConvUnit(m.conv, m.bn if m.has_bn else None, m.has_act), after))
            self._units = plan
        return self._units

    def _padded(self, key, u, cout_to, cin_to, first):
        """Zero-padded copy of a unit's operands (weights, scale, shift), cached per version of the unit's own operands."""
        def build():
            w = u.conv.weight.detach()
            cout, cin, k, _ = w.shape
            wp = torch.zeros(cout_to, cin_to, k, k, dtype=torch.float32, device=w.device)
            wp[:cout, :cin] = w
            w_op = wp.contiguous() if first else _ops.pack_weight_f16(wp.contiguous(), 0)
            scale = torch.zeros(cout_to, dtype=torch.float32, device=w.device)
            shift = torch.zeros(cout_to, dtype=torch.float32, device=w.device)
            scale[:cout], shift[:cout] = u.scale, u.shift
            return w_op, scale, shift
        return self._cache.fetch(key, (), build, extra=(u._wver, u._bver))

    def forward(self, x):
        if self.training:
            return self.train_forward(x)
        if not x.is_cuda:
            raise RuntimeError('Tiny: input must be a CUDA tensor; there is no CPU fallback')
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('Tiny expects fp32 [B,3,H,W] with H, W multiples of 32, got %s' % (tuple(x.shape),))
        x = x.contiguous().float()
        plan = self._plan()
        for i, (u, _) in enumerate(plan):
            u.refresh(first_layer=(i == 0))
        u0, after0 = plan[0]
        if after0 != 'pool' or u0.cout > 32:
            raise RuntimeError('Tiny: the first unit must have <= 32 filters and be followed by MaxPool2d(2)')
        w0, sc0, sh0 = self._padded('u0', u0, 32, 3, True)
        cur = _ops.conv0_bn_leaky_pool(x, w0, sc0, sh0, u0.slope)          # [B,H/2,W/2,32], channels >= cout are exact zeros
        chan = 32                                                          # channels per pixel of `cur`
        for i, (u, after) in enumerate(plan[1:], 1):
            last = i == len(plan) - 1
            cout_to = u.cout if last else _ops.round_up(u.cout, 8)          # stored width; the head writes fp32 NCHW at its own
            cin_to = _ops.round_up(chan, 32)
            if u.cin != cin_to or u.cout != cout_to:                       # zero-padded to the producer's width and the stored one
                w_op, scale, shift = self._padded('u%d' % i, u, cout_to, cin_to, False)
            else:
                w_op, scale, shift = u.w16, u.scale, u.shift
            if chan % 32:
                def conv(**kw):
                    return _ops.conv_bn_act_tail(cur, w_op, scale, shift, u.slope, chan, **kw)
            else:
                def conv(**kw):
                    return _ops.conv_bn_act(cur, w_op, scale, shift, u.slope, **kw)
            if last:
                return conv(out_mode=_ops.OUT_F32_NCHW)
            fuse = after == 'pool' and chan == 32 and u.ksize == 3 and cout_to <= 64
            if fuse:
                cur = conv(flags=_ops.CONV_POOL2X2)
            else:
                cur = conv()
                if after == 'pool':
                    cur = _ops.maxpool2x2(cur)
                elif after == 'pool_s1':
                    cur = _ops.maxpool2x2_s1(cur)
            chan = cout_to
