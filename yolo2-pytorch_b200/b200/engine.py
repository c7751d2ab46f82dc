"""Execution plan of the Darknet-19 forward pass on the CUDA kernels.

The plugin module (`model.yolo2.Darknet`) only holds parameters with the reference's state_dict
names; this engine turns them into kernel operands (fp16 KRSC weights, folded BN scale/shift),
owns one set of fp16 NHWC activation buffers per input shape (sized once, reused every call -- HBM
is 180 GB, the whole B=32 @ 416 plan is < 1 GB) and issues the kernel chain on torch's current
stream.  The 1280-channel concat buffer is written in place by the reorg kernel (channels 0..255)
and by layers2.7 (channels 256..1279), so torch.cat (model/yolo2.py:129) never runs.
"""
import os

import torch

from . import ops

# Strict precision (`precision = 'strict'`): which operand roundings stay fp16-only, per unit ('a' = input activation, 'w' = weight).
# Every unit not listed removes both with the split-precision conv (yb_conv_bn_act_split_fwd: a_hi*w_hi + a_lo*w_hi + a_hi*w_lo in one
# fp32 accumulator).  Error budget (tools/error_budget.py, CPU simulation of exactly these roundings): each of the 46 (unit, operand)
# roundings adds ~2e-4 relative rms to the head feature -- 1.7e-3 .. 2.0e-3 max-norm with all of them (the default 'fast' mode) --
# and keeping only the ones below leaves 4.2e-4 .. 5.6e-4, inside the reference contract of 1e-3 (BASELINE.json north_star).  The
# first two layers and the passthrough contribute half as much as the others (1e-4) and have dedicated kernels; layers3.0 is the
# single most expensive unit (3.99 GFLOP/image); layers1.4 keeps its input rounding (1.2e-4) so that layers1.2 stays on the
# halo-tile kernel with the fused max-pool.
STRICT_KEEP = {'layers1.0': 'aw', 'layers1.2': 'aw', 'layers1.4': 'a', 'passthrough': 'aw', 'layers3.0': 'aw'}
PRECISIONS = ('fast', 'strict')


class ConvUnit(object):
    """Operands of one `model.yolo2.Conv2d` unit (conv [+BN] [+leaky]); cached per parameter version."""

    def __init__(self, conv, bn, act):
        self.conv, self.bn, self.act = conv, bn, act
        self._wver = None
        self._bver = None
        self.w16 = self.scale = self.shift = None
        # strict precision: which operand of this unit is split into fp16 hi + lo (set by DarknetEngine.set_precision)
        self.split_a = self.split_w = False
        self.out_lo = False      # the epilogue also writes the rounding residual (a consumer reads [hi | lo])

    @property
    def cout(self):
        return self.conv.weight.shape[0]

    @property
    def cin(self):
        return self.conv.weight.shape[1]

    @property
    def ksize(self):
        return self.conv.weight.shape[2]

    @property
    def slope(self):
        return 0.1 if self.act else 1.0

    def refresh(self, first_layer=False, force=False):
        """Re-derive the kernel operands when the parameters changed.  `force` skips the version check: training
        steps always re-pack, because fused multi-tensor optimizers (torch.optim.Adam(fused=True)) update parameters
        without advancing torch's version counter."""
        w = self.conv.weight
        wver = (w.data_ptr(), w._version)
        wver = wver + (self.split_a, self.split_w)
        if force or wver != self._wver:
            if first_layer:
                self.w16 = w.detach().contiguous()
            elif self.split_a or self.split_w:
                self.w16 = ops.pack_weight_split_f16(w.detach().contiguous(), self.split_a, self.split_w)
            else:
                self.w16 = ops.pack_weight_f16(w.detach().contiguous(), 0)
            self._wver = wver
        if self.bn is not None:
            ts = (self.bn.weight, self.bn.bias, self.bn.running_mean, self.bn.running_var)
            bver = tuple((t.data_ptr(), t._version) for t in ts)
            if bver != self._bver:
                self.scale, self.shift = ops.bn_fold(*(t.detach().contiguous() for t in ts), eps=self.bn.eps)
                self._bver = bver
        else:
            b = self.conv.bias
            bver = None if b is None else (b.data_ptr(), b._version)
            if bver != self._bver or self.scale is None:
                self.scale = torch.ones(self.cout, dtype=torch.float32, device=w.device)
                self.shift = (b.detach().float().contiguous().clone() if b is not None
                              else torch.zeros(self.cout, dtype=torch.float32, device=w.device))
                self._bver = bver


class StrictPlan(object):
    """Activation buffers of the strict-precision forward: a unit whose consumer splits its input activation stores
    [hi | lo] (2*Cout channels per pixel), everything else as in DarknetPlan."""

    def __init__(self, eng, batch, height, width, device):
        f16 = dict(dtype=torch.float16, device=device)

        def buf(u, h, w):
            return torch.empty(batch, h, w, u.cout * (2 if u.out_lo else 1), **f16)

        h, w = height // 2, width // 2
        self.a0 = torch.empty(batch, h, w, eng.units1[0].cout, **f16)
        self.l1 = []
        for u, pooled in zip(eng.units1[1:], eng.pools1[1:]):
            out = buf(u, h, w)
            if pooled:
                h, w = h // 2, w // 2
                self.l1.append((out, buf(u, h, w)))
            else:
                self.l1.append((out, None))
        self.pt = buf(eng.unit_pt, h, w)
        h, w = h // 2, w // 2
        self.x1_pool = buf(eng.units1[-1], h, w)
        self.cat_c = eng.unit_pt.cout * 4 + eng.units2[-1].cout
        self.cat = torch.empty(batch, h, w, self.cat_c * (2 if eng.units3[0].split_a else 1), **f16)
        self.l2 = [buf(u, h, w) for u in eng.units2[:-1]]
        self.l3 = buf(eng.units3[0], h, w)
        self.feature = torch.empty(batch, eng.units3[1].cout, h, w, dtype=torch.float32, device=device)
        self.workspace = ops.conv_workspace(device)


class DarknetPlan(object):
    """Activation buffers for one (batch, height, width)."""

    def __init__(self, units1, units2, unit_pt, units3, pools1, batch, height, width, device):
        f16 = dict(dtype=torch.float16, device=device)
        self.batch, self.height, self.width = batch, height, width
        h, w = height // 2, width // 2
        self.a0 = torch.empty(batch, h, w, units1[0].cout, **f16)
        self.l1 = []   # (out, pooled or None) per layers1 unit after the first
        for u, pooled in zip(units1[1:], pools1[1:]):
            out = torch.empty(batch, h, w, u.cout, **f16)
            if pooled:
                h, w = h // 2, w // 2
                self.l1.append((out, torch.empty(batch, h, w, u.cout, **f16)))
            else:
                self.l1.append((out, None))
        self.h16, self.w16 = h, w
        self.pt = torch.empty(batch, h, w, unit_pt.cout, **f16)
        self.x1_pool = torch.empty(batch, h // 2, w // 2, units1[-1].cout, **f16)
        h, w = h // 2, w // 2
        self.h32, self.w32 = h, w
        self.cat_ch = unit_pt.cout * 4 + units2[-1].cout
        self.cat = torch.empty(batch, h, w, self.cat_ch, **f16)
        self.l2 = [torch.empty(batch, h, w, u.cout, **f16) for u in units2[:-1]]
        self.l3 = torch.empty(batch, h, w, units3[0].cout, **f16)
        self.feature = torch.empty(batch, units3[1].cout, h, w, dtype=torch.float32, device=device)
        # stream-K scratch (partial sums + flags): per plan, because plans are what run concurrently on different streams
        self.workspace = ops.conv_workspace(device)


class DarknetEngine(object):
    def __init__(self, dnn):
        """`dnn` is a model.yolo2.Darknet (parameter holder).  Units are discovered from its
        nn.Sequential containers so channel-pruned checkpoints (model.ConfigChannels) just work."""
        def unit(m):
            return ConvUnit(m.conv, m.bn if m.has_bn else None, m.has_act)

        self.units1, self.pools1, self._k1 = [], [], []
        mods = list(dnn.layers1)
        for i, m in enumerate(mods):
            if m.is_pool:
                continue
            self.units1.append(unit(m))
            self.pools1.append(i + 1 < len(mods) and mods[i + 1].is_pool)
            self._k1.append('layers1.%d' % i)
        self.units2 = [unit(m) for m in dnn.layers2 if not m.is_pool]
        self._k2 = ['layers2.%d' % i for i, m in enumerate(dnn.layers2) if not m.is_pool]
        self.unit_pt = unit(dnn.passthrough)
        self.units3 = [unit(m) for m in dnn.layers3]
        self.plans = {}
        if not self.pools1[0]:
            raise RuntimeError('Darknet: layers1.0 must be followed by MaxPool2d (fused first-layer kernel)')
        self.precision = 'fast'
        self.set_precision(os.environ.get('YB_PRECISION', 'fast'))

    def unit_keys(self):
        return self._k1 + self._k2 + ['passthrough', 'layers3.0', 'layers3.1']

    def set_precision(self, precision, keep=None):
        """'fast' (default): fp16 operands, one wgmma pass per unit; measured end-to-end drift of the head feature vs the
        reference's fp32 1.1e-3 .. 2.0e-3 (max|d| / max|ref|).  'strict': split-precision operands on every unit except `keep`
        (default STRICT_KEEP) -- inside the reference contract of 1e-3 at ~2.6x the tensor-core work."""
        if precision not in PRECISIONS:
            raise ValueError('precision must be one of %s' % (PRECISIONS,))
        keep = STRICT_KEEP if keep is None else keep
        units = dict(zip(self.unit_keys(), self.all_units()))
        for key, u in units.items():
            k = keep.get(key, '') if precision == 'strict' else 'aw'
            u.split_a, u.split_w, u.out_lo = 'a' not in k, 'w' not in k, False
        units[self._k1[0]].split_a = units[self._k1[0]].split_w = False      # first layer: dedicated fp32-input kernel
        units[self._k1[1]].split_a = False                                   # its input comes from that kernel (hi only)
        # producers of split activations also write the rounding residual
        chain1 = self.units1
        for prev, nxt in zip(chain1[:-1], chain1[1:]):
            prev.out_lo = nxt.split_a
        chain1[-1].out_lo = self.unit_pt.split_a or self.units2[0].split_a
        for prev, nxt in zip(self.units2[:-1], self.units2[1:]):
            prev.out_lo = nxt.split_a
        self.units2[-1].out_lo = self.unit_pt.out_lo = self.units3[0].split_a
        self.units3[0].out_lo = self.units3[1].split_a
        chain1[0].out_lo = False
        # a consumer whose producer cannot deliver lo reads hi only
        self.precision = precision
        self.plans = {}
        self.invalidate()

    def all_units(self):
        return self.units1 + self.units2 + [self.unit_pt] + self.units3

    def plan(self, batch, height, width, device, plan_id=0):
        key = (batch, height, width, str(device), plan_id)
        p = self.plans.get(key)
        if p is None and self.precision == 'strict':
            p = self.plans[key] = StrictPlan(self, batch, height, width, device)
        if p is None:
            p = DarknetPlan(self.units1, self.units2, self.unit_pt, self.units3, self.pools1, batch, height, width, device)
            self.plans[key] = p
        return p

    def refresh(self, force=False):
        for i, u in enumerate(self.all_units()):
            u.refresh(first_layer=(i == 0), force=force)

    def invalidate(self):
        """Forget every cached operand (called when the module switches between train() and eval())."""
        for u in self.all_units():
            u._wver = None
            u._bver = None

    def forward(self, x, conv_flags=0, ref=False, collect=None, plan_id=0):
        """x: fp32 NCHW [B,3,H,W] on the GPU -> feature fp32 NCHW [B,A*(5+C),H/32,W/32]
        (a plan-owned buffer, overwritten by the next call with the same shape).
        `collect` (dict) receives references to every unit's fp16 NHWC output (tests)."""
        if not x.is_cuda:
            raise RuntimeError('Darknet: input must be a CUDA tensor; there is no CPU fallback')
        u8 = x.dtype == torch.uint8          # raw RGB frames [B,H,W,3]: the kernel applies ToTensor's 1/255
        if u8:
            b, h, w, c = x.shape
        else:
            b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('Darknet expects fp32 [B,3,H,W] or uint8 [B,H,W,3] with H, W multiples of 32, got %s' % (tuple(x.shape),))
        x = x.contiguous() if u8 else x.contiguous().float()
        self.refresh()
        p = self.plan(b, h, w, x.device, plan_id)   # plan_id: independent buffer sets for concurrent streams
        if self.precision == 'strict':
            return self._forward_strict(x, u8, p, conv_flags, collect)

        def conv(u, src, dst, **kw):
            return ops.conv_bn_act(src, u.w16, u.scale, u.shift, u.slope, out=dst, flags=conv_flags, ref=ref, workspace=p.workspace, **kw)

        u0 = self.units1[0]
        conv0 = ops.conv0_u8_bn_leaky_pool if u8 else ops.conv0_bn_leaky_pool
        cur = conv0(x, u0.w16, u0.scale, u0.shift, u0.slope, out=p.a0)
        if collect is not None:
            collect['layers1.0(pooled)'] = cur
        x1 = None
        last1 = self.units1[-1]
        for u, (out, pooled), key in zip(self.units1[1:], p.l1, self._k1[1:]):
            # layers1.2 (3x3, Cin = 32) has a kernel whose epilogue applies the MaxPool2d that follows it, so the
            # 208x208x64 activation never goes to HBM; tests that inspect every layer (collect / ref) keep the two steps
            fuse_pool = (pooled is not None and u is not last1 and collect is None and not ref and u.cin == 32 and u.ksize == 3
                         and u.cout <= 64 and (conv_flags & (ops.CONV_NO_SMALLK | ops.CONV_C32_IM2COL)) == 0 and conv_flags < 256)
            if fuse_pool:
                ops.conv_bn_act(cur, u.w16, u.scale, u.shift, u.slope, out=pooled, flags=conv_flags | ops.CONV_POOL2X2)
                cur = pooled
                continue
            conv(u, cur, out)
            if collect is not None:
                collect[key] = out
            x1 = out
            cur = ops.maxpool2x2(out, out=pooled) if pooled is not None else out
        # passthrough branch -> channels [0, 4*Cpt) of the concat buffer
        conv(self.unit_pt, x1, p.pt)
        if collect is not None:
            collect['passthrough'] = p.pt
        ops.reorg_f16(p.pt, p.cat, 0)
        # trunk
        cur = ops.maxpool2x2(x1, out=p.x1_pool)
        for u, out, key in zip(self.units2[:-1], p.l2, self._k2):
            conv(u, cur, out)
            if collect is not None:
                collect[key] = out
            cur = out
        conv(self.units2[-1], cur, p.cat, y_ch_off=self.unit_pt.cout * 4)
        conv(self.units3[0], p.cat, p.l3)
        conv(self.units3[1], p.l3, p.feature, out_mode=ops.OUT_F32_NCHW)
        if collect is not None:
            collect['cat'] = p.cat
            collect['layers3.0'] = p.l3
        return p.feature

    def _forward_strict(self, x, u8, p, conv_flags, collect):
        """Same chain with split-precision operands (see STRICT_KEEP).  Buffers of units with `out_lo` hold [hi | lo]."""
        def view(t, c, lo):
            return (t[..., :c].float() + t[..., c:2 * c].float()) if lo else t[..., :c]

        def conv(u, src, src_c, src_lo, dst, y_ch_off=0, lo_ch_off=None, out_mode=ops.OUT_F16_NHWC):
            """src holds src_c channels (+ src_c of residuals when src_lo)."""
            split_a = u.split_a and src_lo
            if lo_ch_off is None:
                lo_ch_off = y_ch_off + u.cout if u.out_lo else -1
            if not (split_a or u.split_w or lo_ch_off >= 0):
                return ops.conv_bn_act(src, u.w16, u.scale, u.shift, u.slope, out=dst, flags=conv_flags, workspace=p.workspace, cin=src_c,
                                       y_ch_off=y_ch_off, out_mode=out_mode)
            if u.split_a and not src_lo:
                raise RuntimeError('strict plan: unit expects [hi | lo] input')
            return ops.conv_bn_act_split(src, u.w16, u.scale, u.shift, u.slope, dst, a_channels=src_c * (2 if split_a else 1), y_ch_off=y_ch_off,
                                         lo_ch_off=lo_ch_off, out_mode=out_mode, flags=conv_flags, workspace=p.workspace)

        u0 = self.units1[0]
        conv0 = ops.conv0_u8_bn_leaky_pool if u8 else ops.conv0_bn_leaky_pool
        cur, cur_c, cur_lo = conv0(x, u0.w16, u0.scale, u0.shift, u0.slope, out=p.a0), u0.cout, False
        if collect is not None:
            collect['layers1.0(pooled)'] = cur
        x1 = None
        for u, (out, pooled), key in zip(self.units1[1:], p.l1, self._k1[1:]):
            plain = not (u.split_a or u.split_w or u.out_lo)
            if (plain and pooled is not None and collect is None and u.cin == 32 and u.ksize == 3 and u.cout <= 64 and conv_flags == 0):
                # layers1.2 keeps its halo-tile kernel with the max-pool fused into the epilogue
                ops.conv_bn_act(cur, u.w16, u.scale, u.shift, u.slope, out=pooled, flags=ops.CONV_POOL2X2)
                cur, cur_c, cur_lo = pooled, u.cout, False
                continue
            conv(u, cur, cur_c, cur_lo, out)
            if collect is not None:
                collect[key] = view(out, u.cout, u.out_lo)
            x1, x1_c, x1_lo = out, u.cout, u.out_lo
            cur, cur_c, cur_lo = out, u.cout, u.out_lo
            if pooled is not None:
                cur = ops.maxpool2x2_split(out, u.cout, pooled) if u.out_lo else ops.maxpool2x2(out, out=pooled)
        cat_lo = self.units3[0].split_a
        upt = self.unit_pt
        conv(upt, x1, x1_c, x1_lo, p.pt)
        if collect is not None:
            collect['passthrough'] = view(p.pt, upt.cout, upt.out_lo)
        ops.reorg_f16(p.pt, p.cat, 0, channels=upt.cout)
        if cat_lo:
            ops.reorg_f16(p.pt, p.cat, p.cat_c, channels=upt.cout, x_ch_off=upt.cout)
        last1 = self.units1[-1]
        cur = ops.maxpool2x2_split(x1, last1.cout, p.x1_pool) if last1.out_lo else ops.maxpool2x2(x1, out=p.x1_pool)
        cur_c, cur_lo = last1.cout, last1.out_lo
        for u, out, key in zip(self.units2[:-1], p.l2, self._k2):
            conv(u, cur, cur_c, cur_lo, out)
            if collect is not None:
                collect[key] = view(out, u.cout, u.out_lo)
            cur, cur_c, cur_lo = out, u.cout, u.out_lo
        u27 = self.units2[-1]
        conv(u27, cur, cur_c, cur_lo, p.cat, y_ch_off=upt.cout * 4, lo_ch_off=(p.cat_c + upt.cout * 4) if cat_lo else -1)
        u30, u31 = self.units3
        conv(u30, p.cat, p.cat_c, cat_lo, p.l3)
        conv(u31, p.l3, u30.cout, u30.out_lo, p.feature, out_mode=ops.OUT_F32_NCHW, lo_ch_off=-1)
        if collect is not None:
            collect['cat'] = view(p.cat, p.cat_c, cat_lo)
            collect['layers3.0'] = view(p.l3, u30.cout, u30.out_lo)
        return p.feature
