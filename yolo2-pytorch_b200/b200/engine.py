"""Execution plan of the Darknet-19 forward pass on the CUDA kernels.

The plugin module (`model.yolo2.Darknet`) only holds parameters with the reference's state_dict
names; this engine turns them into kernel operands (fp16 KRSC weights, folded BN scale/shift),
owns one set of fp16 NHWC activation buffers per input shape (sized once, reused every call -- HBM
is 180 GB, the whole B=32 @ 416 plan is < 1 GB) and issues the kernel chain on torch's current
stream.  The 1280-channel concat buffer is written in place by the reorg kernel (channels 0..255)
and by layers2.7 (channels 256..1279), so torch.cat (model/yolo2.py:129) never runs.
"""
import os
import weakref

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


class OperandCache(dict):
    """Kernel operands built from module tensors (packed weights, folded BatchNorms), one entry per key."""

    def fetch(self, key, tensors, build, extra=()):
        """The value stored under `key` while every tensor's (data_ptr, _version) and `extra` are unchanged, else `build()`, stored in its
        place.  A hit returns the same object: CUDA graphs captured over a forward read the cached buffers by address.  `tensors=()` gives
        a constant built once."""
        ver = tuple((t.data_ptr(), t._version) for t in tensors) + tuple(extra)
        hit = self.get(key)
        if hit is None or hit[0] != ver:
            hit = self[key] = (ver, build())
        return hit[1]


def epilogue_tensors(bn, bias=None):
    """The tensors `fold_epilogue(bn, bias)` reads."""
    ts = () if bias is None else (bias,)
    return ts if bn is None else ts + (bn.weight, bn.bias, bn.running_mean, bn.running_var)


def fold_epilogue(bn, bias, cout_pad=None):
    """(scale, shift) of a conv's epilogue: BatchNorm `bn` folded (the conv's `bias`, if it has one, folded into the shift), or (1, bias)
    without BatchNorm; padded to `cout_pad` filters with (1, 0)."""
    if bias is not None:
        bias = bias.detach().float().contiguous()
    if bn is None:
        s, t = torch.ones_like(bias), bias
    else:
        s, t = ops.bn_fold(*(p.detach().float().contiguous() for p in epilogue_tensors(bn)), eps=bn.eps)
        if bias is not None:
            t = t + s * bias
    n = 0 if cout_pad is None else cout_pad - s.numel()
    if n:
        s = torch.cat([s, torch.ones(n, dtype=torch.float32, device=s.device)])
        t = torch.cat([t, torch.zeros(n, dtype=torch.float32, device=t.device)])
    return s, t


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
        # channel layout of a channel-pruned network (DarknetEngine._set_layout): the unit reads in_ch channels per pixel and stores out_ch,
        # its own input channel i sits at channel cin_index[i] of the input (None: at i), and its packed weight has k_ch input channels
        # per tap (round_up(in_ch, 32); zero past the real ones)
        self.in_ch, self.out_ch, self.k_ch, self.cin_index = self.cin, self.cout, self.cin, None

    @property
    def padded(self):
        """Whether the operands are zero-padded to a channel layout other than the conv's own widths."""
        return self.in_ch != self.cin or self.k_ch != self.cin or self.out_ch != self.cout or self.cin_index is not None

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
            if self.padded:
                self.w16 = self._layout_weight(w.detach(), first_layer)
            elif first_layer:
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
                self._pad_epilogue()
                self._bver = bver
        else:
            b = self.conv.bias
            bver = None if b is None else (b.data_ptr(), b._version)
            if bver != self._bver or self.scale is None:
                self.scale = torch.ones(self.cout, dtype=torch.float32, device=w.device)
                self.shift = (b.detach().float().contiguous().clone() if b is not None
                              else torch.zeros(self.cout, dtype=torch.float32, device=w.device))
                self._pad_epilogue()
                self._bver = bver

    def _layout_weight(self, w, first_layer):
        """The weight scattered onto the unit's channel layout: filters [cout, out_ch) and input channels outside cin_index are zero.
        fp32 [out_ch,3,k,k] for the first-layer kernel, else fp16 [out_ch,k,k,k_ch]."""
        cout, cin, k, _ = w.shape
        wp = torch.zeros(self.out_ch, cin if first_layer else self.k_ch, k, k, dtype=torch.float32, device=w.device)
        idx = torch.arange(cin) if self.cin_index is None else self.cin_index
        wp[:cout, idx.to(w.device)] = w.float()
        return wp.contiguous() if first_layer else ops.pack_weight_f16(wp.contiguous(), 0)

    def _pad_epilogue(self):
        """Scale 1 and shift 0 on the zero filters [cout, out_ch): they store exact zeros."""
        n = self.out_ch - self.cout
        if n:
            self.scale = torch.cat([self.scale, torch.ones(n, dtype=torch.float32, device=self.scale.device)])
            self.shift = torch.cat([self.shift, torch.zeros(n, dtype=torch.float32, device=self.shift.device)])


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
        self.a0 = torch.empty(batch, h, w, units1[0].out_ch, **f16)
        self.l1 = []   # (out, pooled or None) per layers1 unit after the first
        for u, pooled in zip(units1[1:], pools1[1:]):
            out = torch.empty(batch, h, w, u.out_ch, **f16)
            if pooled:
                h, w = h // 2, w // 2
                self.l1.append((out, torch.empty(batch, h, w, u.out_ch, **f16)))
            else:
                self.l1.append((out, None))
        self.h16, self.w16 = h, w
        self.pt = torch.empty(batch, h, w, unit_pt.out_ch, **f16)
        self.x1_pool = torch.empty(batch, h // 2, w // 2, units1[-1].out_ch, **f16)
        h, w = h // 2, w // 2
        self.h32, self.w32 = h, w
        self.cat_ch = unit_pt.out_ch * 4 + units2[-1].out_ch
        self.cat = torch.empty(batch, h, w, self.cat_ch, **f16)
        self.l2 = [torch.empty(batch, h, w, u.out_ch, **f16) for u in units2[:-1]]
        self.l3 = torch.empty(batch, h, w, units3[0].out_ch, **f16)
        self.feature = torch.empty(batch, units3[1].cout, h, w, dtype=torch.float32, device=device)
        # stream-K scratch (partial sums + flags): per plan, because plans are what run concurrently on different streams
        self.workspace = ops.conv_workspace(device)


class DarknetEngine(object):
    def __init__(self, dnn):
        """`dnn` is a model.yolo2.Darknet (parameter holder).  Units are discovered from its nn.Sequential containers, so channel-pruned
        checkpoints (model.ConfigChannels) and `ratio` models run at their own widths on the layout of `_set_layout`."""
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
        self._dnn = weakref.ref(dnn)        # its input_transform: the table uint8 frames go through
        self.plans = {}
        if not self.pools1[0]:
            raise RuntimeError('Darknet: layers1.0 must be followed by MaxPool2d (fused first-layer kernel)')
        self._set_layout()
        self.precision = 'fast'
        self.set_precision(os.environ.get('YB_PRECISION', 'fast'))
        # the fast forward fuses a layers1 max-pool into the conv before it wherever the library has a pooled form for that launch;
        # False keeps the 3x3 Cin = 32 halo kernel's fusion only (A/B runs and tests)
        self.fuse_wide_pool = True
        self._pool_ok = {}
        # the fast forward also runs a layers1 1x1 unit in the epilogue of the conv before it wherever the library accepts that pair
        # (layers1.4 -> 1.5 at 416x416), so the producer's output never goes to HBM; False keeps the separate launches
        self.fuse_chain = True
        self._chain_ok = {}

    def _set_layout(self):
        """Channel layout of the activation buffers.  Every unit stores round_up(Cout, 8) channels (the extra filters are zero with scale 1
        and shift 0, so they hold exact zeros); layers1.0 stores the first-layer kernel's 32.  The passthrough stores P = round_up(Cpt, 8),
        the reorg writes its 4 offsets as 4 groups of P channels and layers2's last unit writes at channel 4P, so the reference's concat
        channel s*Cpt + c (model/yolo2.py:129, the map of get_mapper(94)) sits at s*P + c and 4*Cpt + j at 4P + j.  Each unit reads its
        producer's stored width; its weight is scattered onto that layout with zeros in the gaps.  At full width (every width a multiple
        of 32) nothing is padded and every operand is the unit's own."""
        u0 = self.units1[0]
        if u0.cout > 32:
            raise ValueError('Darknet: %s has %d filters; the first-layer kernel runs at most 32' % (self._k1[0], u0.cout))
        u0.out_ch = 32
        prev = 32
        for u in self.units1[1:] + self.units2:         # layers2.1 reads the pooled output of layers1's last unit
            u.in_ch, u.out_ch = prev, ops.round_up(u.cout, 8)
            prev = u.out_ch
        pt, u27 = self.unit_pt, self.units2[-1]
        pt.in_ch, pt.out_ch = self.units1[-1].out_ch, ops.round_up(pt.cout, 8)
        u30, u31 = self.units3
        u30.in_ch, u30.out_ch = 4 * pt.out_ch + u27.out_ch, ops.round_up(u30.cout, 8)
        if pt.out_ch != pt.cout:
            u30.cin_index = self.concat_index(pt.cout, pt.out_ch, u27.cout)
        u31.in_ch = u30.out_ch      # the head stores fp32 NCHW at its own width
        for u in self.all_units()[1:]:
            u.k_ch = ops.round_up(u.in_ch, 32)

    @staticmethod
    def concat_index(c_pt, p, c_trunk):
        """Layout channel of each channel of the reference's concat [reorg(passthrough) | layers2]: s*c_pt + c -> s*p + c, 4*c_pt + j -> 4p + j."""
        return torch.cat([torch.arange(c_pt) + s * p for s in range(4)] + [torch.arange(c_trunk) + 4 * p])

    def padded_unit(self):
        """The state_dict prefix of the first unit whose operands are padded to the channel layout, or None at full width."""
        for key, u in zip(self.unit_keys(), self.all_units()):
            if u.padded:
                return key
        return None

    def _chained_form(self, u, v, x, conv_flags):
        """Whether the library runs unit u on input x [B,H,W,C] with the 1x1 unit v fused into its epilogue, with the same bits as v's
        own launch (which must not split along K), asked once per shape."""
        b, h, w, _ = x.shape
        key = (u.in_ch, u.out_ch, u.ksize, v.out_ch, b, h, w, conv_flags)
        ok = self._chain_ok.get(key)
        if ok is None:
            ok = v.ksize == 1 and u.in_ch % 32 == 0 and v.in_ch == u.out_ch and v.out_ch <= 64 and v.out_ch % 8 == 0
            if ok:
                try:
                    ok = (ops.conv_choice(b, h, w, u.in_ch, u.out_ch, u.ksize, flags=conv_flags | ops.CONV_CHAIN1X1)['kernel'] == 'conv_wide_kernel'
                          and not ops.conv_choice(b, h, w, v.in_ch, v.out_ch, 1, flags=conv_flags)['streamk'])
                except RuntimeError:
                    ok = False
            self._chain_ok[key] = ok
        return ok

    def _pooled_form(self, u, x, conv_flags):
        """Whether the library runs unit u on input x [B,H,W,C] with the 2x2 max-pool fused on the two-consumer tile (asked once per shape)."""
        b, h, w, _ = x.shape
        key = (u.in_ch, u.out_ch, u.ksize, b, h, w, conv_flags)
        ok = self._pool_ok.get(key)
        if ok is None:
            try:
                ok = (u.in_ch % 32 == 0 and
                      ops.conv_choice(b, h, w, u.in_ch, u.out_ch, u.ksize, flags=conv_flags | ops.CONV_POOL2X2)['kernel'] == 'conv_wide_kernel')
            except RuntimeError:
                ok = False
            self._pool_ok[key] = ok
        return ok

    def unit_keys(self):
        return self._k1 + self._k2 + ['passthrough', 'layers3.0', 'layers3.1']

    def set_precision(self, precision, keep=None):
        """'fast' (default): fp16 operands, one wgmma pass per unit; measured end-to-end drift of the head feature vs the
        reference's fp32 1.1e-3 .. 2.0e-3 (max|d| / max|ref|).  'strict': split-precision operands on every unit except `keep`
        (default STRICT_KEEP) -- inside the reference contract of 1e-3 at ~2.6x the tensor-core work."""
        if precision not in PRECISIONS:
            raise ValueError('precision must be one of %s' % (PRECISIONS,))
        padded = self.padded_unit()
        if precision == 'strict' and padded is not None:
            raise ValueError("Darknet: precision 'strict' needs every width a multiple of 32 and layers1.0 at 32 filters; %s is pruned to "
                             "another width" % padded)
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
        """x: fp32 NCHW [B,3,H,W] on the GPU, or uint8 NHWC frames [B,H,W,3] -> feature fp32 NCHW [B,A*(5+C),H/32,W/32]
        (a plan-owned buffer, overwritten by the next call with the same shape).  uint8 frames go through the Darknet's input_transform
        table in the first-layer kernel, or without one through ToTensor's 1/255 scaling.
        `collect` (dict) receives references to every unit's fp16 NHWC output (tests)."""
        if not x.is_cuda:
            raise RuntimeError('Darknet: input must be a CUDA tensor; there is no CPU fallback')
        u8 = x.dtype == torch.uint8          # raw RGB frames [B,H,W,3]: the kernel applies the input transform
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
            if u.in_ch % 32:
                if ref:
                    raise ValueError('Darknet: the CUDA-core reference conv has no channel-tail form')
                return ops.conv_bn_act_tail(src, u.w16, u.scale, u.shift, u.slope, u.in_ch, out=dst, flags=conv_flags, **kw)
            return ops.conv_bn_act(src, u.w16, u.scale, u.shift, u.slope, out=dst, flags=conv_flags, ref=ref, workspace=p.workspace, **kw)

        cur = self._conv0(x, u8, p.a0)
        if collect is not None:
            collect['layers1.0(pooled)'] = cur
        x1 = None
        last1 = self.units1[-1]
        l1 = list(zip(self.units1[1:], p.l1, self._k1[1:]))
        chained = False         # this unit already ran in the previous launch's epilogue
        for i, (u, (out, pooled), key) in enumerate(l1):
            if chained:
                x1 = out
                cur = ops.maxpool2x2(out, out=pooled) if pooled is not None else out
                chained = False
                continue
            # a 1x1 unit that reads only this unit's output (layers1.5 after 1.4 at 416x416) runs in this launch's epilogue
            if (self.fuse_chain and pooled is None and collect is None and not ref and i + 1 < len(l1)
                    and self._chained_form(u, l1[i + 1][0], cur, conv_flags)):
                v, (v_out, _), _ = l1[i + 1]
                ops.conv_bn_act(cur, u.w16, u.scale, u.shift, u.slope, out=v_out, flags=conv_flags, workspace=p.workspace,
                                chain=(v.w16, v.scale, v.shift, v.slope))
                chained = True
                continue
            # layers1.2 (3x3, Cin = 32) has a kernel whose epilogue applies the MaxPool2d that follows it, so the
            # 208x208x64 activation never goes to HBM, and so do the 3x3 layers on the two-consumer tile (layers1.6 and 1.10 at
            # 416x416); tests that inspect every layer (collect / ref) keep the two steps.  last1's full-resolution output feeds the
            # passthrough, so its pool stays a kernel of its own.
            fuse_pool = pooled is not None and u is not last1 and collect is None and not ref and (
                (u.in_ch == 32 and u.ksize == 3 and u.out_ch <= 64 and (conv_flags & (ops.CONV_NO_SMALLK | ops.CONV_C32_IM2COL)) == 0
                 and conv_flags < 256) or (self.fuse_wide_pool and self._pooled_form(u, cur, conv_flags)))
            if fuse_pool:
                ops.conv_bn_act(cur, u.w16, u.scale, u.shift, u.slope, out=pooled, flags=conv_flags | ops.CONV_POOL2X2, workspace=p.workspace)
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
        conv(self.units2[-1], cur, p.cat, y_ch_off=self.unit_pt.out_ch * 4)
        conv(self.units3[0], p.cat, p.l3)
        conv(self.units3[1], p.l3, p.feature, out_mode=ops.OUT_F32_NCHW)
        if collect is not None:
            collect['cat'] = p.cat
            collect['layers3.0'] = p.l3
        return p.feature

    def _conv0(self, x, u8, out):
        """layers1.0 + its max-pool into `out`: fp32 image, or uint8 frames through the input transform's table (1/255 without one)."""
        u0 = self.units1[0]
        t = getattr(self._dnn(), 'input_transform', None) if u8 else None
        if t is not None:
            return ops.conv0_bn_leaky_pool(x, u0.w16, u0.scale, u0.shift, u0.slope, out=out, lut=t.lut(x.device))
        conv0 = ops.conv0_u8_bn_leaky_pool if u8 else ops.conv0_bn_leaky_pool
        return conv0(x, u0.w16, u0.scale, u0.shift, u0.slope, out=out)

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

        cur, cur_c, cur_lo = self._conv0(x, u8, p.a0), self.units1[0].cout, False
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
