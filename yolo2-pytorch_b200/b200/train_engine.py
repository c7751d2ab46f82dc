"""Training-mode forward and backward of the Darknet-19 backbone on the CUDA kernels.

What the reference gets from torch autograd over nn.Conv2d / BatchNorm2d(train) / LeakyReLU / MaxPool2d /
reorg / cat (model/yolo2.py:49-65,125-130; train.py:344-351) is issued here as an explicit kernel chain:

  forward, per unit : wgmma conv -> raw z (fp16 NHWC) -> batch statistics (double) -> running-stat update
                      (momentum 0.01) -> normalise + leaky (+ 2x2 max-pool) -> a
  backward, per unit: leaky/BN(/pool) backward in two passes (reduce, apply) -> dgamma, dbeta, dz (fp16)
                      -> wgmma weight gradient (pixels are the reduction dim) + wgmma data gradient
                      (the forward kernel on dz with rotated, transposed weights)

Gradients travel in fp16 multiplied by `grad_scale` (static loss scaling; parameter gradients are un-scaled in fp32).
BatchNorm statistics are per process (per GPU), exactly like the per-replica statistics of the reference's
nn.DataParallel.
"""
import os

import numpy as np
import torch

from . import ddp as _ddp
from . import ops

SLOPE = 0.1


class _Saved(object):
    pass


class _NullCtx(object):
    def __enter__(self):
        return None

    def __exit__(self, *exc):
        return False


class PackPlan(object):
    """Every unit's forward (w16) and data-gradient (rotated, transposed) fp16 operand re-derived from the fp32 parameters by ONE launch
    (yb_pack_weights_batch).  A training step must re-pack all of them -- the optimizer just changed the weights, and fused optimizers do not
    advance torch's version counters -- which used to be two latency-bound launches per unit.  The output buffers are persistent (the unit
    table holds their addresses), so the plan is rebuilt when a parameter moves."""
    DTYPE = np.dtype([('w', '<u8'), ('f', '<u8'), ('d', '<u8'), ('cout', '<i4'), ('cin', '<i4'), ('k', '<i4'), ('cp', '<i4'), ('b0', '<i4'), ('cib', '<i4')])

    def __init__(self, entries, device):
        """entries: [(key, weight [Cout,Cin,k,k] fp32, want_fwd, want_dgrad, cout_pad)]"""
        assert self.DTYPE.itemsize == 48
        table = np.zeros(len(entries), dtype=self.DTYPE)
        self.key = tuple(w.data_ptr() for _, w, _, _, _ in entries)
        self.fwd, self.dgrad = {}, {}
        blocks = 0
        for i, (key, w, want_f, want_d, cp) in enumerate(entries):
            cout, cin, k, _ = w.shape
            cp = max(cout, cp)
            if cin % 2 or cp % 2 or k not in (1, 3) or w.dtype != torch.float32 or not w.is_contiguous():
                raise ValueError('PackPlan: unsupported weight %s %s' % (key, tuple(w.shape)))
            f = torch.empty(cout, k, k, cin, dtype=torch.float16, device=device) if want_f else None
            d = torch.empty(cin, k, k, cp, dtype=torch.float16, device=device) if want_d else None
            cib = -(-cin // (32 if k == 3 else 256))
            table[i] = (w.data_ptr(), 0 if f is None else f.data_ptr(), 0 if d is None else d.data_ptr(), cout, cin, k, cp, blocks, cib)
            blocks += -(-cp // 64) * cib
            if f is not None:
                self.fwd[key] = f
            if d is not None:
                self.dgrad[key] = d
        self.blocks = blocks
        self.count = len(entries)
        self.table = torch.from_numpy(table.view(np.uint8).copy()).to(device)

    def run(self):
        ops.call('yb_pack_weights_batch', self.table, self.count, self.blocks)


class DarknetTrainer(object):
    def __init__(self, engine, grad_scale=16384.0):
        self.engine = engine
        self.grad_scale = float(grad_scale)
        self.sums = {}       # per-unit double[2C] accumulators (self-cleaning)
        self.wd_cache = {}   # dgrad weight buffers per unit (contents re-packed every step)
        # data parallel: b200.ddp.GradientAllReducer attached by train.iterate; every gradient kernel writes into the reducer-visible
        # arena and reports it (`_emit`) so the bucket's all-reduce starts while the rest of the backward chain is still running
        self.slope = SLOPE     # negative slope of the activation (LeakyReLU(0.1) for the yolo2 backbones, 0 = ReLU for MobileNet)
        self.reducer = None
        self.arena = None
        self.found_inf = None  # device float[1]: 1 when the last backward produced a non-finite gradient (then zeroed), see backward()
        self._arenas = {}      # one per (device, parameter set, reducer): CUDA graphs keep writing the arena they were captured with
        self._main = None
        # BN batch statistics in the conv epilogue (yb_conv_bn_act_stats_fwd) instead of yb_bn_stats; YB_FUSE_STATS=0 for A/B runs
        self.fuse_stats = os.environ.get('YB_FUSE_STATS', '1') != '0'
        self._fused_stats = False
        # weight gradients on a second stream (overlap with the BatchNorm backward chain); YB_WGRAD_STREAM=0 for A/B runs
        self.wgrad_stream = os.environ.get('YB_WGRAD_STREAM', '1') != '0'
        self._side_streams = {}
        self._side_busy = False
        self._pack_plan = None
        self._tracked = []

    def _bump_tracked(self):
        """`num_batches_tracked += 1` of every BatchNorm of the step as ONE multi-tensor kernel instead of one tiny launch per layer."""
        if self._tracked:
            torch._foreach_add_(self._tracked, 1)
            self._tracked = []

    # ---- helpers -------------------------------------------------------------------------------------
    def _slope(self, u):
        """Activation slope of a unit's train-mode BatchNorm + activation: its own `train_slope` (ResNet units: 0 = ReLU, 1 = identity),
        else the trainer's."""
        return getattr(u, 'train_slope', self.slope)

    @staticmethod
    def _pnames(key, u):
        """State-dict names of a unit's (conv weight, BN weight, BN bias): `key.conv.weight`, `key.bn.*` unless the unit carries `pnames`."""
        return getattr(u, 'pnames', None) or (key + '.conv.weight', key + '.bn.weight', key + '.bn.bias')

    def _emit(self, name, grads):
        if self.reducer is not None:
            dev = grads[name].device
            side = self._side_streams.get(dev) if self._side_busy else None
            self.reducer.on_grad(name, grads[name], streams=(self._main, side))

    def grad_order(self):
        """State-dict names of all parameters in the order the backward chain produces their gradients."""
        eng = self.engine
        names = ['layers3.1.conv.bias', 'layers3.1.conv.weight']
        for key in ['layers3.0'] + list(reversed(eng._k2)) + ['passthrough'] + list(reversed(eng._k1)):
            names += [key + '.bn.weight', key + '.bn.bias', key + '.conv.weight']
        return names

    def _ensure_arena(self, dnn, device):
        """Persistent flat fp32 gradient buffer (b200.ddp.GradArena): gradient kernels write straight into their slots, `.grad`
        of every parameter is a view of it, buckets of it are all-reduced in place."""
        params = dict(dnn.named_parameters())
        key = (str(device), tuple((n, tuple(p.shape)) for n, p in params.items()), id(self.reducer))
        self.arena = self._arenas.get(key)
        if self.arena is None:
            order = [n for n in self.grad_order() if n in params]
            if set(order) != set(params):
                raise RuntimeError('Darknet trainer: unexpected parameter set %s' % sorted(set(params) ^ set(order))[:4])
            bucket_bytes = self.reducer.bucket_bytes if self.reducer is not None else (32 << 20)
            self.arena = self._arenas[key] = _ddp.GradArena([(n, tuple(params[n].shape)) for n in order], device, bucket_bytes)
            if self.reducer is not None:
                self.reducer.attach(self.arena)
        return self.arena

    @property
    def _unscale(self):
        """Inverse loss scale, with the 1 / world of the data-parallel gradient average folded in."""
        return 1.0 / (self.grad_scale * (self.reducer.grad_divisor if self.reducer is not None else 1.0))

    def _repack(self, device):
        """All kernel operands that depend on the parameters, re-derived for this step: one batched pack launch for the fp16 weight
        operands (forward + data gradient); the first layer reads its fp32 weights and the head its fp32 bias in place.  The eval-mode
        BatchNorm fold is NOT refreshed here (training uses batch statistics); `Darknet.train(False)` invalidates it."""
        eng = self.engine
        units, keys = eng.all_units(), eng.unit_keys()
        ptrs = tuple(u.conv.weight.data_ptr() for u in units[1:])
        plan = self._pack_plan
        if plan is None or plan.key != ptrs or plan.table.device != device:
            entries = []
            for u, key in zip(units[1:], keys[1:]):
                cpad = (u.cout + 31) // 32 * 32 if u.bn is None else 0          # the head's filters are padded to the dz buffer's width
                entries.append((key, u.conv.weight.detach(), True, True, cpad))
            plan = self._pack_plan = PackPlan(entries, device)
        plan.run()
        units[0].w16 = units[0].conv.weight.detach().contiguous()
        for u, key in zip(units[1:], keys[1:]):
            u.w16 = plan.fwd[key]
            u._wver = None                      # the eval path re-checks (and may re-pack into its own buffer)
            self.wd_cache[key] = plan.dgrad[key]
        head = units[-1]
        if head.bn is None:
            one, _ = self._ones(head.cout, device)
            head.scale = one
            head.shift = head.conv.bias.detach() if head.conv.bias is not None else self._ones(head.cout, device)[1]
            head._bver = None

    def _sums(self, key, channels, device):
        t = self.sums.get(key)
        if t is None or t.numel() != 2 * channels or t.device != device:
            t = torch.zeros(2 * channels, dtype=torch.float64, device=device)
            self.sums[key] = t
        return t

    def _ones(self, c, device):
        key = ('ones', c, str(device))
        t = self.sums.get(key)
        if t is None:
            t = (torch.ones(c, dtype=torch.float32, device=device), torch.zeros(c, dtype=torch.float32, device=device))
            self.sums[key] = t
        return t

    def _raw_conv(self, u, src, out=None, key=None, **kw):
        """Raw conv output z.  With `key` (a BN unit of the generic kernel) the batch statistics are accumulated in the
        conv epilogue into the unit's double accumulators, so `_bn_forward` does not read z again."""
        one, zero = self._ones(u.cout, src.device)
        self._fused_stats = False
        c32 = u.cin == 32 and u.ksize == 3 and u.cout <= 64          # the halo-tile kernel: fused statistics need exact 16 x 8 tiling
        if key is not None and self.fuse_stats and not (c32 and (src.shape[1] % 16 or src.shape[2] % 8)):
            self._fused_stats = True
            return ops.conv_bn_act_stats(src, u.w16, one, zero, 1.0, self._sums(('f', key), u.cout, src.device), out=out)
        return ops.conv_bn_act(src, u.w16, one, zero, 1.0, out=out, **kw)

    def _bn_forward(self, key, u, z, rows):
        bn = u.bn
        c = u.cout
        dev = z.device
        sums = self._sums(('f', key), c, dev)
        mean = torch.empty(c, dtype=torch.float32, device=dev)
        invstd = torch.empty(c, dtype=torch.float32, device=dev)
        if not getattr(self, '_fused_stats', False):
            ops.call('yb_bn_stats', z, z.shape[-1], rows, c, sums)
        self._fused_stats = False
        ops.call('yb_bn_finalize', sums, rows, c, float(bn.eps), float(bn.momentum), bn.running_mean, bn.running_var, mean, invstd)
        if bn.num_batches_tracked is not None:
            self._tracked.append(bn.num_batches_tracked)      # incremented together at the end of the forward pass (_bump_tracked)
        u._bver = None      # running stats changed behind torch's version counter: re-fold on the next eval forward
        return mean, invstd

    def _apply(self, u, z, mean, invstd, b, h, w, pool, out=None, a_off=0):
        c = u.cout
        if out is None:
            out = torch.empty(b, h // 2 if pool else h, w // 2 if pool else w, c, dtype=torch.float16, device=z.device)
        ops.call('yb_bn_act_apply', z, z.shape[-1], mean, invstd, u.bn.weight.detach(), u.bn.bias.detach(), self._slope(u), out, out.shape[-1], a_off,
                 b, h, w, c, int(pool))
        return out

    def _bn_backward(self, key, s, b, grads, da, dap, dz, ld_dz):
        u = s.u
        c = u.cout
        dev = s.z.device
        sums = self._sums(('b', key), c, dev)
        args = (s.z, s.z.shape[-1], s.mean, s.invstd, u.bn.weight.detach(), u.bn.bias.detach(), self._slope(u), da, 0 if da is None else da.shape[-1], 0, dap,
                0 if dap is None else dap.shape[-1], 0, b, s.h, s.w, c, 1 if dap is not None else 0, sums)
        ops.call('yb_bn_act_bwd', 0, *args, None, 0, 1)
        ops.call('yb_bn_act_bwd', 1, *args, dz, ld_dz, 1)
        _, gname, bname = self._pnames(key, u)
        dgamma, dbeta = self.arena.views[gname], self.arena.views[bname]
        ops.call('yb_bn_param_grad', sums, c, dgamma, dbeta, 1, self._unscale)
        grads[gname], grads[bname] = dgamma, dbeta
        self._emit(gname, grads)
        self._emit(bname, grads)

    # ---- forward -------------------------------------------------------------------------------------
    def forward(self, x):
        self._tracked = []
        eng = self.engine
        if not x.is_cuda:
            raise RuntimeError('Darknet training: input must be a CUDA tensor')
        b, _, h, w = x.shape
        x = x.contiguous().float()
        if eng.precision != 'fast':
            raise RuntimeError("Darknet training uses fp16 operands with fp32 accumulation; precision='strict' is an inference mode "
                               "(call dnn.engine.set_precision('fast') before train())")
        self._repack(x.device)       # every step: do not trust parameter version counters (fused optimizers do not advance them)
        for u in eng.all_units()[:-1]:
            if u.bn is None:
                raise NotImplementedError('training path requires batch_norm/enable = 1')
        dev = x.device
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w = x, b, h, w
        saved.units = {}

        def record(key, u, ain, z, mean, invstd, hh, ww, pooled):
            s = _Saved()
            s.u, s.ain, s.z, s.mean, s.invstd, s.h, s.w, s.pooled = u, ain, z, mean, invstd, hh, ww, pooled
            saved.units[key] = s

        # layers1.0 (direct from the fp32 image)
        u0 = eng.units1[0]
        z = torch.empty(b, h, w, u0.cout, dtype=torch.float16, device=dev)
        if self.fuse_stats and h % 32 == 0 and w % 16 == 0:
            # batch statistics accumulated by the conv kernel's copy-out loop: z is not read again for them
            ops.call('yb_conv0_raw_stats_fwd', x, u0.w16, z, self._sums(('f', 'layers1.0'), u0.cout, dev), b, h, w, u0.cout)
            self._fused_stats = True
        else:
            ops.call('yb_conv0_raw_fwd', x, u0.w16, z, b, h, w, u0.cout)
        mean, invstd = self._bn_forward('layers1.0', u0, z, b * h * w)
        cur = self._apply(u0, z, mean, invstd, b, h, w, True)
        record('layers1.0', u0, None, z, mean, invstd, h, w, True)
        hh, ww = h // 2, w // 2
        for u, key, pooled in zip(eng.units1[1:], eng._k1[1:], eng.pools1[1:]):
            z = self._raw_conv(u, cur, key=key)
            mean, invstd = self._bn_forward(key, u, z, b * hh * ww)
            last = key == eng._k1[-1]
            a = self._apply(u, z, mean, invstd, b, hh, ww, pooled and not last)
            record(key, u, cur, z, mean, invstd, hh, ww, pooled)
            cur = a
            if pooled and not last:
                hh, ww = hh // 2, ww // 2
        x1 = cur                                    # layers1.16 output, unpooled (hh x ww)
        # passthrough -> reorg -> concat[..., :4*Cpt]
        upt = eng.unit_pt
        cat_ch = upt.cout * 4 + eng.units2[-1].cout
        cat = torch.empty(b, hh // 2, ww // 2, cat_ch, dtype=torch.float16, device=dev)
        z = self._raw_conv(upt, x1, key='passthrough')
        mean, invstd = self._bn_forward('passthrough', upt, z, b * hh * ww)
        a_pt = self._apply(upt, z, mean, invstd, b, hh, ww, False)
        record('passthrough', upt, x1, z, mean, invstd, hh, ww, False)
        ops.reorg_f16(a_pt, cat, 0)
        # trunk
        cur = ops.maxpool2x2(x1)
        h32, w32 = hh // 2, ww // 2
        for i, (u, key) in enumerate(zip(eng.units2, eng._k2)):
            z = self._raw_conv(u, cur, key=key)
            mean, invstd = self._bn_forward(key, u, z, b * h32 * w32)
            if i == len(eng.units2) - 1:
                self._apply(u, z, mean, invstd, b, h32, w32, False, out=cat, a_off=upt.cout * 4)
                a = cat
            else:
                a = self._apply(u, z, mean, invstd, b, h32, w32, False)
            record(key, u, cur, z, mean, invstd, h32, w32, False)
            cur = a
        saved.keys2 = list(eng._k2[:len(eng.units2)])
        u30, u31 = eng.units3
        z = self._raw_conv(u30, cat, key='layers3.0')
        mean, invstd = self._bn_forward('layers3.0', u30, z, b * h32 * w32)
        a30 = self._apply(u30, z, mean, invstd, b, h32, w32, False)
        record('layers3.0', u30, cat, z, mean, invstd, h32, w32, False)
        feature = ops.conv_bn_act(a30, u31.w16, u31.scale, u31.shift, 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a30, saved.cat, saved.x1, saved.h16, saved.w16, saved.h32, saved.w32 = a30, cat, x1, hh, ww, h32, w32
        self._bump_tracked()
        return feature, saved

    # ---- backward ------------------------------------------------------------------------------------
    def _wd(self, key, u, cout_pad=0):
        """Data-gradient operand of a unit (rotated, transposed fp16 weights), re-packed every step into a reused buffer."""
        w = u.conv.weight
        cout, cin, k, _ = w.shape
        cp = max(cout, cout_pad)
        wd = self.wd_cache.get(key)
        plan = self._pack_plan
        if plan is not None and wd is not None and plan.dgrad.get(key) is wd and wd.shape == (cin, k, k, cp):
            return wd                         # packed by this step's batched launch (_repack)
        if wd is None or wd.shape != (cin, k, k, cp) or wd.device != w.device:
            wd = torch.empty(cin, k, k, cp, dtype=torch.float16, device=w.device)
            self.wd_cache[key] = wd
        ops.call('yb_pack_weight_dgrad_f16', w.detach().contiguous(), wd, cout, cin, k, cp)
        return wd

    def _wgrad(self, u, ain, dz, b, hh, ww, grads, name, cout=None):
        """Weight gradient of one unit.  It depends only on (ain, dz) and nothing downstream depends on it before the
        optimizer, so it is issued on a second stream: the tensor-bound wgrad kernel then overlaps the HBM-bound
        BatchNorm backward of the next unit (and its data gradient) instead of queueing in front of them.  The fork /
        join is plain stream-event ordering, so it is captured as parallel branches of the step's CUDA graph."""
        cout = u.cout if cout is None else cout
        cin, k = u.cin, u.ksize
        dev = dz.device
        side = self._side(dev)
        if side is not None:
            main = torch.cuda.current_stream(dev)
            try:
                fork = torch.cuda.Event()
                fork.record(main)
                side.wait_event(fork)
            except Exception as ex:
                raise RuntimeError('weight-gradient fork for %s failed (main %r, side %r): %s' % (name, main, side, ex)) from ex
            dz.record_stream(side)          # dz / ain are main-stream allocations still read by the side stream
            ain.record_stream(side)
            self._side_busy = True
        with torch.cuda.stream(side) if side is not None else _NullCtx():
            dw_krsc = torch.empty(cout, k, k, cin, dtype=torch.float32, device=dev)
            ops.call('yb_conv_wgrad', ain, dz, dw_krsc, b, hh, ww, cin, cout, k, ain.shape[-1], dz.shape[-1])
            wname = self._pnames(name, u)[0]
            dw = self.arena.views[wname]                                                     # [cout, cin, k, k] slot of the gradient arena
            ops.call('yb_unpack_wgrad', dw_krsc, dw, cout, cin, k, self._unscale)            # layout change + inverse loss scale (/ world)
            grads[wname] = dw
            self._emit(wname, grads)

    def _side(self, dev):
        # only while the step is being captured into a CUDA graph: in eager mode the step is host-bound and the extra
        # event / stream bookkeeping costs more (measured +2.6 ms) than the overlap gains (0.1 ms)
        if not self.wgrad_stream or not torch.cuda.is_current_stream_capturing():
            return None
        st = self._side_streams.get(dev)
        if st is None:
            st = torch.cuda.Stream(device=dev)
            self._side_streams[dev] = st
        return st

    def _join(self, dev):
        """Main stream waits for everything issued on the wgrad stream (end of backward: the optimizer reads the grads)."""
        if self._side_busy:
            torch.cuda.current_stream(dev).wait_stream(self._side_streams[dev])
            self._side_busy = False

    def _unit_backward(self, key, s, b, grads, da=None, da_off=0, dap=None, dap_off=0, need_dgrad=True):
        """Backward of one BN unit; returns the gradient w.r.t. the unit's input activation (or None)."""
        u = s.u
        c = u.cout
        dev = s.z.device
        window = 1 if (dap is not None) else 0
        sums = self._sums(('b', key), c, dev)
        bnw, bnb = u.bn.weight.detach(), u.bn.bias.detach()
        args = (s.z, s.z.shape[-1], s.mean, s.invstd, bnw, bnb, self._slope(u), da, 0 if da is None else da.shape[-1], da_off, dap,
                0 if dap is None else dap.shape[-1], dap_off, b, s.h, s.w, c, window, sums)
        ops.call('yb_bn_act_bwd', 0, *args, None, 0, 1)
        _, gname, bname = self._pnames(key, u)
        dgamma = self.arena.views[gname]
        dbeta = self.arena.views[bname]
        dz = torch.empty(b, s.h, s.w, c, dtype=torch.float16, device=dev)
        ops.call('yb_bn_act_bwd', 1, *args, dz, c, 1)
        ops.call('yb_bn_param_grad', sums, c, dgamma, dbeta, 1, self._unscale)     # un-scales (/ world), then clears the accumulators
        grads[gname] = dgamma
        grads[bname] = dbeta
        self._emit(gname, grads)
        self._emit(bname, grads)
        if s.ain is None:
            return dz
        self._wgrad(u, s.ain, dz, b, s.h, s.w, grads, key)
        if not need_dgrad:
            return None
        one, zero = self._ones(u.cin, dev)
        return ops.conv_bn_act(dz, self._wd(key, u), one, zero, 1.0)

    def backward(self, saved, dfeature, dnn=None):
        """dfeature: fp32 NCHW gradient of the loss w.r.t. the head output.  Returns {state_dict key: fp32 grad}: views of the
        persistent gradient arena, already averaged over the data-parallel ranks when a reducer is attached."""
        eng = self.engine
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._ensure_arena(dnn if dnn is not None else self._dnn, dev)
        self._main = torch.cuda.current_stream(dev)
        u30, u31 = eng.units3
        h32, w32 = saved.h32, saved.w32
        chead = u31.cout
        cpad = (chead + 31) // 32 * 32
        # head: bias gradient from the unscaled fp32 gradient, dz scaled into fp16
        dzh = torch.empty(b, h32, w32, cpad, dtype=torch.float16, device=dev)
        dbias = self.arena.views['layers3.1.conv.bias']
        scaled = (dfeature.contiguous().float() * self.grad_scale)
        ops.call('yb_head_grad_prepare', scaled, dzh, dbias, b, chead, cpad, h32 * w32)
        grads['layers3.1.conv.bias'] = dbias.mul_(self._unscale)
        self._emit('layers3.1.conv.bias', grads)
        self._wgrad(u31, saved.a30, dzh, b, h32, w32, grads, 'layers3.1', cout=chead)
        one, zero = self._ones(u31.cin, dev)
        da = ops.conv_bn_act(dzh, self._wd('layers3.1', u31, cpad), one, zero, 1.0)
        # layers3.0 -> gradient of the concat buffer
        dcat = self._unit_backward('layers3.0', saved.units['layers3.0'], b, grads, da=da)
        cpt4 = eng.unit_pt.cout * 4
        # trunk: layers2.* (the last one reads its gradient from channels [cpt4, ...) of dcat)
        g, g_off = dcat, cpt4
        for key in reversed(saved.keys2):
            g = self._unit_backward(key, saved.units[key], b, grads, da=g, da_off=g_off)
            g_off = 0
        d_x1_pool = g                                              # [B,h32,w32,C16]
        # passthrough branch
        d_apt = torch.empty(b, saved.h16, saved.w16, eng.unit_pt.cout, dtype=torch.float16, device=dev)
        ops.call('yb_reorg_bwd_f16', dcat, dcat.shape[-1], 0, d_apt, b, saved.h16, saved.w16, eng.unit_pt.cout)
        d_x1 = self._unit_backward('passthrough', saved.units['passthrough'], b, grads, da=d_apt)
        # layers1.* in reverse; the branch point layers1.16 gets both gradients
        keys1 = eng._k1
        g_da, g_dap = d_x1, d_x1_pool
        for key in reversed(keys1[1:]):
            s = saved.units[key]
            g = self._unit_backward(key, s, b, grads, da=g_da, dap=g_dap)
            prev_key = keys1[keys1.index(key) - 1]
            prev_pooled = saved.units[prev_key].pooled
            g_da, g_dap = (None, g) if prev_pooled else (g, None)
        # layers1.0: weight gradient straight from the fp32 image
        s0 = saved.units['layers1.0']
        dw0 = self.arena.views['layers1.0.conv.weight']
        if g_da is None and g_dap is not None and saved.h % 8 == 0 and saved.w % 32 == 0 and os.environ.get('YB_CONV0_WGRAD_FUSED', '1') != '0':
            # reduce pass of the BatchNorm backward, then the weight-gradient kernel forms dz itself (in shared memory, from z and the pooled
            # gradient): the 2 x 708 MB (B = 64 @ 416) write + read of dz and one launch disappear
            u0 = s0.u
            sums = self._sums(('b', 'layers1.0'), u0.cout, dev)
            bnw, bnb = u0.bn.weight.detach(), u0.bn.bias.detach()
            ops.call('yb_bn_act_bwd', 0, s0.z, s0.z.shape[-1], s0.mean, s0.invstd, bnw, bnb, self.slope, None, 0, 0, g_dap, g_dap.shape[-1], 0,
                     b, s0.h, s0.w, u0.cout, 1, sums, None, 0, 1)
            ops.call('yb_conv0_wgrad_bn', saved.x, s0.z, g_dap, g_dap.shape[-1], 0, s0.mean, s0.invstd, bnw, bnb, self.slope, sums, dw0, b, saved.h, saved.w)
            dgamma, dbeta = self.arena.views['layers1.0.bn.weight'], self.arena.views['layers1.0.bn.bias']
            ops.call('yb_bn_param_grad', sums, u0.cout, dgamma, dbeta, 1, self._unscale)          # also clears the accumulators (after their last reader)
            grads['layers1.0.bn.weight'], grads['layers1.0.bn.bias'] = dgamma, dbeta
            self._emit('layers1.0.bn.weight', grads)
            self._emit('layers1.0.bn.bias', grads)
        else:
            dz0 = self._unit_backward('layers1.0', s0, b, grads, da=g_da, dap=g_dap)
            ops.call('yb_conv0_wgrad', saved.x, dz0, dw0, b, saved.h, saved.w)
        grads['layers1.0.conv.weight'] = dw0.mul_(self._unscale)
        self._emit('layers1.0.conv.weight', grads)
        self._join(dev)
        if self.reducer is not None:
            self.reducer.finish()          # main stream waits for every bucket's all-reduce (no host wait)
        # fp16 gradient overflow guard (after the exchange, so every rank takes the same decision): `found_inf` is raised and the
        # gradients are zeroed instead of poisoning the optimizer state; train.iterate hands the flag to optimizers that can skip
        if self.found_inf is None or self.found_inf.device != dev:
            self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)      # 0-dim like GradScaler's (fused optimizers subtract it from their step counters)
        ops.call('yb_grad_guard', self.arena.flat, self.arena.flat.numel(), self.found_inf, 1)
        return grads


class TinyTrainer(DarknetTrainer):
    """Training-mode forward / backward of `model.yolo2.Tiny` (reference model/yolo2.py:140-173) on the same kernels: a plain chain of
    conv units, five of them followed by MaxPool2d(2) (fused into the normalise kernel), the sixth by ConstantPad2d + MaxPool2d(2, stride 1).

    The 16-channel first layer rides on the 32-filter first-layer kernels: its weights are zero-padded to 32 outputs, BatchNorm runs over the
    16 real channels of the 32-wide buffers (the kernels take the channel count and the pixel pitch separately), the padding channels stay
    exactly zero, and the second unit's weights are zero-padded on the input side to match (its weight gradient is cut back to 16 inputs)."""

    def __init__(self, dnn, grad_scale=16384.0):
        DarknetTrainer.__init__(self, _TinyEngineView(dnn), grad_scale)
        self.dnn = dnn
        self._zero_bufs = {}

    def grad_order(self):
        keys = [key for key, _, _ in self.dnn.unit_keys()]
        names = [keys[-1] + '.conv.bias', keys[-1] + '.conv.weight']
        for key in reversed(keys[:-1]):
            names += [key + '.bn.weight', key + '.bn.bias', key + '.conv.weight']
        return names

    def _zeros(self, tag, shape, device):
        """Persistent zero-initialised fp16 buffer whose padding channels are never written."""
        t = self._zero_bufs.get(tag)
        if t is None or tuple(t.shape) != tuple(shape) or t.device != device:
            t = torch.zeros(shape, dtype=torch.float16, device=device)
            self._zero_bufs[tag] = t
        return t

    def forward(self, x):
        self._tracked = []
        if not x.is_cuda:
            raise RuntimeError('Tiny training: input must be a CUDA tensor')
        b, _, h, w = x.shape
        x = x.contiguous().float()
        dev = x.device
        plan = self.dnn.unit_keys()
        units = [u for _, u, _ in plan]
        for i, u in enumerate(units):
            u.refresh(first_layer=(i == 0), force=True)
            if u.bn is None and i != len(units) - 1:
                raise NotImplementedError('training path requires batch_norm/enable = 1')
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w, saved.units, saved.order = x, b, h, w, {}, []
        # unit 0: 3 -> C0 (<= 32) on the first-layer kernel, filters zero-padded to 32
        key0, u0, after0 = plan[0]
        c0 = u0.cout
        if c0 > 32 or after0 != 'pool':
            raise RuntimeError('Tiny: the first unit must have <= 32 filters and be followed by MaxPool2d(2)')
        w0 = torch.zeros(32, 3, 3, 3, dtype=torch.float32, device=dev)
        w0[:c0].copy_(u0.conv.weight.detach())
        z = self._zeros(('z0', b, h, w), (b, h, w, 32), dev)
        ops.call('yb_conv0_raw_fwd', x, w0, z, b, h, w, 32)
        mean, invstd = self._bn_forward(key0, u0, z, b * h * w)
        cur = self._zeros(('a0', b, h, w), (b, h // 2, w // 2, 32), dev)
        self._apply(u0, z, mean, invstd, b, h, w, True, out=cur)
        s = _Saved()
        s.u, s.ain, s.z, s.mean, s.invstd, s.h, s.w, s.pooled = u0, None, z, mean, invstd, h, w, True
        saved.units[key0] = s
        saved.order.append((key0, after0))
        hh, ww, chan = h // 2, w // 2, 32
        for key, u, after in plan[1:-1]:
            if u.cin != chan:
                # input side zero-padded to the producer's buffer width (unit 1: 16 -> 32)
                wp = torch.zeros(u.cout, chan, u.ksize, u.ksize, dtype=torch.float32, device=dev)
                wp[:, :u.cin].copy_(u.conv.weight.detach())
                w16 = ops.pack_weight_f16(wp, 0)
            else:
                w16 = u.w16
            one, zero = self._ones(u.cout, dev)
            if self.fuse_stats and not (chan == 32 and u.ksize == 3 and u.cout <= 64):
                z = ops.conv_bn_act_stats(cur, w16, one, zero, 1.0, self._sums(('f', key), u.cout, dev))
                self._fused_stats = True
            else:
                z = ops.conv_bn_act(cur, w16, one, zero, 1.0)
                self._fused_stats = False
            mean, invstd = self._bn_forward(key, u, z, b * hh * ww)
            a = self._apply(u, z, mean, invstd, b, hh, ww, after == 'pool')
            s = _Saved()
            s.u, s.ain, s.z, s.mean, s.invstd, s.h, s.w, s.pooled, s.cin_pad = u, cur, z, mean, invstd, hh, ww, after == 'pool', chan
            if after == 'pool':
                hh, ww = hh // 2, ww // 2
            elif after == 'pool_s1':
                s.a_unpooled = a
                a = ops.maxpool2x2_s1(a)
            saved.units[key] = s
            saved.order.append((key, after))
            cur, chan = a, u.cout
        key_h, u_h, _ = plan[-1]
        feature = ops.conv_bn_act(cur, u_h.w16, u_h.scale, u_h.shift, 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww, saved.head = cur, hh, ww, (key_h, u_h)
        self._bump_tracked()
        return feature, saved

    def backward(self, saved, dfeature, dnn=None):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._ensure_arena(self.dnn, dev)
        self._main = torch.cuda.current_stream(dev)
        self._x = saved.x
        key_h, u_h = saved.head
        hh, ww = saved.hh, saved.ww
        chead = u_h.cout
        cpad = (chead + 31) // 32 * 32
        dzh = torch.empty(b, hh, ww, cpad, dtype=torch.float16, device=dev)
        dbias = self.arena.views[key_h + '.conv.bias']
        ops.call('yb_head_grad_prepare', dfeature.contiguous().float() * self.grad_scale, dzh, dbias, b, chead, cpad, hh * ww)
        grads[key_h + '.conv.bias'] = dbias.mul_(self._unscale)
        self._emit(key_h + '.conv.bias', grads)
        self._wgrad(u_h, saved.a_last, dzh, b, hh, ww, grads, key_h, cout=chead)
        one, zero = self._ones(u_h.cin, dev)
        g = ops.conv_bn_act(dzh, self._wd(key_h, u_h, cpad), one, zero, 1.0)
        for key, after in reversed(saved.order):
            s = saved.units[key]
            u = s.u
            if after == 'pool_s1':
                da = torch.empty_like(s.a_unpooled)
                ops.call('yb_maxpool2x2_s1_bwd_f16', s.a_unpooled, g, da, b, s.h, s.w, u.cout)
                g = da
            pooled = after == 'pool'
            if s.ain is None:
                # first layer: dz into the 32-wide zero-padded buffer the first-layer weight-gradient kernel reads
                g = self._tiny_unit0_backward(key, s, b, grads, g)
                break
            if getattr(s, 'cin_pad', u.cin) != u.cin:
                g = self._tiny_padded_unit_backward(key, s, b, grads, g, pooled)
            else:
                g = self._unit_backward(key, s, b, grads, da=None if pooled else g, dap=g if pooled else None)
        self._join(dev)
        if self.reducer is not None:
            self.reducer.finish()
        if self.found_inf is None or self.found_inf.device != dev:
            self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)
        ops.call('yb_grad_guard', self.arena.flat, self.arena.flat.numel(), self.found_inf, 1)
        return grads

    def _tiny_unit0_backward(self, key, s, b, grads, g):
        dev = s.z.device
        dz = self._zeros(('dz0', b, s.h, s.w), (b, s.h, s.w, 32), dev)          # channels >= cout stay zero
        self._bn_backward(key, s, b, grads, None, g, dz, 32)
        dw32 = torch.empty(32, 3, 3, 3, dtype=torch.float32, device=dev)
        ops.call('yb_conv0_wgrad', self._x, dz, dw32, b, s.h, s.w)
        dw = self.arena.views[key + '.conv.weight']
        dw.copy_(dw32[:s.u.cout]).mul_(self._unscale)
        grads[key + '.conv.weight'] = dw
        self._emit(key + '.conv.weight', grads)
        return None

    def _tiny_padded_unit_backward(self, key, s, b, grads, g, pooled):
        """Unit whose input buffer is wider than its Cin (zero-padded): the weight gradient is computed over the padded width and cut back."""
        u = s.u
        dev = s.z.device
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=dev)
        self._bn_backward(key, s, b, grads, None if pooled else g, g if pooled else None, dz, u.cout)
        k, cp = u.ksize, s.cin_pad
        dw_krsc = torch.empty(u.cout, k, k, cp, dtype=torch.float32, device=dev)
        ops.call('yb_conv_wgrad', s.ain, dz, dw_krsc, b, s.h, s.w, cp, u.cout, k, s.ain.shape[-1], dz.shape[-1])
        full = torch.empty(u.cout, cp, k, k, dtype=torch.float32, device=dev)
        ops.call('yb_unpack_wgrad', dw_krsc, full, u.cout, cp, k, self._unscale)
        dw = self.arena.views[key + '.conv.weight']
        dw.copy_(full[:, :u.cin])
        grads[key + '.conv.weight'] = dw
        self._emit(key + '.conv.weight', grads)
        one, zero = self._ones(u.cin, dev)
        return ops.conv_bn_act(dz, self._wd(key, u), one, zero, 1.0)      # [B, h, w, Cin]: the producer's real channels


class _TinyEngineView(object):
    """The two things DarknetTrainer reads from an engine, for a plain chain."""
    precision = 'fast'

    def __init__(self, dnn):
        self._dnn = dnn


class _BNUnit(object):
    """What the BatchNorm helpers read of a unit, for layers that are not wgmma conv units (first conv, depthwise)."""

    def __init__(self, bn, cout):
        self.bn, self.cout = bn, cout
        self._bver = None


class MobileNetTrainer(DarknetTrainer):
    """Training-mode forward / backward of `model.mobilenet.MobileNet` (reference model/mobilenet.py:25-85): conv_bn(3, 32, stride 2), thirteen
    [depthwise 3x3 (stride 1 or 2) + BN + ReLU, pointwise 1x1 + BN + ReLU] units, a 1x1 head with bias.  Pointwise convs, their weight /
    data gradients and the head run on the wgmma kernels of the Darknet path; the depthwise and first-layer kernels are HBM-bound CUDA-core
    kernels (csrc/mobilenet_ops.cu).  BatchNorm momentum is the PyTorch default 0.1 here (read from the modules), the activation ReLU."""

    def __init__(self, dnn, grad_scale=16384.0):
        DarknetTrainer.__init__(self, _TinyEngineView(dnn), grad_scale)
        self.dnn = dnn
        self.slope = 0.0
        self._units = None

    def _plan(self):
        if self._units is None:
            from . import engine as _engine
            layers = list(self.dnn.layers)
            first = layers[0]
            plan = dict(first=_BNUnit(first.bn, first.conv.weight.shape[0]), units=[], head=layers[-1])
            for i, unit in enumerate(layers[1:-1], 1):
                ch = unit.dw.conv.weight.shape[0]
                plan['units'].append(dict(key='layers.%d' % i, dw=_BNUnit(unit.dw.bn, ch), dw_conv=unit.dw.conv, stride=unit.dw.conv.stride[0],
                                          pw=_engine.ConvUnit(unit.pw.conv, unit.pw.bn, True)))
            self._units = plan
        return self._units

    def grad_order(self):
        names = ['layers.14.bias', 'layers.14.weight']
        for i in range(13, 0, -1):
            names += ['layers.%d.pw.bn.weight' % i, 'layers.%d.pw.bn.bias' % i, 'layers.%d.pw.conv.weight' % i,
                      'layers.%d.dw.bn.weight' % i, 'layers.%d.dw.bn.bias' % i, 'layers.%d.dw.conv.weight' % i]
        return names + ['layers.0.bn.weight', 'layers.0.bn.bias', 'layers.0.conv.weight']

    def forward(self, x):
        self._tracked = []
        if not x.is_cuda:
            raise RuntimeError('MobileNet training: input must be a CUDA tensor')
        b, _, h, w = x.shape
        x = x.contiguous().float()
        dev = x.device
        plan = self._plan()
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w, saved.units = x, b, h, w, []
        first = self.dnn.layers[0]
        if first.conv.weight.shape[0] != 32:
            raise ValueError('MobileNet: the first layer must have 32 output channels')
        hh, ww = h // 2, w // 2
        z = torch.empty(b, hh, ww, 32, dtype=torch.float16, device=dev)
        ops.call('yb_mb_conv0_raw_fwd', x, first.conv.weight.detach().contiguous(), z, b, h, w)
        u0 = plan['first']
        mean, invstd = self._bn_forward('layers.0', u0, z, b * hh * ww)
        cur = self._apply(u0, z, mean, invstd, b, hh, ww, False)
        s0 = _Saved()
        s0.u, s0.z, s0.mean, s0.invstd, s0.h, s0.w = u0, z, mean, invstd, hh, ww
        saved.first = s0
        for rec in plan['units']:
            key, stride = rec['key'], rec['stride']
            ch = rec['dw'].cout
            oh, ow = hh // stride, ww // stride
            # depthwise
            zd = torch.empty(b, oh, ow, ch, dtype=torch.float16, device=dev)
            wd = rec['dw_conv'].weight.detach().contiguous().view(ch, 9)
            ops.call('yb_dwconv3x3_raw_fwd', cur, wd, zd, b, hh, ww, ch, stride)
            mean, invstd = self._bn_forward(key + '.dw', rec['dw'], zd, b * oh * ow)
            ad = self._apply(rec['dw'], zd, mean, invstd, b, oh, ow, False)
            sd = _Saved()
            sd.u, sd.ain, sd.z, sd.mean, sd.invstd, sd.h, sd.w, sd.in_h, sd.in_w, sd.stride, sd.wd = rec['dw'], cur, zd, mean, invstd, oh, ow, hh, ww, stride, wd
            # pointwise
            up = rec['pw']
            up.refresh(force=True)
            zp = self._raw_conv(up, ad, key=key + '.pw')
            mean, invstd = self._bn_forward(key + '.pw', up, zp, b * oh * ow)
            ap = self._apply(up, zp, mean, invstd, b, oh, ow, False)
            sp = _Saved()
            sp.u, sp.ain, sp.z, sp.mean, sp.invstd, sp.h, sp.w, sp.pooled = up, ad, zp, mean, invstd, oh, ow, False
            saved.units.append((key, sd, sp))
            cur, hh, ww = ap, oh, ow
        head = plan['head']
        cout = head.weight.shape[0]
        w16 = ops.pack_weight_f16(head.weight.detach().contiguous(), 0)
        ones = torch.ones(cout, dtype=torch.float32, device=dev)
        feature = ops.conv_bn_act(cur, w16, ones, head.bias.detach().float().contiguous(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, hh, ww
        self._bump_tracked()
        return feature, saved

    def backward(self, saved, dfeature, dnn=None):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._ensure_arena(self.dnn, dev)
        self._main = torch.cuda.current_stream(dev)
        head = self._plan()['head']
        hh, ww = saved.hh, saved.ww
        chead, cin = head.weight.shape[0], head.weight.shape[1]
        cpad = (chead + 31) // 32 * 32
        dzh = torch.empty(b, hh, ww, cpad, dtype=torch.float16, device=dev)
        dbias = self.arena.views['layers.14.bias']
        ops.call('yb_head_grad_prepare', dfeature.contiguous().float() * self.grad_scale, dzh, dbias, b, chead, cpad, hh * ww)
        grads['layers.14.bias'] = dbias.mul_(self._unscale)
        self._emit('layers.14.bias', grads)
        # head weight gradient / data gradient (1x1)
        dw_krsc = torch.empty(chead, 1, 1, cin, dtype=torch.float32, device=dev)
        ops.call('yb_conv_wgrad', saved.a_last, dzh, dw_krsc, b, hh, ww, cin, chead, 1, saved.a_last.shape[-1], dzh.shape[-1])
        dwh = self.arena.views['layers.14.weight']
        ops.call('yb_unpack_wgrad', dw_krsc, dwh, chead, cin, 1, self._unscale)
        grads['layers.14.weight'] = dwh
        self._emit('layers.14.weight', grads)
        wdh = torch.empty(cin, 1, 1, cpad, dtype=torch.float16, device=dev)
        ops.call('yb_pack_weight_dgrad_f16', head.weight.detach().contiguous(), wdh, chead, cin, 1, cpad)
        one, zero = self._ones(cin, dev)
        g = ops.conv_bn_act(dzh, wdh, one, zero, 1.0)
        for key, sd, sp in reversed(saved.units):
            # pointwise unit: generic BN backward + wgmma weight / data gradient (state-dict names layers.N.pw.*)
            g = self._unit_backward(key + '.pw', sp, b, grads, da=g)
            # depthwise unit
            ch = sd.u.cout
            dz = torch.empty(b, sd.h, sd.w, ch, dtype=torch.float16, device=dev)
            self._bn_backward(key + '.dw', sd, b, grads, g, None, dz, ch)
            dwd = self.arena.views[key + '.dw.conv.weight']
            ops.call('yb_dwconv3x3_wgrad', sd.ain, dz, dwd, b, sd.in_h, sd.in_w, ch, sd.stride)
            grads[key + '.dw.conv.weight'] = dwd.mul_(self._unscale)
            self._emit(key + '.dw.conv.weight', grads)
            g = torch.empty(b, sd.in_h, sd.in_w, ch, dtype=torch.float16, device=dev)
            ops.call('yb_dwconv3x3_dgrad', dz, sd.wd, g, b, sd.in_h, sd.in_w, ch, sd.stride)
        s0 = saved.first
        dz0 = torch.empty(b, s0.h, s0.w, 32, dtype=torch.float16, device=dev)
        self._bn_backward('layers.0', s0, b, grads, g, None, dz0, 32)
        dw0 = self.arena.views['layers.0.conv.weight']
        ops.call('yb_mb_conv0_wgrad', saved.x, dz0, dw0, b, saved.h, saved.w)
        grads['layers.0.conv.weight'] = dw0.mul_(self._unscale)
        self._emit('layers.0.conv.weight', grads)
        self._join(dev)
        if self.reducer is not None:
            self.reducer.finish()
        if self.found_inf is None or self.found_inf.device != dev:
            self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)
        ops.call('yb_grad_guard', self.arena.flat, self.arena.flat.numel(), self.found_inf, 1)
        return grads


class _ResUnit(object):
    """One conv + BatchNorm unit of a ResNet (stem, block conv, downsample) as the trainer helpers read it: its own activation slope
    (0 = ReLU, 1 = identity before the residual join) and its torchvision-style state-dict names."""

    def __init__(self, key, conv, bn, slope, pnames):
        self.key, self.conv, self.bn, self.train_slope, self.pnames = key, conv, bn, slope, pnames
        self.stride, self.ksize = conv.stride[0], conv.kernel_size[0]
        self.cout, self.cin = conv.weight.shape[0], conv.weight.shape[1]
        self.w16 = None
        self._bver = None


class ResNetTrainer(DarknetTrainer):
    """Training-mode forward / backward of `model.resnet.ResNet` (reference model/resnet.py:28-142): stem conv 7x7 stride 2 + BN + ReLU,
    MaxPool2d(3, 2, 1), BasicBlock / Bottleneck stacks, a 1x1 head with bias.

    Forward per unit: raw wgmma conv -> batch statistics -> running-stat update (momentum read from the module, 0.1) -> normalise + ReLU
    (slope 0), or identity (slope 1) on the last unit of a block and on the downsample; the join is yb_add_relu_f16.  A stride-2 3x3 conv runs
    at stride 1 and keeps the even pixels (yb_subsample2_f16), its statistics taken after the selection; the 1x1 stride-2 downsample reads the
    subsampled input.  Backward of a stride-2 3x3 conv is the transpose: dz zero-inserted to full resolution (yb_upsample2_zero_f16), then the
    stride-1 weight and data gradients.  At each block boundary yb_residual_bwd_f16 sums the main path's data gradient and the skip path's and
    applies the previous block's ReLU mask in one pass.  The stem's gradient runs through the max-pool backward (first maximum of each window),
    the BN + ReLU backward and a CUDA-core weight-gradient kernel on the fp32 image."""

    def __init__(self, dnn, grad_scale=16384.0):
        DarknetTrainer.__init__(self, _TinyEngineView(dnn), grad_scale)
        self.dnn = dnn
        self.slope = 0.0
        self._blocks = None

    def _plan(self):
        if self._blocks is None:
            net = self.dnn
            blocks = []
            for lname in ('layer1', 'layer2', 'layer3', 'layer4'):
                for bname, blk in getattr(net, lname).named_children():
                    p = '%s.%s' % (lname, bname)
                    units = []
                    for name, conv, bn, relu in blk.units():
                        bnn = '%s.bn%s' % (p, name[len('conv'):])
                        units.append(_ResUnit('%s.%s' % (p, name), conv, bn, 0.0 if relu else 1.0, ('%s.%s.weight' % (p, name), bnn + '.weight', bnn + '.bias')))
                    ds = None
                    if blk.downsample is not None:
                        ds = _ResUnit(p + '.downsample', blk.downsample[0], blk.downsample[1], 1.0,
                                      (p + '.downsample.0.weight', p + '.downsample.1.weight', p + '.downsample.1.bias'))
                    blocks.append((p, units, ds))
            self._stem = _ResUnit('conv1', net.conv1, net.bn1, 0.0, ('conv1.weight', 'bn1.weight', 'bn1.bias'))
            self._head = _ResUnit('conv', net.conv, None, 1.0, ('conv.weight', None, None))
            self._blocks = blocks
        return self._blocks

    def _conv_units(self):
        return [u for _, units, ds in self._plan() for u in units + ([ds] if ds is not None else [])]

    def grad_order(self):
        names = ['conv.bias', 'conv.weight']
        for _, units, ds in reversed(self._plan()):
            for u in list(reversed(units)) + ([ds] if ds is not None else []):
                names += [u.pnames[1], u.pnames[2], u.pnames[0]]
        return names + ['bn1.weight', 'bn1.bias', 'conv1.weight']

    def _repack(self, device):
        """Forward and data-gradient fp16 operands of every 1x1 / 3x3 conv and the head in ONE batched launch (the stem reads its fp32
        weights in place)."""
        units = self._conv_units() + [self._head]
        ptrs = tuple(u.conv.weight.data_ptr() for u in units)
        plan = self._pack_plan
        if plan is None or plan.key != ptrs or plan.table.device != device:
            cpad = (self._head.cout + 31) // 32 * 32          # the head's filters are padded to the dz buffer's width
            plan = self._pack_plan = PackPlan([(u.key, u.conv.weight.detach(), True, True, cpad if u is self._head else 0) for u in units], device)
        plan.run()
        for u in units:
            u.w16 = plan.fwd[u.key]
            self.wd_cache[u.key] = plan.dgrad[u.key]

    def _subsample(self, x):
        b, h, w, c = x.shape
        out = torch.empty(b, (h + 1) // 2, (w + 1) // 2, c, dtype=torch.float16, device=x.device)
        ops.call('yb_subsample2_f16', x, out, b, h, w, c)
        return out

    def _unit_forward(self, u, src, b, hh, ww):
        s = _Saved()
        if u.stride == 2 and u.ksize == 1:
            src = self._subsample(src)                     # kept: the weight gradient reads it
            hh, ww = src.shape[1], src.shape[2]
        s.u, s.ain, s.in_h, s.in_w = u, src, hh, ww
        if u.stride == 2 and u.ksize == 3:
            # statistics over the selected (stride-2) pixels only: not from the full-resolution conv epilogue
            z = self._subsample(self._raw_conv(u, src))
            oh, ow = z.shape[1], z.shape[2]
        else:
            z = self._raw_conv(u, src, key=u.key)
            oh, ow = hh, ww
        mean, invstd = self._bn_forward(u.key, u, z, b * oh * ow)
        a = self._apply(u, z, mean, invstd, b, oh, ow, False)
        s.z, s.mean, s.invstd, s.h, s.w = z, mean, invstd, oh, ow
        return a, s

    def forward(self, x):
        self._tracked = []
        if not x.is_cuda:
            raise RuntimeError('ResNet training: input must be a CUDA tensor')
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('ResNet expects [B,3,H,W] with H, W multiples of 32')
        net = self.dnn
        if tuple(net.conv1.weight.shape) != (64, 3, 7, 7):
            raise ValueError('ResNet: the stem must be a 7x7 conv with 64 output channels')
        x = x.contiguous().float()
        dev = x.device
        blocks = self._plan()
        self._repack(dev)
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w = x, b, h, w
        # stem: raw conv -> BN (batch statistics) -> ReLU -> max-pool
        st = self._stem
        hh, ww = h // 2, w // 2
        z = torch.empty(b, hh, ww, 64, dtype=torch.float16, device=dev)
        ops.call('yb_stem7x7_raw_fwd', x, st.conv.weight.detach(), z, b, h, w)
        mean, invstd = self._bn_forward(st.key, st, z, b * hh * ww)
        a = self._apply(st, z, mean, invstd, b, hh, ww, False)
        s = _Saved()
        s.u, s.ain, s.z, s.mean, s.invstd, s.h, s.w = st, None, z, mean, invstd, hh, ww
        saved.stem, saved.stem_a = s, a
        cur = torch.empty(b, hh // 2, ww // 2, 64, dtype=torch.float16, device=dev)
        ops.call('yb_maxpool3x3_s2_f16', a, cur, b, hh, ww, 64)
        hh, ww = hh // 2, ww // 2
        saved.pool = cur
        saved.blocks = []
        for _, units, ds in blocks:
            xin, in_h, in_w = cur, hh, ww
            recs = []
            for u in units:
                cur, s = self._unit_forward(u, cur, b, hh, ww)
                hh, ww = s.h, s.w
                recs.append(s)
            if ds is not None:
                res, sds = self._unit_forward(ds, xin, b, in_h, in_w)
            else:
                res, sds = xin, None
            if res.shape != cur.shape:
                raise RuntimeError('ResNet training: residual %s does not match the block output %s' % (tuple(res.shape), tuple(cur.shape)))
            ops.call('yb_add_relu_f16', cur, res, cur, cur.numel())      # in place: the units keep z, not their output
            saved.blocks.append((xin, in_h, in_w, recs, sds))
        head = self._head
        one, _ = self._ones(head.cout, dev)
        feature = ops.conv_bn_act(cur, head.w16, one, head.conv.bias.detach(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, hh, ww
        self._bump_tracked()
        return feature, saved

    def _res_unit_backward(self, s, b, grads, da):
        """Backward of one block unit from the gradient of its output; returns the gradient of its input (s.ain's resolution)."""
        u = s.u
        if not (u.stride == 2 and u.ksize == 3):
            return self._unit_backward(u.key, s, b, grads, da=da)
        dev = s.z.device
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=dev)
        self._bn_backward(u.key, s, b, grads, da, None, dz, u.cout)
        dzf = torch.empty(b, s.in_h, s.in_w, u.cout, dtype=torch.float16, device=dev)
        ops.call('yb_upsample2_zero_f16', dz, dzf, b, s.in_h, s.in_w, u.cout)
        self._wgrad(u, s.ain, dzf, b, s.in_h, s.in_w, grads, u.key)
        one, zero = self._ones(u.cin, dev)
        return ops.conv_bn_act(dzf, self._wd(u.key, u), one, zero, 1.0)

    def backward(self, saved, dfeature, dnn=None):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._ensure_arena(self.dnn, dev)
        self._main = torch.cuda.current_stream(dev)
        head = self._head
        hh, ww = saved.hh, saved.ww
        chead, cin = head.cout, head.cin
        cpad = (chead + 31) // 32 * 32
        dzh = torch.empty(b, hh, ww, cpad, dtype=torch.float16, device=dev)
        dbias = self.arena.views['conv.bias']
        ops.call('yb_head_grad_prepare', dfeature.contiguous().float() * self.grad_scale, dzh, dbias, b, chead, cpad, hh * ww)
        grads['conv.bias'] = dbias.mul_(self._unscale)
        self._emit('conv.bias', grads)
        self._wgrad(head, saved.a_last, dzh, b, hh, ww, grads, head.key, cout=chead)
        one, zero = self._ones(cin, dev)
        gh = ops.conv_bn_act(dzh, self._wd(head.key, head, cpad), one, zero, 1.0)
        g = torch.empty_like(gh)
        ops.call('yb_residual_bwd_f16', saved.a_last, gh, None, 1, g, b, hh, ww, cin)        # through the last block's ReLU
        # g: gradient of the pre-ReLU sum of the current block (main path + skip)
        for (xin, in_h, in_w, recs, sds), (_, units, ds) in reversed(list(zip(saved.blocks, self._plan()))):
            gm = g
            for s in reversed(recs):
                gm = self._res_unit_backward(s, b, grads, gm)
            if sds is not None:
                gb, stride_b = self._res_unit_backward(sds, b, grads, g), sds.u.stride
            else:
                gb, stride_b = g, 1
            mask = None if xin is saved.pool else xin           # layer1.0's input is the max-pool output: no ReLU in between
            g = torch.empty_like(xin)
            ops.call('yb_residual_bwd_f16', mask, gm, gb, stride_b, g, b, in_h, in_w, xin.shape[-1])
        # stem: max-pool backward -> BN + ReLU backward -> weight gradient from the fp32 image
        st = saved.stem
        da = torch.empty_like(saved.stem_a)
        ops.call('yb_maxpool3x3_s2_bwd_f16', saved.stem_a, g, da, b, st.h, st.w, 64)
        dz = torch.empty(b, st.h, st.w, 64, dtype=torch.float16, device=dev)
        self._bn_backward(st.u.key, st, b, grads, da, None, dz, 64)
        dw = self.arena.views['conv1.weight']
        ops.call('yb_stem7x7_wgrad', saved.x, dz, dw, b, saved.h, saved.w)
        grads['conv1.weight'] = dw.mul_(self._unscale)
        self._emit('conv1.weight', grads)
        self._join(dev)
        if self.reducer is not None:
            self.reducer.finish()
        if self.found_inf is None or self.found_inf.device != dev:
            self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)
        ops.call('yb_grad_guard', self.arena.flat, self.arena.flat.numel(), self.found_inf, 1)
        return grads
