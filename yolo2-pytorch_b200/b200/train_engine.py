"""Training-mode forward and backward of the backbones (Darknet-19, Tiny, MobileNet, ResNet, VGG, Inception, DenseNet) on the CUDA kernels.

What the reference gets from torch autograd over nn.Conv2d / BatchNorm2d(train) / LeakyReLU / MaxPool2d /
reorg / cat (model/yolo2.py:49-65,125-130; train.py:344-351) is issued here as an explicit kernel chain:

  forward, per unit : wgmma conv -> raw z (fp16 NHWC) -> batch statistics (double) -> running-stat update
                      (momentum 0.01) -> normalise + leaky (+ 2x2 max-pool) -> a
  backward, per unit: leaky/BN(/pool) backward in two passes (reduce, apply) -> dgamma, dbeta, dz (fp16)
                      -> wgmma weight gradient (pixels are the reduction dim) + wgmma data gradient
                      (the forward kernel on dz with rotated, transposed weights)

Gradients travel in fp16 multiplied by `grad_scale` (static loss scaling; parameter gradients are un-scaled in fp32), or, with
`set_loss_scale('dynamic')`, by `grad_scale` times a device power-of-two factor that backs off on overflow and grows back.
BatchNorm statistics are per process (per GPU), exactly like the per-replica statistics of the reference's
nn.DataParallel.

`TrainerBase` holds everything that does not depend on a network's topology; each trainer class describes only its
own: unit order, `grad_order()`, first layer or stem, joins, pools, reorg.
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


class TrainerBase(object):
    """What every training chain shares, whatever its topology: the step state (gradient arena, data-parallel reducer, overflow flag,
    BatchNorm accumulators, weight-gradient stream), the forward and backward pieces of a conv + BatchNorm unit, the head's gradient, and
    the start and end of a step.  A subclass names the network (`NAME`), lists its parameters in the order its backward produces their
    gradients (`grad_order()`) and, to use the shared `_head_backward`, its head (`_head_unit()`)."""
    NAME = 'network'

    def __init__(self, dnn, grad_scale=16384.0, slope=SLOPE):
        self.dnn = dnn
        self.grad_scale = float(grad_scale)
        self.slope = slope       # negative slope of the activation (LeakyReLU(0.1) for the yolo2 backbones, 0 = ReLU for MobileNet / ResNet)
        self.sums = {}           # per-unit double[2C] accumulators (self-cleaning)
        self._ones_cache = {}    # fp32 (ones, zeros) per channel count and device: identity scale / shift of raw convs
        self.wd_cache = {}       # dgrad weight buffers per unit (contents re-packed every step)
        # data parallel: b200.ddp.GradientAllReducer attached by train.iterate; every gradient kernel writes into the reducer-visible
        # arena and reports it (`_emit`) so the bucket's all-reduce starts while the rest of the backward chain is still running
        self.reducer = None
        self.arena = None
        self.found_inf = None  # device float[1]: 1 when the last backward produced a non-finite gradient (then zeroed), see _finish_backward()
        # loss scaling: 'static' runs at grad_scale; 'dynamic' at grad_scale * loss_factor (set_loss_scale)
        self.loss_scale = 'static'
        self.growth_interval = 2000
        self.loss_factor = None      # device fp32 0-dim, a power of two in [2^-24, 2^24], starts at 1
        self.growth_tracker = None   # device int32 0-dim: clean steps in a row since the factor last moved
        self._arenas = {}      # one per (device, parameter set, reducer): CUDA graphs keep writing the arena they were captured with
        self._main = None
        # BN batch statistics in the conv epilogue (yb_conv_bn_act_stats_fwd) instead of yb_bn_stats; YB_FUSE_STATS=0 for A/B runs
        self.fuse_stats = os.environ.get('YB_FUSE_STATS', '1') != '0'
        # weight gradients on a second stream (overlap with the BatchNorm backward chain); YB_WGRAD_STREAM=0 for A/B runs
        self.wgrad_stream = os.environ.get('YB_WGRAD_STREAM', '1') != '0'
        self._side_streams = {}
        self._side_busy = False
        self._pack_plan = None
        self._tracked = []

    # ---- step state ----------------------------------------------------------------------------------
    def _start_forward(self, x):
        """Start of a training step: no BatchNorm counted yet; returns the image as contiguous fp32."""
        self._tracked = []
        if not x.is_cuda:
            raise RuntimeError('%s training: input must be a CUDA tensor' % self.NAME)
        return x.contiguous().float()

    def _bump_tracked(self):
        """`num_batches_tracked += 1` of every BatchNorm of the step as ONE multi-tensor kernel instead of one tiny launch per layer."""
        if self._tracked:
            torch._foreach_add_(self._tracked, 1)
            self._tracked = []

    def _start_backward(self, dev):
        """Start of the backward chain: the gradient arena of this parameter set, and the stream the chain runs on."""
        self._ensure_arena(self.dnn, dev)
        self._main = torch.cuda.current_stream(dev)

    def _finish_backward(self, dev):
        """End of the backward chain: the main stream waits for the weight-gradient stream and for every bucket's all-reduce (no host
        wait), then the fp16 gradient overflow guard runs (after the exchange, so every rank takes the same decision): `found_inf` is raised
        and the gradients are zeroed instead of poisoning the optimizer state; train.iterate hands the flag to optimizers that can skip.
        In dynamic mode the guard also divides the gradients by the loss factor and moves the factor (yb_grad_unscale_guard)."""
        self._join(dev)
        if self.reducer is not None:
            self.reducer.finish()
        if self.found_inf is None or self.found_inf.device != dev:
            self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)      # 0-dim like GradScaler's (fused optimizers subtract it from their step counters)
        if self.loss_scale == 'dynamic':
            factor, tracker = self.loss_scale_state(dev)
            ops.call('yb_grad_unscale_guard', self.arena.flat, self.arena.flat.numel(), self.found_inf, factor, tracker, self.growth_interval)
        else:
            ops.call('yb_grad_guard', self.arena.flat, self.arena.flat.numel(), self.found_inf, 1)

    def set_loss_scale(self, mode, growth_interval=2000):
        """'static': the backward runs at `grad_scale` (the default).  'dynamic': at `grad_scale` times a device power-of-two factor that
        starts at 1, halves on every step whose gradients overflow (the step is skipped or null, see `found_inf`) and doubles after
        `growth_interval` clean steps in a row, like torch.amp.GradScaler.  Powers of two make a dynamic step at factor 2^k compute the
        same gradients as a static one at grad_scale * 2^k."""
        if mode not in ('static', 'dynamic'):
            raise ValueError('loss_scale must be static or dynamic, got %r' % (mode,))
        if int(growth_interval) != growth_interval or growth_interval <= 0:
            raise ValueError('loss_scale_growth_interval must be a positive integer, got %r' % (growth_interval,))
        self.loss_scale, self.growth_interval = mode, int(growth_interval)

    def loss_scale_state(self, dev):
        """The dynamic factor and growth tracker on `dev` (created at 1 and 0 on first use), or [] in static mode."""
        if self.loss_scale != 'dynamic':
            return []
        if self.loss_factor is None or self.loss_factor.device != dev:
            self.loss_factor = torch.ones((), dtype=torch.float32, device=dev)
            self.growth_tracker = torch.zeros((), dtype=torch.int32, device=dev)
        return [self.loss_factor, self.growth_tracker]

    def _ensure_arena(self, dnn, device):
        """Persistent flat fp32 gradient buffer (b200.ddp.GradArena) for the parameters of `dnn` (the trainer's module): gradient
        kernels write straight into their slots, `.grad` of every parameter is a view of it, buckets of it are all-reduced in place."""
        params = dict(dnn.named_parameters())
        key = (str(device), tuple((n, tuple(p.shape)) for n, p in params.items()), id(self.reducer))
        self.arena = self._arenas.get(key)
        if self.arena is None:
            order = [n for n in self.grad_order() if n in params]
            if set(order) != set(params):
                raise RuntimeError('%s trainer: unexpected parameter set %s' % (self.NAME, sorted(set(params) ^ set(order))[:4]))
            bucket_bytes = self.reducer.bucket_bytes if self.reducer is not None else (32 << 20)
            self.arena = self._arenas[key] = _ddp.GradArena([(n, tuple(params[n].shape)) for n in order], device, bucket_bytes)
            if self.reducer is not None:
                self.reducer.attach(self.arena)
        return self.arena

    def _emit(self, name, grads):
        if self.reducer is not None:
            dev = grads[name].device
            side = self._side_streams.get(dev) if self._side_busy else None
            self.reducer.on_grad(name, grads[name], streams=(self._main, side))

    @property
    def _unscale(self):
        """Inverse loss scale, with the 1 / world of the data-parallel gradient average folded in."""
        return 1.0 / (self.grad_scale * (self.reducer.grad_divisor if self.reducer is not None else 1.0))

    def _pack(self, entries, device):
        """Forward and data-gradient fp16 operands of the units `entries` = [(key, unit, cout_pad)] in ONE batched launch (PackPlan); the
        plan is rebuilt when a weight moved."""
        plan = self._pack_plan
        if plan is None or plan.key != tuple(u.conv.weight.data_ptr() for _, u, _ in entries) or plan.table.device != device:
            plan = self._pack_plan = PackPlan([(key, u.conv.weight.detach(), True, True, cp) for key, u, cp in entries], device)
        plan.run()
        for key, u, _ in entries:
            u.w16 = plan.fwd[key]
            self.wd_cache[key] = plan.dgrad[key]

    def _sums(self, key, channels, device):
        t = self.sums.get(key)
        if t is None or t.numel() != 2 * channels or t.device != device:
            t = torch.zeros(2 * channels, dtype=torch.float64, device=device)
            self.sums[key] = t
        return t

    def _ones(self, c, device):
        key = (c, str(device))
        t = self._ones_cache.get(key)
        if t is None:
            t = (torch.ones(c, dtype=torch.float32, device=device), torch.zeros(c, dtype=torch.float32, device=device))
            self._ones_cache[key] = t
        return t

    # ---- unit helpers --------------------------------------------------------------------------------
    def _slope(self, u):
        """Activation slope of a unit's train-mode BatchNorm + activation: its own `train_slope` (ResNet units: 0 = ReLU, 1 = identity),
        else the trainer's."""
        return getattr(u, 'train_slope', self.slope)

    @staticmethod
    def _pnames(key, u):
        """State-dict names of a unit's (conv weight, BN weight, BN bias): `key.conv.weight`, `key.bn.*` unless the unit carries `pnames`."""
        return getattr(u, 'pnames', None) or (key + '.conv.weight', key + '.bn.weight', key + '.bn.bias')

    @staticmethod
    def _saved_unit(u, ain, z, mean, invstd, hh, ww, pooled=False, **extra):
        """What the backward of a unit reads: the unit, its input activation (None: the image), z and the batch statistics, the output
        size and whether the output is max-pooled, plus whatever the topology needs (`extra`)."""
        s = _Saved()
        s.u, s.ain, s.z, s.mean, s.invstd, s.h, s.w, s.pooled = u, ain, z, mean, invstd, hh, ww, pooled
        s.__dict__.update(extra)
        return s

    # ---- forward -------------------------------------------------------------------------------------
    def _raw_conv(self, u, src, key=None):
        """Raw conv output z, and whether its batch statistics were accumulated.  With `key` (a BN unit of the generic kernel) they are
        accumulated in the conv epilogue into the unit's double accumulators when the shape allows, so `_bn_forward` does not read z
        again.  Returns (z, stats_done)."""
        one, zero = self._ones(u.cout, src.device)
        c32 = u.cin == 32 and u.ksize == 3 and u.cout <= 64          # the halo-tile kernel: fused statistics need exact 16 x 8 tiling
        if key is not None and self.fuse_stats and not (c32 and (src.shape[1] % 16 or src.shape[2] % 8)):
            return ops.conv_bn_act_stats(src, u.w16, one, zero, 1.0, self._sums(('f', key), u.cout, src.device)), True
        return ops.conv_bn_act(src, u.w16, one, zero, 1.0), False

    def _bn_forward(self, key, u, z, rows, stats_done):
        """Batch statistics of z (accumulated here by yb_bn_stats unless the conv that wrote z already did: `stats_done`) -> mean, invstd and
        the running-statistics update."""
        bn = u.bn
        c = u.cout
        dev = z.device
        sums = self._sums(('f', key), c, dev)
        mean = torch.empty(c, dtype=torch.float32, device=dev)
        invstd = torch.empty(c, dtype=torch.float32, device=dev)
        if not stats_done:
            ops.call('yb_bn_stats', z, z.shape[-1], rows, c, sums)
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

    # ---- backward ------------------------------------------------------------------------------------
    def _bn_act_backward(self, key, s, b, da=None, da_off=0, dap=None, dap_off=0, dz=None):
        """BatchNorm + activation (+ 2x2 max-pool) backward of a saved unit from the gradient of its output: `da` unpooled (read at channel
        `da_off`), `dap` through the unit's max-pool (at channel `dap_off`).  The reduce pass accumulates into the unit's double
        accumulators; with `dz` the apply pass then writes the gradient of z.  Returns the accumulators."""
        u = s.u
        sums = self._sums(('b', key), u.cout, s.z.device)
        args = (s.z, s.z.shape[-1], s.mean, s.invstd, u.bn.weight.detach(), u.bn.bias.detach(), self._slope(u), da, 0 if da is None else da.shape[-1],
                da_off, dap, 0 if dap is None else dap.shape[-1], dap_off, b, s.h, s.w, u.cout, int(dap is not None), sums)
        ops.call('yb_bn_act_bwd', 0, *args, None, 0, 1)
        if dz is not None:
            ops.call('yb_bn_act_bwd', 1, *args, dz, dz.shape[-1], 1)
        return sums

    def _bn_param_grad(self, key, u, sums, grads):
        """dgamma, dbeta of a unit from its backward accumulators into the arena (un-scaled, / world), then the accumulators are cleared."""
        _, gname, bname = self._pnames(key, u)
        dgamma, dbeta = self.arena.views[gname], self.arena.views[bname]
        ops.call('yb_bn_param_grad', sums, u.cout, dgamma, dbeta, 1, self._unscale)
        grads[gname], grads[bname] = dgamma, dbeta
        self._emit(gname, grads)
        self._emit(bname, grads)

    def _bn_backward(self, key, s, b, grads, dz, da=None, da_off=0, dap=None, dap_off=0):
        """Both passes of the BatchNorm + activation backward into dz, then dgamma and dbeta."""
        self._bn_param_grad(key, s.u, self._bn_act_backward(key, s, b, da, da_off, dap, dap_off, dz), grads)

    def _wd(self, key, u, cout_pad=0):
        """Data-gradient operand of a unit (rotated, transposed fp16 weights), re-packed every step into a reused buffer."""
        w = u.conv.weight
        cout, cin, k, _ = w.shape
        cp = max(cout, cout_pad)
        wd = self.wd_cache.get(key)
        plan = self._pack_plan
        if plan is not None and wd is not None and plan.dgrad.get(key) is wd and wd.shape == (cin, k, k, cp):
            return wd                         # packed by this step's batched launch (_pack)
        if wd is None or wd.shape != (cin, k, k, cp) or wd.device != w.device:
            wd = torch.empty(cin, k, k, cp, dtype=torch.float16, device=w.device)
            self.wd_cache[key] = wd
        ops.call('yb_pack_weight_dgrad_f16', w.detach().contiguous(), wd, cout, cin, k, cp)
        return wd

    def _dgrad(self, key, u, dz, cout_pad=0):
        """Gradient at a unit's input: the forward conv kernel on dz with the unit's data-gradient operand."""
        one, zero = self._ones(u.cin, dz.device)
        return ops.conv_bn_act(dz, self._wd(key, u, cout_pad), one, zero, 1.0)

    def _wgrad(self, u, ain, dz, b, hh, ww, grads, name):
        """Weight gradient of one unit.  It depends only on (ain, dz) and nothing downstream depends on it before the
        optimizer, so it is issued on a second stream: the tensor-bound wgrad kernel then overlaps the HBM-bound
        BatchNorm backward of the next unit (and its data gradient) instead of queueing in front of them.  The fork /
        join is plain stream-event ordering, so it is captured as parallel branches of the step's CUDA graph."""
        cout, cin, k = u.cout, u.cin, u.ksize
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

    def _unit_backward(self, key, s, b, grads, da=None, da_off=0, dap=None, dap_off=0):
        """Backward of one BN unit; returns the gradient w.r.t. the unit's input activation, or dz when the unit reads the image."""
        u = s.u
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=s.z.device)
        self._bn_backward(key, s, b, grads, dz, da, da_off, dap, dap_off)
        if s.ain is None:
            return dz
        self._wgrad(u, s.ain, dz, b, s.h, s.w, grads, key)
        return self._dgrad(key, u, dz)

    # ---- the 7x7 stem of ResNet and DenseNet (`self._stem`: its conv + BatchNorm unit) -------------------------------------
    def _stem_forward(self, x, out=None):
        """Stem on the fp32 image x [B,3,H,W]: raw 7x7 stride-2 conv -> BN (batch statistics) -> ReLU -> 3x3 stride-2 max-pool, into a new
        tensor or, with `out`, into channels [0, 64) of `out` (DenseNet's first block buffer).  Returns (saved unit, activation before the
        pool, pooled output)."""
        b, _, h, w = x.shape
        dev = x.device
        st = self._stem
        hh, ww = h // 2, w // 2
        z = torch.empty(b, hh, ww, 64, dtype=torch.float16, device=dev)
        ops.call('yb_stem7x7_raw_fwd', x, st.conv.weight.detach(), z, b, h, w)
        mean, invstd = self._bn_forward(st.key, st, z, b * hh * ww, False)
        a = self._apply(st, z, mean, invstd, b, hh, ww, False)
        if out is None:
            pooled = torch.empty(b, hh // 2, ww // 2, 64, dtype=torch.float16, device=dev)
            ops.call('yb_maxpool3x3_s2_f16', a, pooled, b, hh, ww, 64)
        else:
            pooled = out
            ops.call('yb_maxpool3x3_s2_ld_f16', a, out, out.shape[-1], 0, b, hh, ww, 64)
        return self._saved_unit(st, None, z, mean, invstd, hh, ww), a, pooled

    def _stem_backward(self, x, st, stem_a, g, grads):
        """Stem backward from the gradient g at the max-pool output: max-pool backward -> BN + ReLU backward -> weight gradient from the fp32
        image.  Returns the gradient at the stem's activation (the max-pool's input)."""
        b, _, h, w = x.shape
        dev = g.device
        da = torch.empty_like(stem_a)
        ops.call('yb_maxpool3x3_s2_bwd_f16', stem_a, g, da, b, st.h, st.w, 64)
        dz = torch.empty(b, st.h, st.w, 64, dtype=torch.float16, device=dev)
        self._bn_backward(st.u.key, st, b, grads, dz, da=da)
        wname = st.u.pnames[0]
        dw = self.arena.views[wname]
        ops.call('yb_stem7x7_wgrad', x, dz, dw, b, h, w)
        grads[wname] = dw.mul_(self._unscale)
        self._emit(wname, grads)
        return da

    def _head_grad(self, bias, chead, a_last, hh, ww, dfeature, grads):
        """Head (1x1 conv with bias) from dfeature, the fp32 NCHW gradient of the loss w.r.t. its output: the bias gradient from the unscaled
        fp32 gradient, and dz scaled into fp16 and padded to a multiple of 32 channels (returned)."""
        b, dev = a_last.shape[0], a_last.device
        cpad = (chead + 31) // 32 * 32
        dzh = torch.empty(b, hh, ww, cpad, dtype=torch.float16, device=dev)
        dbias = self.arena.views[bias]
        dscaled = dfeature.contiguous().float() * self.grad_scale
        if self.loss_scale == 'dynamic':
            dscaled.mul_(self.loss_scale_state(dev)[0])      # exact: the factor is a power of two
        ops.call('yb_head_grad_prepare', dscaled, dzh, dbias, b, chead, cpad, hh * ww)
        grads[bias] = dbias.mul_(self._unscale)
        self._emit(bias, grads)
        return dzh

    def _head_backward(self, a_last, hh, ww, dfeature, grads):
        """Head: bias gradient and padded dz (`_head_grad`), weight gradient, and the data gradient at the head's input."""
        key, u, bias = self._head_unit()
        dzh = self._head_grad(bias, u.cout, a_last, hh, ww, dfeature, grads)
        self._wgrad(u, a_last, dzh, a_last.shape[0], hh, ww, grads, key)
        return self._dgrad(key, u, dzh, dzh.shape[-1])


class DarknetTrainer(TrainerBase):
    """Training-mode forward / backward of `model.yolo2.Darknet` (Darknet-19 with the passthrough, reorg and concat) on the units of its
    inference engine (`dnn.engine`)."""
    NAME = 'Darknet'

    @property
    def engine(self):
        return self.dnn.engine

    def grad_order(self):
        """State-dict names of all parameters in the order the backward chain produces their gradients."""
        eng = self.engine
        names = ['layers3.1.conv.bias', 'layers3.1.conv.weight']
        for key in ['layers3.0'] + list(reversed(eng._k2)) + ['passthrough'] + list(reversed(eng._k1)):
            names += [key + '.bn.weight', key + '.bn.bias', key + '.conv.weight']
        return names

    def _head_unit(self):
        return 'layers3.1', self.engine.units3[1], 'layers3.1.conv.bias'

    def _repack(self, device):
        """All kernel operands that depend on the parameters, re-derived for this step: one batched pack launch for the fp16 weight
        operands (forward + data gradient); the first layer reads its fp32 weights and the head its fp32 bias in place.  The eval-mode
        BatchNorm fold is NOT refreshed here (training uses batch statistics); `Darknet.train(False)` invalidates it."""
        eng = self.engine
        units, keys = eng.all_units(), eng.unit_keys()
        # the head's filters are padded to the dz buffer's width
        self._pack([(key, u, (u.cout + 31) // 32 * 32 if u.bn is None else 0) for u, key in zip(units[1:], keys[1:])], device)
        units[0].w16 = units[0].conv.weight.detach().contiguous()
        for u in units[1:]:
            u._wver = None                      # the eval path re-checks (and may re-pack into its own buffer)
        head = units[-1]
        if head.bn is None:
            one, zero = self._ones(head.cout, device)
            head.scale = one
            head.shift = head.conv.bias.detach() if head.conv.bias is not None else zero
            head._bver = None

    def _first_forward(self, x):
        """layers1.0 on the fp32 image: raw conv (batch statistics in its copy-out loop when the shape allows) -> BN -> leaky + 2x2 max-pool.
        Returns (saved unit, pooled activation)."""
        u0 = self.engine.units1[0]
        b, _, h, w = x.shape
        dev = x.device
        z = torch.empty(b, h, w, u0.cout, dtype=torch.float16, device=dev)
        stats_done = self.fuse_stats and h % 32 == 0 and w % 16 == 0
        if stats_done:
            # batch statistics accumulated by the conv kernel's copy-out loop: z is not read again for them
            ops.call('yb_conv0_raw_stats_fwd', x, u0.w16, z, self._sums(('f', 'layers1.0'), u0.cout, dev), b, h, w, u0.cout)
        else:
            ops.call('yb_conv0_raw_fwd', x, u0.w16, z, b, h, w, u0.cout)
        mean, invstd = self._bn_forward('layers1.0', u0, z, b * h * w, stats_done)
        a = self._apply(u0, z, mean, invstd, b, h, w, True)
        return self._saved_unit(u0, None, z, mean, invstd, h, w, True), a

    def _bn_unit_forward(self, key, u, src, b, hh, ww, pool, pooled=None, out=None, a_off=0):
        """One BN unit on its input src [B,hh,ww,*]: raw conv -> batch statistics -> normalise + leaky (+ 2x2 max-pool), the activation
        written into `out` at channel `a_off` when given.  `pooled` (default: `pool`) is what the backward chain is told about the unit's
        output.  Returns (activation, saved unit)."""
        z, stats_done = self._raw_conv(u, src, key=key)
        mean, invstd = self._bn_forward(key, u, z, b * hh * ww, stats_done)
        a = self._apply(u, z, mean, invstd, b, hh, ww, pool, out=out, a_off=a_off)
        return a, self._saved_unit(u, src, z, mean, invstd, hh, ww, pool if pooled is None else pooled)

    @staticmethod
    def _reorg_forward(a_pt, cat):
        """Passthrough activation [B,h,w,C] -> space-to-depth(2) into channels [0, 4C) of the concat buffer [B,h/2,w/2,*]."""
        ops.reorg_f16(a_pt, cat, 0)

    @staticmethod
    def _reorg_backward(dcat, b, h, w, c):
        """Gradient of the passthrough activation [B,h,w,C] from channels [0, 4C) of the concat gradient (the transpose of reorg)."""
        d_apt = torch.empty(b, h, w, c, dtype=torch.float16, device=dcat.device)
        ops.call('yb_reorg_bwd_f16', dcat, dcat.shape[-1], 0, d_apt, b, h, w, c)
        return d_apt

    def forward(self, x):
        x = self._start_forward(x)
        eng = self.engine
        b, _, h, w = x.shape
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
        # layers1.0 (direct from the fp32 image)
        saved.units['layers1.0'], cur = self._first_forward(x)
        hh, ww = h // 2, w // 2
        for u, key, pooled in zip(eng.units1[1:], eng._k1[1:], eng.pools1[1:]):
            last = key == eng._k1[-1]
            cur, saved.units[key] = self._bn_unit_forward(key, u, cur, b, hh, ww, pooled and not last, pooled)
            if pooled and not last:
                hh, ww = hh // 2, ww // 2
        x1 = cur                                    # layers1.16 output, unpooled (hh x ww)
        # passthrough -> reorg -> concat[..., :4*Cpt]
        upt = eng.unit_pt
        cat_ch = upt.cout * 4 + eng.units2[-1].cout
        cat = torch.empty(b, hh // 2, ww // 2, cat_ch, dtype=torch.float16, device=dev)
        a_pt, saved.units['passthrough'] = self._bn_unit_forward('passthrough', upt, x1, b, hh, ww, False)
        self._reorg_forward(a_pt, cat)
        # trunk
        cur = ops.maxpool2x2(x1)
        h32, w32 = hh // 2, ww // 2
        for i, (u, key) in enumerate(zip(eng.units2, eng._k2)):
            if i == len(eng.units2) - 1:
                cur, saved.units[key] = self._bn_unit_forward(key, u, cur, b, h32, w32, False, out=cat, a_off=upt.cout * 4)
            else:
                cur, saved.units[key] = self._bn_unit_forward(key, u, cur, b, h32, w32, False)
        saved.keys2 = list(eng._k2[:len(eng.units2)])
        u30, u31 = eng.units3
        a30, saved.units['layers3.0'] = self._bn_unit_forward('layers3.0', u30, cat, b, h32, w32, False)
        feature = ops.conv_bn_act(a30, u31.w16, u31.scale, u31.shift, 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a30, saved.cat, saved.x1, saved.h16, saved.w16, saved.h32, saved.w32 = a30, cat, x1, hh, ww, h32, w32
        self._bump_tracked()
        return feature, saved

    def _first_backward(self, x, s0, g_da, g_dap, grads):
        """layers1.0 backward from the gradient of its activation (g_da unpooled, g_dap through its max-pool): BN + leaky (+ pool) backward
        and the weight gradient from the fp32 image x."""
        b, _, h, w = x.shape
        dw0 = self.arena.views['layers1.0.conv.weight']
        if g_da is None and g_dap is not None and h % 8 == 0 and w % 32 == 0 and os.environ.get('YB_CONV0_WGRAD_FUSED', '1') != '0':
            # reduce pass of the BatchNorm backward, then the weight-gradient kernel forms dz itself (in shared memory, from z and the pooled
            # gradient): the 2 x 708 MB (B = 64 @ 416) write + read of dz and one launch disappear
            u0 = s0.u
            sums = self._bn_act_backward('layers1.0', s0, b, dap=g_dap)
            ops.call('yb_conv0_wgrad_bn', x, s0.z, g_dap, g_dap.shape[-1], 0, s0.mean, s0.invstd, u0.bn.weight.detach(), u0.bn.bias.detach(),
                     self._slope(u0), sums, dw0, b, h, w)
            self._bn_param_grad('layers1.0', u0, sums, grads)          # also clears the accumulators (after their last reader)
        else:
            dz0 = self._unit_backward('layers1.0', s0, b, grads, da=g_da, dap=g_dap)
            ops.call('yb_conv0_wgrad', x, dz0, dw0, b, h, w)
        grads['layers1.0.conv.weight'] = dw0.mul_(self._unscale)
        self._emit('layers1.0.conv.weight', grads)

    def backward(self, saved, dfeature):
        """dfeature: fp32 NCHW gradient of the loss w.r.t. the head output.  Returns {state_dict key: fp32 grad}: views of the
        persistent gradient arena, already averaged over the data-parallel ranks when a reducer is attached."""
        eng = self.engine
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        da = self._head_backward(saved.a30, saved.h32, saved.w32, dfeature, grads)
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
        d_apt = self._reorg_backward(dcat, b, saved.h16, saved.w16, eng.unit_pt.cout)
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
        self._first_backward(saved.x, saved.units['layers1.0'], g_da, g_dap, grads)
        self._finish_backward(dev)
        return grads


class TinyTrainer(TrainerBase):
    """Training-mode forward / backward of `model.yolo2.Tiny` (reference model/yolo2.py:140-173) on the same kernels: a plain chain of
    conv units, five of them followed by MaxPool2d(2) (fused into the normalise kernel), the sixth by ConstantPad2d + MaxPool2d(2, stride 1).

    The 16-channel first layer rides on the 32-filter first-layer kernels: its weights are zero-padded to 32 outputs, BatchNorm runs over the
    16 real channels of the 32-wide buffers (the kernels take the channel count and the pixel pitch separately), the padding channels stay
    exactly zero, and the second unit's weights are zero-padded on the input side to match (its weight gradient is cut back to 16 inputs)."""
    NAME = 'Tiny'

    def __init__(self, dnn, grad_scale=16384.0):
        TrainerBase.__init__(self, dnn, grad_scale)
        self._zero_bufs = {}

    def grad_order(self):
        keys = [key for key, _, _ in self.dnn.unit_keys()]
        names = [keys[-1] + '.conv.bias', keys[-1] + '.conv.weight']
        for key in reversed(keys[:-1]):
            names += [key + '.bn.weight', key + '.bn.bias', key + '.conv.weight']
        return names

    def _head_unit(self):
        key_h, u_h, _ = self.dnn.unit_keys()[-1]
        return key_h, u_h, key_h + '.conv.bias'

    def _zeros(self, tag, shape, device):
        """Persistent zero-initialised fp16 buffer whose padding channels are never written."""
        t = self._zero_bufs.get(tag)
        if t is None or tuple(t.shape) != tuple(shape) or t.device != device:
            t = torch.zeros(shape, dtype=torch.float16, device=device)
            self._zero_bufs[tag] = t
        return t

    def forward(self, x):
        x = self._start_forward(x)
        b, _, h, w = x.shape
        plan = self.dnn.unit_keys()
        units = [u for _, u, _ in plan]
        for i, u in enumerate(units):
            u.refresh(first_layer=(i == 0), force=True)
            if u.bn is None and i != len(units) - 1:
                raise NotImplementedError('training path requires batch_norm/enable = 1')
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w, saved.units, saved.order = x, b, h, w, {}, []
        # unit 0: 3 -> C0 (<= 32) on the first-layer kernel, filters zero-padded to 32
        key0, _, after0 = plan[0]
        saved.units[key0], cur = self._first_forward(x)
        saved.order.append((key0, after0))
        hh, ww = h // 2, w // 2
        for key, u, after in plan[1:-1]:
            cur, saved.units[key] = self._chain_unit_forward(key, u, after, cur, b, hh, ww)
            saved.order.append((key, after))
            if after == 'pool':
                hh, ww = hh // 2, ww // 2
        key_h, u_h, _ = plan[-1]
        feature = ops.conv_bn_act(cur, u_h.w16, u_h.scale, u_h.shift, 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww, saved.head = cur, hh, ww, (key_h, u_h)
        self._bump_tracked()
        return feature, saved

    def _first_forward(self, x):
        """Unit 0 (3 -> C0 <= 32) on the first-layer kernel with its filters zero-padded to 32: raw conv -> BN over the C0 real channels ->
        leaky + 2x2 max-pool into a persistent 32-wide buffer whose padding channels stay zero.  Returns (saved unit, pooled activation)."""
        b, _, h, w = x.shape
        dev = x.device
        key0, u0, after0 = self.dnn.unit_keys()[0]
        c0 = u0.cout
        if c0 > 32 or after0 != 'pool':
            raise RuntimeError('Tiny: the first unit must have <= 32 filters and be followed by MaxPool2d(2)')
        w0 = torch.zeros(32, 3, 3, 3, dtype=torch.float32, device=dev)
        w0[:c0].copy_(u0.conv.weight.detach())
        z = self._zeros(('z0', b, h, w), (b, h, w, 32), dev)
        ops.call('yb_conv0_raw_fwd', x, w0, z, b, h, w, 32)
        mean, invstd = self._bn_forward(key0, u0, z, b * h * w, False)
        cur = self._zeros(('a0', b, h, w), (b, h // 2, w // 2, 32), dev)
        self._apply(u0, z, mean, invstd, b, h, w, True, out=cur)
        return self._saved_unit(u0, None, z, mean, invstd, h, w, True, x=x), cur      # the weight gradient reads the image

    def _chain_unit_forward(self, key, u, after, cur, b, hh, ww):
        """One chain unit on its input cur [B,hh,ww,chan]: raw conv (weights zero-padded on the input side when chan > Cin) -> BN -> leaky,
        then the 2x2 max-pool (after = 'pool', fused) or ConstantPad2d + MaxPool2d(2, stride 1) (after = 'pool_s1').  Returns (output,
        saved unit)."""
        dev = cur.device
        chan = cur.shape[-1]
        if u.cin != chan:
            # input side zero-padded to the producer's buffer width (unit 1: 16 -> 32)
            wp = torch.zeros(u.cout, chan, u.ksize, u.ksize, dtype=torch.float32, device=dev)
            wp[:, :u.cin].copy_(u.conv.weight.detach())
            w16 = ops.pack_weight_f16(wp, 0)
        else:
            w16 = u.w16
        one, zero = self._ones(u.cout, dev)
        stats_done = self.fuse_stats and not (chan == 32 and u.ksize == 3 and u.cout <= 64)
        if stats_done:
            z = ops.conv_bn_act_stats(cur, w16, one, zero, 1.0, self._sums(('f', key), u.cout, dev))
        else:
            z = ops.conv_bn_act(cur, w16, one, zero, 1.0)
        mean, invstd = self._bn_forward(key, u, z, b * hh * ww, stats_done)
        a = self._apply(u, z, mean, invstd, b, hh, ww, after == 'pool')
        s = self._saved_unit(u, cur, z, mean, invstd, hh, ww, after == 'pool', cin_pad=chan)
        if after == 'pool_s1':
            s.a_unpooled = a
            a = ops.maxpool2x2_s1(a)
        return a, s

    def backward(self, saved, dfeature):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        g = self._head_backward(saved.a_last, saved.hh, saved.ww, dfeature, grads)
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
                self._tiny_unit0_backward(key, s, b, grads, g)
                break
            if s.cin_pad != u.cin:
                g = self._tiny_padded_unit_backward(key, s, b, grads, g, pooled)
            else:
                g = self._unit_backward(key, s, b, grads, da=None if pooled else g, dap=g if pooled else None)
        self._finish_backward(dev)
        return grads

    def _tiny_unit0_backward(self, key, s, b, grads, g):
        """Unit 0 from the gradient g through its max-pool: dz into a 32-wide buffer whose padding channels stay zero, then the 32-filter
        first-layer weight gradient from the fp32 image the unit saved (s.x), cut back to the C0 real filters."""
        dev = s.z.device
        dz = self._zeros(('dz0', b, s.h, s.w), (b, s.h, s.w, 32), dev)          # channels >= cout stay zero
        self._bn_backward(key, s, b, grads, dz, dap=g)
        dw32 = torch.empty(32, 3, 3, 3, dtype=torch.float32, device=dev)
        ops.call('yb_conv0_wgrad', s.x, dz, dw32, b, s.h, s.w)
        dw = self.arena.views[key + '.conv.weight']
        dw.copy_(dw32[:s.u.cout]).mul_(self._unscale)
        grads[key + '.conv.weight'] = dw
        self._emit(key + '.conv.weight', grads)

    def _tiny_padded_unit_backward(self, key, s, b, grads, g, pooled):
        """Unit whose input buffer is wider than its Cin (zero-padded): the weight gradient is computed over the padded width and cut back."""
        u = s.u
        dev = s.z.device
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=dev)
        self._bn_backward(key, s, b, grads, dz, da=None if pooled else g, dap=g if pooled else None)
        k, cp = u.ksize, s.cin_pad
        dw_krsc = torch.empty(u.cout, k, k, cp, dtype=torch.float32, device=dev)
        ops.call('yb_conv_wgrad', s.ain, dz, dw_krsc, b, s.h, s.w, cp, u.cout, k, s.ain.shape[-1], dz.shape[-1])
        full = torch.empty(u.cout, cp, k, k, dtype=torch.float32, device=dev)
        ops.call('yb_unpack_wgrad', dw_krsc, full, u.cout, cp, k, self._unscale)
        dw = self.arena.views[key + '.conv.weight']
        dw.copy_(full[:, :u.cin])
        grads[key + '.conv.weight'] = dw
        self._emit(key + '.conv.weight', grads)
        return self._dgrad(key, u, dz)      # [B, h, w, Cin]: the producer's real channels


class _BNUnit(object):
    """What the BatchNorm helpers read of a unit, for layers that are not wgmma conv units (first conv, depthwise)."""

    def __init__(self, bn, cout):
        self.bn, self.cout = bn, cout
        self._bver = None


class MobileNetTrainer(TrainerBase):
    """Training-mode forward / backward of `model.mobilenet.MobileNet` (reference model/mobilenet.py:25-85): conv_bn(3, 32, stride 2), thirteen
    [depthwise 3x3 (stride 1 or 2) + BN + ReLU, pointwise 1x1 + BN + ReLU] units, a 1x1 head with bias.  Pointwise convs, their weight /
    data gradients and the head run on the wgmma kernels of the Darknet path; the depthwise and first-layer kernels are HBM-bound CUDA-core
    kernels (csrc/mobilenet_ops.cu).  BatchNorm momentum is the PyTorch default 0.1 here (read from the modules), the activation ReLU."""
    NAME = 'MobileNet'

    def __init__(self, dnn, grad_scale=16384.0):
        TrainerBase.__init__(self, dnn, grad_scale, slope=0.0)
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
        x = self._start_forward(x)
        b, _, h, w = x.shape
        dev = x.device
        plan = self._plan()
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w, saved.units = x, b, h, w, []
        first = self.dnn.layers[0]
        if first.conv.weight.shape[0] != 32:
            raise ValueError('MobileNet: the first layer must have 32 output channels')
        saved.first, cur = self._first_forward(x)
        hh, ww = h // 2, w // 2
        for rec in plan['units']:
            ad, sd = self._dw_forward(rec, cur, b, hh, ww)
            cur, sp = self._pw_forward(rec, ad, b, sd.h, sd.w)
            saved.units.append((rec['key'], sd, sp))
            hh, ww = sd.h, sd.w
        head = plan['head']
        cout = head.weight.shape[0]
        w16 = ops.pack_weight_f16(head.weight.detach().contiguous(), 0)
        ones = torch.ones(cout, dtype=torch.float32, device=dev)
        feature = ops.conv_bn_act(cur, w16, ones, head.bias.detach().float().contiguous(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, hh, ww
        self._bump_tracked()
        return feature, saved

    def _first_forward(self, x):
        """conv_bn(3, 32, stride 2) on the fp32 image: raw conv -> BN (batch statistics) -> ReLU.  Returns (saved unit, activation)."""
        b, _, h, w = x.shape
        hh, ww = h // 2, w // 2
        z = torch.empty(b, hh, ww, 32, dtype=torch.float16, device=x.device)
        ops.call('yb_mb_conv0_raw_fwd', x, self.dnn.layers[0].conv.weight.detach().contiguous(), z, b, h, w)
        u0 = self._plan()['first']
        mean, invstd = self._bn_forward('layers.0', u0, z, b * hh * ww, False)
        a = self._apply(u0, z, mean, invstd, b, hh, ww, False)
        return self._saved_unit(u0, None, z, mean, invstd, hh, ww), a

    def _dw_forward(self, rec, cur, b, hh, ww):
        """Depthwise 3x3 unit (stride 1 or 2) on its input cur [B,hh,ww,C]: raw conv -> BN -> ReLU.  Returns (activation, saved unit)."""
        key, stride = rec['key'], rec['stride']
        ch = rec['dw'].cout
        oh, ow = hh // stride, ww // stride
        zd = torch.empty(b, oh, ow, ch, dtype=torch.float16, device=cur.device)
        wd = rec['dw_conv'].weight.detach().contiguous().view(ch, 9)
        ops.call('yb_dwconv3x3_raw_fwd', cur, wd, zd, b, hh, ww, ch, stride)
        mean, invstd = self._bn_forward(key + '.dw', rec['dw'], zd, b * oh * ow, False)
        ad = self._apply(rec['dw'], zd, mean, invstd, b, oh, ow, False)
        return ad, self._saved_unit(rec['dw'], cur, zd, mean, invstd, oh, ow, in_h=hh, in_w=ww, stride=stride, wd=wd)

    def _pw_forward(self, rec, ad, b, oh, ow):
        """Pointwise 1x1 unit on the wgmma conv: raw conv (statistics in its epilogue) -> BN -> ReLU.  Returns (activation, saved unit)."""
        key = rec['key']
        up = rec['pw']
        up.refresh(force=True)
        zp, stats_done = self._raw_conv(up, ad, key=key + '.pw')
        mean, invstd = self._bn_forward(key + '.pw', up, zp, b * oh * ow, stats_done)
        ap = self._apply(up, zp, mean, invstd, b, oh, ow, False)
        return ap, self._saved_unit(up, ad, zp, mean, invstd, oh, ow)

    def _dw_backward(self, key, sd, b, grads, g):
        """Depthwise unit backward from the gradient g of its activation: BN + ReLU backward, depthwise weight and data gradients.  Returns the
        gradient of the unit's input."""
        ch = sd.u.cout
        dev = g.device
        dz = torch.empty(b, sd.h, sd.w, ch, dtype=torch.float16, device=dev)
        self._bn_backward(key + '.dw', sd, b, grads, dz, da=g)
        dwd = self.arena.views[key + '.dw.conv.weight']
        ops.call('yb_dwconv3x3_wgrad', sd.ain, dz, dwd, b, sd.in_h, sd.in_w, ch, sd.stride)
        grads[key + '.dw.conv.weight'] = dwd.mul_(self._unscale)
        self._emit(key + '.dw.conv.weight', grads)
        gin = torch.empty(b, sd.in_h, sd.in_w, ch, dtype=torch.float16, device=dev)
        ops.call('yb_dwconv3x3_dgrad', dz, sd.wd, gin, b, sd.in_h, sd.in_w, ch, sd.stride)
        return gin

    def _first_backward(self, x, s0, g, grads):
        """First layer backward from the gradient g of its activation: BN + ReLU backward, then the weight gradient from the fp32 image."""
        b, _, h, w = x.shape
        dz0 = torch.empty(b, s0.h, s0.w, 32, dtype=torch.float16, device=g.device)
        self._bn_backward('layers.0', s0, b, grads, dz0, da=g)
        dw0 = self.arena.views['layers.0.conv.weight']
        ops.call('yb_mb_conv0_wgrad', x, dz0, dw0, b, h, w)
        grads['layers.0.conv.weight'] = dw0.mul_(self._unscale)
        self._emit('layers.0.conv.weight', grads)

    def _head_backward(self, a_last, hh, ww, dfeature, grads):
        """Head (1x1 conv with bias): bias gradient and padded dz (`_head_grad`), then the weight gradient and the data gradient at the head's
        input, both on the main stream."""
        b, dev = a_last.shape[0], a_last.device
        head = self._plan()['head']
        chead, cin = head.weight.shape[0], head.weight.shape[1]
        dzh = self._head_grad('layers.14.bias', chead, a_last, hh, ww, dfeature, grads)
        cpad = dzh.shape[-1]
        dw_krsc = torch.empty(chead, 1, 1, cin, dtype=torch.float32, device=dev)
        ops.call('yb_conv_wgrad', a_last, dzh, dw_krsc, b, hh, ww, cin, chead, 1, a_last.shape[-1], dzh.shape[-1])
        dwh = self.arena.views['layers.14.weight']
        ops.call('yb_unpack_wgrad', dw_krsc, dwh, chead, cin, 1, self._unscale)
        grads['layers.14.weight'] = dwh
        self._emit('layers.14.weight', grads)
        wdh = torch.empty(cin, 1, 1, cpad, dtype=torch.float16, device=dev)
        ops.call('yb_pack_weight_dgrad_f16', head.weight.detach().contiguous(), wdh, chead, cin, 1, cpad)
        one, zero = self._ones(cin, dev)
        return ops.conv_bn_act(dzh, wdh, one, zero, 1.0)

    def backward(self, saved, dfeature):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        g = self._head_backward(saved.a_last, saved.hh, saved.ww, dfeature, grads)
        for key, sd, sp in reversed(saved.units):
            # pointwise unit: generic BN backward + wgmma weight / data gradient (state-dict names layers.N.pw.*)
            g = self._unit_backward(key + '.pw', sp, b, grads, da=g)
            g = self._dw_backward(key, sd, b, grads, g)
        self._first_backward(saved.x, saved.first, g, grads)
        self._finish_backward(dev)
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


class ResNetTrainer(TrainerBase):
    """Training-mode forward / backward of `model.resnet.ResNet` (reference model/resnet.py:28-142): stem conv 7x7 stride 2 + BN + ReLU,
    MaxPool2d(3, 2, 1), BasicBlock / Bottleneck stacks, a 1x1 head with bias.

    Forward per unit: raw wgmma conv -> batch statistics -> running-stat update (momentum read from the module, 0.1) -> normalise + ReLU
    (slope 0), or identity (slope 1) on the last unit of a block and on the downsample; the join is yb_add_relu_f16.  A stride-2 3x3 conv runs
    at stride 1 and keeps the even pixels (yb_subsample2_f16), its statistics taken after the selection; the 1x1 stride-2 downsample reads the
    subsampled input.  Backward of a stride-2 3x3 conv is the transpose: dz zero-inserted to full resolution (yb_upsample2_zero_f16), then the
    stride-1 weight and data gradients.  At each block boundary yb_residual_bwd_f16 sums the main path's data gradient and the skip path's and
    applies the previous block's ReLU mask in one pass.  The stem's gradient runs through the max-pool backward (first maximum of each window),
    the BN + ReLU backward and a CUDA-core weight-gradient kernel on the fp32 image.

    The static loss scale depends on the depth (`default_grad_scale`, from the number of blocks).  The largest stored |gradient| is the stem
    conv's dz, and it grows with the number of train-mode BatchNorms between it and the head: on the synthetic step of the tests (8 x 160^2)
    the fp32 restatement's largest |dL/dz| is 0.11 (resnet50), 0.43 (resnet101) and 3.3 (resnet152), so at 16384 resnet152's would come
    within 1.2x of 65504.  resnet18 / 34 / 50 keep 16384; resnet101 takes 4096 and resnet152 1024.  The GPU's own steps then store at most
    2015 (resnet101, 8 x 160^2), 575 (resnet101, 2 x 416^2) and 3594 (resnet152, 8 x 160^2): 18- to 114-fold below 65504 (DESIGN §6)."""
    NAME = 'ResNet'
    GRAD_SCALES = ((16, 16384.0), (33, 4096.0), (None, 1024.0))     # (up to this many blocks, static loss scale)

    def __init__(self, dnn, grad_scale=None):
        if grad_scale is None:
            grad_scale = self.default_grad_scale(sum(len(getattr(dnn, name)) for name in ('layer1', 'layer2', 'layer3', 'layer4')))
        TrainerBase.__init__(self, dnn, grad_scale, slope=0.0)
        self._blocks = None

    @classmethod
    def default_grad_scale(cls, blocks):
        """Static loss scale of a ResNet with `blocks` residual blocks: 16384 up to resnet50's 16, 4096 up to resnet101's 33, else 1024."""
        return next(scale for limit, scale in cls.GRAD_SCALES if limit is None or blocks <= limit)

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

    def _head_unit(self):
        return self._head.key, self._head, 'conv.bias'

    def _repack(self, device):
        """Forward and data-gradient fp16 operands of every 1x1 / 3x3 conv and the head in ONE batched launch (the stem reads its fp32
        weights in place)."""
        cpad = (self._head.cout + 31) // 32 * 32          # the head's filters are padded to the dz buffer's width
        self._pack([(u.key, u, 0) for u in self._conv_units()] + [(self._head.key, self._head, cpad)], device)

    def _subsample(self, x):
        b, h, w, c = x.shape
        out = torch.empty(b, (h + 1) // 2, (w + 1) // 2, c, dtype=torch.float16, device=x.device)
        ops.call('yb_subsample2_f16', x, out, b, h, w, c)
        return out

    def _unit_forward(self, u, src, b, hh, ww):
        if u.stride == 2 and u.ksize == 1:
            src = self._subsample(src)                     # kept: the weight gradient reads it
            hh, ww = src.shape[1], src.shape[2]
        if u.stride == 2 and u.ksize == 3:
            # statistics over the selected (stride-2) pixels only: not from the full-resolution conv epilogue
            z, _ = self._raw_conv(u, src)
            z = self._subsample(z)
            stats_done = False
            oh, ow = z.shape[1], z.shape[2]
        else:
            z, stats_done = self._raw_conv(u, src, key=u.key)
            oh, ow = hh, ww
        mean, invstd = self._bn_forward(u.key, u, z, b * oh * ow, stats_done)
        a = self._apply(u, z, mean, invstd, b, oh, ow, False)
        return a, self._saved_unit(u, src, z, mean, invstd, oh, ow, in_h=hh, in_w=ww)

    def forward(self, x):
        x = self._start_forward(x)
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('ResNet expects [B,3,H,W] with H, W multiples of 32')
        net = self.dnn
        if tuple(net.conv1.weight.shape) != (64, 3, 7, 7):
            raise ValueError('ResNet: the stem must be a 7x7 conv with 64 output channels')
        dev = x.device
        blocks = self._plan()
        self._repack(dev)
        saved = _Saved()
        saved.x, saved.b, saved.h, saved.w = x, b, h, w
        saved.stem, saved.stem_a, cur = self._stem_forward(x)
        hh, ww = h // 4, w // 4
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
            self._join_forward(cur, res)
            saved.blocks.append((xin, in_h, in_w, recs, sds))
        head = self._head
        one, _ = self._ones(head.cout, dev)
        feature = ops.conv_bn_act(cur, head.w16, one, head.conv.bias.detach(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, hh, ww
        self._bump_tracked()
        return feature, saved

    @staticmethod
    def _join_forward(cur, res):
        """Block join: cur = relu(cur + res), in place (the units keep z, not their output)."""
        if res.shape != cur.shape:
            raise RuntimeError('ResNet training: residual %s does not match the block output %s' % (tuple(res.shape), tuple(cur.shape)))
        ops.call('yb_add_relu_f16', cur, res, cur, cur.numel())

    @staticmethod
    def _join_backward(mask, gm, gb, stride_b, b, h, w):
        """Gradient at a block boundary: (mask > 0) ? gm + S^T gb : 0 in one pass, where gm is the main path's input gradient, gb the skip
        path's (at 1 / stride_b resolution, or None) and mask the previous block's ReLU output (None: no ReLU in between)."""
        g = torch.empty_like(gm)
        ops.call('yb_residual_bwd_f16', mask, gm, gb, stride_b, g, b, h, w, gm.shape[-1])
        return g

    def _res_unit_backward(self, s, b, grads, da):
        """Backward of one block unit from the gradient of its output; returns the gradient of its input (s.ain's resolution)."""
        u = s.u
        if not (u.stride == 2 and u.ksize == 3):
            return self._unit_backward(u.key, s, b, grads, da=da)
        dev = s.z.device
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=dev)
        self._bn_backward(u.key, s, b, grads, dz, da=da)
        dzf = torch.empty(b, s.in_h, s.in_w, u.cout, dtype=torch.float16, device=dev)
        ops.call('yb_upsample2_zero_f16', dz, dzf, b, s.in_h, s.in_w, u.cout)
        self._wgrad(u, s.ain, dzf, b, s.in_h, s.in_w, grads, u.key)
        return self._dgrad(u.key, u, dzf)

    def backward(self, saved, dfeature):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        hh, ww = saved.hh, saved.ww
        gh = self._head_backward(saved.a_last, hh, ww, dfeature, grads)
        g = self._join_backward(saved.a_last, gh, None, 1, b, hh, ww)        # through the last block's ReLU
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
            g = self._join_backward(mask, gm, gb, stride_b, b, in_h, in_w)
        self._stem_backward(saved.x, saved.stem, saved.stem_a, g, grads)
        self._finish_backward(dev)
        return grads


class VGGTrainer(TrainerBase):
    """Training-mode forward / backward of `model.vgg.VGG` (reference model/vgg.py): a chain of 3x3 conv units, each conv (with bias) -> BatchNorm2d
    -> ReLU (`_bn` constructors) or conv -> ReLU, some followed by MaxPool2d(2, 2), then the 1x1 head with bias.

    BatchNorm units are the shared unit: raw conv (bias in the shift, so the running mean sees it; batch statistics in the conv epilogue) ->
    batch statistics -> running-stat update (momentum and eps from the module) -> normalise + ReLU, with the following max-pool fused into the
    normalise pass; their backward routes through the pool.  The conv bias before a BatchNorm has an exactly zero gradient (the normalisation
    removes any per-channel constant), so its arena slot is zero.  Plain units run the inference epilogue (scale 1, shift = bias, ReLU) and
    keep the unpooled activation a; a following max-pool is a separate yb_maxpool2x2_f16.  Their backward is yb_bn_act_bwd with has_bn = 0
    and slope 0 on a (for ReLU, a > 0 exactly where the conv output is), routed through the pool to the first maximum of each window; the
    reduce pass's per-channel sum is the bias gradient.  features.0 reads the fp32 image (yb_conv0_c64_bn_act_fwd: raw with scale 1, shift =
    bias and slope 1 for a BatchNorm unit, else activated) and its weight gradient is yb_conv0_c64_wgrad; it needs no data gradient."""
    NAME = 'VGG'

    def __init__(self, dnn, grad_scale=16384.0):
        TrainerBase.__init__(self, dnn, grad_scale, slope=0.0)
        self._units = None
        self._scratch = {}

    def _plan(self):
        if self._units is None:
            names = {m: n for n, m in self.dnn.named_modules()}
            units = []
            for i, mu in enumerate(self.dnn.units):
                key = names[mu.conv]
                bn = names[mu.bn] if mu.bn is not None else None
                u = _ResUnit(key, mu.conv, mu.bn, 0.0, (key + '.weight', bn and bn + '.weight', bn and bn + '.bias'))
                u.bias_name, u.pool = key + '.bias', mu.pool
                units.append(u)
            self._units = units
            self._head = _ResUnit('conv', self.dnn.conv, None, 1.0, ('conv.weight', None, None))
        return self._units

    def grad_order(self):
        names = ['conv.bias', 'conv.weight']
        for u in reversed(self._plan()):
            if u.bn is not None:
                names += [u.pnames[1], u.pnames[2]]
            names += [u.bias_name, u.pnames[0]]
        return names

    def _head_unit(self):
        return self._head.key, self._head, 'conv.bias'

    def _check(self):
        units = self._plan()
        if units[0].cout != 64:
            raise ValueError('VGG training: features.0 must have 64 filters (has %d)' % units[0].cout)
        for u in units[1:]:
            if u.cout % 32:
                raise ValueError('VGG training: %s has %d filters; training needs multiples of 32' % (u.key, u.cout))

    def _repack(self, device):
        """Forward and data-gradient fp16 operands of every conv after the first and of the head in ONE batched launch."""
        cpad = (self._head.cout + 31) // 32 * 32          # the head's filters are padded to the dz buffer's width
        self._pack([(u.key, u, 0) for u in self._plan()[1:]] + [(self._head.key, self._head, cpad)], device)

    def _buf(self, tag, c, device):
        t = self._scratch.get((tag, c, str(device)))
        if t is None:
            t = self._scratch[(tag, c, str(device))] = torch.empty(c, dtype=torch.float32, device=device)
        return t

    def forward(self, x):
        x = self._start_forward(x)
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('VGG expects [B,3,H,W] with H, W multiples of 32')
        self._check()
        dev = x.device
        units = self._plan()
        self._repack(dev)
        saved = _Saved()
        saved.x, saved.b, saved.units = x, b, []
        hh, ww = h, w
        cur = None
        for i, u in enumerate(units):
            cur, s = self._unit_forward(u, x if i == 0 else cur, b, hh, ww)
            saved.units.append(s)
            if u.pool:
                hh, ww = hh // 2, ww // 2
        head = self._head
        one, _ = self._ones(head.cout, dev)
        feature = ops.conv_bn_act(cur, head.w16, one, head.conv.bias.detach(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, hh, ww
        self._bump_tracked()
        return feature, saved

    def _unit_forward(self, u, src, b, hh, ww):
        """One unit on its input (the fp32 image for features.0): returns (its output, pooled when a MaxPool2d follows; saved unit)."""
        dev = src.device
        bias = u.conv.bias.detach()
        first = src.dim() == 4 and src.dtype == torch.float32
        if u.bn is not None:
            one, _ = self._ones(u.cout, dev)
            if first:
                z = ops.conv0_c64_bn_act(src, u.conv.weight.detach().contiguous(), one, bias, 1.0)
                stats_done = False
            elif self.fuse_stats:
                z, stats_done = ops.conv_bn_act_stats(src, u.w16, one, bias, 1.0, self._sums(('f', u.key), u.cout, dev)), True
            else:
                z, stats_done = ops.conv_bn_act(src, u.w16, one, bias, 1.0), False
            mean, invstd = self._bn_forward(u.key, u, z, b * hh * ww, stats_done)
            a = self._apply(u, z, mean, invstd, b, hh, ww, u.pool)
            return a, self._saved_unit(u, None if first else src, z, mean, invstd, hh, ww, u.pool)
        one, _ = self._ones(u.cout, dev)
        if first:
            a = ops.conv0_c64_bn_act(src, u.conv.weight.detach().contiguous(), one, bias, 0.0)
        else:
            a = ops.conv_bn_act(src, u.w16, one, bias, 0.0)
        out = ops.maxpool2x2(a) if u.pool else a
        return out, self._saved_unit(u, None if first else src, a, None, None, hh, ww, u.pool)

    def _plain_backward(self, s, b, grads, g):
        """Plain unit: ReLU (+ max-pool) backward on the stored activation into dz, and the bias gradient from the reduce pass's sums."""
        u = s.u
        dev = s.z.device
        da, dap = (None, g) if s.pooled else (g, None)
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=dev)
        sums = self._sums(('b', u.key), u.cout, dev)
        args = (s.z, u.cout, None, None, None, None, 0.0, da, 0 if da is None else da.shape[-1], 0, dap, 0 if dap is None else dap.shape[-1], 0,
                b, s.h, s.w, u.cout, int(dap is not None), sums)
        ops.call('yb_bn_act_bwd', 0, *args, None, 0, 0)
        ops.call('yb_bn_act_bwd', 1, *args, dz, u.cout, 0)
        dbias = self.arena.views[u.bias_name]
        ops.call('yb_bn_param_grad', sums, u.cout, self._buf('dgamma', u.cout, dev), dbias, 1, self._unscale)
        grads[u.bias_name] = dbias
        self._emit(u.bias_name, grads)
        return dz

    def _bn_unit_backward(self, s, b, grads, g):
        """BatchNorm unit: the shared BN + ReLU (+ pool) backward into dz, dgamma and dbeta; the conv bias before it gets its zero gradient."""
        u = s.u
        da, dap = (None, g) if s.pooled else (g, None)
        dz = torch.empty(b, s.h, s.w, u.cout, dtype=torch.float16, device=s.z.device)
        self._bn_backward(u.key, s, b, grads, dz, da=da, dap=dap)
        dbias = self.arena.views[u.bias_name]
        dbias.zero_()
        grads[u.bias_name] = dbias
        self._emit(u.bias_name, grads)
        return dz

    def backward(self, saved, dfeature):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        g = self._head_backward(saved.a_last, saved.hh, saved.ww, dfeature, grads)
        for s in reversed(saved.units):
            u = s.u
            dz = self._bn_unit_backward(s, b, grads, g) if u.bn is not None else self._plain_backward(s, b, grads, g)
            if s.ain is not None:
                self._wgrad(u, s.ain, dz, b, s.h, s.w, grads, u.key)
                g = self._dgrad(u.key, u, dz)
                continue
            x = saved.x
            dw = self.arena.views[u.pnames[0]]
            ops.call('yb_conv0_c64_wgrad', x, dz, dw, b, x.shape[2], x.shape[3])
            grads[u.pnames[0]] = dw.mul_(self._unscale)
            self._emit(u.pnames[0], grads)
        self._finish_backward(dev)
        return grads


class _IncUnit(object):
    """One torchvision BasicConv2d of Inception-v3 (conv without bias -> BatchNorm2d(eps 1e-3) -> ReLU) as the Inception trainer reads it:
    its geometry, its filter count rounded up to a multiple of 32 (the 80- and 48-filter convs run with zero filters) and the width of the
    buffer it reads (`cin_pad`: zero channels beyond the module's Cin get zero weights)."""

    def __init__(self, key, unit, cin_pad):
        conv = unit.conv
        self.key, self.conv, self.bn = key, conv, unit.bn
        self.kh, self.kw = conv.kernel_size
        self.stride, self.pad = conv.stride[0], tuple(conv.padding)
        self.cout, self.cin = conv.weight.shape[0], conv.weight.shape[1]
        self.cout_pad, self.cin_pad = (self.cout + 31) // 32 * 32, cin_pad
        self.pnames = (key + '.conv.weight', key + '.bn.weight', key + '.bn.bias')
        self.w16 = self.wd = None


class KhwPackPlan(object):
    """Every kh x kw unit's forward operand [cout_pad,kh,kw,cin_pad] and data-gradient operand [cin_pad,kh,kw,cout_pad] (fp16) re-derived from
    the fp32 weights by ONE launch (yb_pack_weights_khw_batch), into persistent buffers whose addresses the device table holds; the plan is
    rebuilt when a weight moves.  The table is `yb_pack_khw_unit` (include/yolo2_b200.h)."""
    DTYPE = np.dtype([('w', '<u8'), ('f', '<u8'), ('d', '<u8'), ('e0', '<i8'), ('cout', '<i4'), ('cin', '<i4'), ('kh', '<i4'), ('kw', '<i4'),
                      ('cp', '<i4'), ('cip', '<i4')])

    def __init__(self, entries, device):
        """entries: [(key, weight [Cout,Cin,kh,kw] fp32 contiguous, cout_pad, cin_pad)]"""
        assert self.DTYPE.itemsize == 56
        table = np.zeros(len(entries), dtype=self.DTYPE)
        self.key = tuple(w.data_ptr() for _, w, _, _ in entries)
        self.fwd, self.dgrad = {}, {}
        e0 = 0
        for i, (key, w, cp, cip) in enumerate(entries):
            cout, cin, kh, kw = w.shape
            if w.dtype != torch.float32 or not w.is_contiguous() or cp < cout or cip < cin:
                raise ValueError('KhwPackPlan: unsupported weight %s %s' % (key, tuple(w.shape)))
            f = self.fwd[key] = torch.empty(cp, kh, kw, cip, dtype=torch.float16, device=device)
            d = self.dgrad[key] = torch.empty(cip, kh, kw, cp, dtype=torch.float16, device=device)
            table[i] = (w.data_ptr(), f.data_ptr(), d.data_ptr(), e0, cout, cin, kh, kw, cp, cip)
            e0 += 2 * f.numel()
        self.total = e0
        self.count = len(entries)
        self.table = torch.from_numpy(table.view(np.uint8).copy()).to(device)

    def run(self):
        ops.call('yb_pack_weights_khw_batch', self.table, self.count, self.total)


def _bn_chunks(c):
    """Channel ranges of a BatchNorm of c channels (a multiple of 16) that the train-mode BatchNorm kernels take one at a time: those kernels need
    C / 8 to divide 256, so 80 runs as 64 + 16, 192 as 128 + 64, 448 as 256 + 128 + 64."""
    out, off = [], 0
    for n in (2048, 1024, 512, 256, 128, 64, 32, 16, 8):
        while c - off >= n:
            out.append((off, n))
            off += n
    if off != c:
        raise ValueError('BatchNorm of %d channels: not a multiple of 8' % c)
    return out


# Mixed block layouts: (BasicConv2d, what it reads, first channel of the block output it writes or None for an intermediate).  'x' is the block
# input, 'pool' its 3x3 average pool (count_include_pad), any other name a unit of the same block.  Consumers follow their producers.
_INCEPTION_BLOCKS = {
    'A': (('branch1x1', 'x', 0), ('branch5x5_1', 'x', None), ('branch5x5_2', 'branch5x5_1', 64), ('branch3x3dbl_1', 'x', None),
          ('branch3x3dbl_2', 'branch3x3dbl_1', None), ('branch3x3dbl_3', 'branch3x3dbl_2', 128), ('branch_pool', 'pool', 224)),
    'B': (('branch3x3', 'x', 0), ('branch3x3dbl_1', 'x', None), ('branch3x3dbl_2', 'branch3x3dbl_1', None), ('branch3x3dbl_3', 'branch3x3dbl_2', 384)),
    'C': (('branch1x1', 'x', 0), ('branch7x7_1', 'x', None), ('branch7x7_2', 'branch7x7_1', None), ('branch7x7_3', 'branch7x7_2', 192),
          ('branch7x7dbl_1', 'x', None), ('branch7x7dbl_2', 'branch7x7dbl_1', None), ('branch7x7dbl_3', 'branch7x7dbl_2', None),
          ('branch7x7dbl_4', 'branch7x7dbl_3', None), ('branch7x7dbl_5', 'branch7x7dbl_4', 384), ('branch_pool', 'pool', 576)),
    'D': (('branch3x3_1', 'x', None), ('branch3x3_2', 'branch3x3_1', 0), ('branch7x7x3_1', 'x', None), ('branch7x7x3_2', 'branch7x7x3_1', None),
          ('branch7x7x3_3', 'branch7x7x3_2', None), ('branch7x7x3_4', 'branch7x7x3_3', 320)),
    'E': (('branch1x1', 'x', 0), ('branch3x3_1', 'x', None), ('branch3x3_2a', 'branch3x3_1', 320), ('branch3x3_2b', 'branch3x3_1', 704),
          ('branch3x3dbl_1', 'x', None), ('branch3x3dbl_2', 'branch3x3dbl_1', None), ('branch3x3dbl_3a', 'branch3x3dbl_2', 1088),
          ('branch3x3dbl_3b', 'branch3x3dbl_2', 1472), ('branch_pool', 'pool', 1856)),
}
# the pool branch of Mixed_6a / Mixed_7a: F.max_pool2d(x, 3, stride=2) into these channels onwards
_INCEPTION_MAXPOOL = {'B': 480, 'D': 512}
_INCEPTION_KIND = {'Mixed_5b': 'A', 'Mixed_5c': 'A', 'Mixed_5d': 'A', 'Mixed_6a': 'B', 'Mixed_6b': 'C', 'Mixed_6c': 'C', 'Mixed_6d': 'C',
                   'Mixed_6e': 'C', 'Mixed_7a': 'D', 'Mixed_7b': 'E', 'Mixed_7c': 'E'}
_INCEPTION_STEM = ('Conv2d_1a_3x3', 'Conv2d_2a_3x3', 'Conv2d_2b_3x3', 'Conv2d_3b_1x1', 'Conv2d_4a_3x3')


class InceptionTrainer(TrainerBase):
    """Training-mode forward / backward of `model.inception3.Inception3` (reference model/inception3.py over torchvision's BasicConv2d and
    InceptionA..E), for any input side >= 75.

    Forward per BasicConv2d: raw yb_conv2d_bn_act_fwd (scale 1, shift 0, slope 1) with the module's kh x kw, stride and padding -> batch
    statistics (yb_bn_stats) -> running-statistics update with the module's eps (1e-3) and momentum (0.1) -> normalise + ReLU into the unit's
    channel range of its block's buffer (no concatenation).  The stem conv is the raw form of the stride-2 first-layer kernel on the fp32 image.

    Backward of a block runs its units in reverse: BatchNorm + ReLU backward from the unit's channel slice of the block gradient (or from the
    joined gradient of its consumers) -> weight gradient (yb_conv2d_wgrad; stride 2 walks the strided im2col box natively) -> data gradient
    (the forward conv on dz with the rotated, transposed weights; a stride-2 conv on the zero-inserted dz).  The gradient at a tensor read by
    several units is their sum (yb_join_f16: fp32, one rounding); the pool branch's contribution is the average pool of its gradient (that pool,
    with a constant divisor and a symmetric window, is its own transpose), the max-pool branch's is yb_maxpool3x3_s2_valid_bwd_f16.  The stem
    runs last: max-pool backward, BatchNorm backward, and the first conv's weight gradient from the fp32 image.

    The static loss scale is 1024, not the other chains' 16384: through 11 Mixed blocks and the stem the largest activation gradient grows
    about 50-fold from the head to the stem (measured on the synthetic step of the tests), so 16384 overflows fp16 in the stem and the
    gradient guard would zero every step."""
    NAME = 'Inception3'

    def __init__(self, dnn, grad_scale=1024.0):
        TrainerBase.__init__(self, dnn, grad_scale, slope=0.0)
        self._units = None

    # ---- plan --------------------------------------------------------------------------------------------
    def _plan(self):
        if self._units is None:
            net = self.dnn
            units = {}
            width = 3
            for name in _INCEPTION_STEM:
                u = units[name] = _IncUnit(name, getattr(net, name), width)
                width = u.cout_pad
            width = units['Conv2d_4a_3x3'].cout_pad
            for name, kind in _INCEPTION_KIND.items():
                m = getattr(net, name)
                for attr, src, _ in _INCEPTION_BLOCKS[kind]:
                    key = '%s.%s' % (name, attr)
                    units[key] = _IncUnit(key, getattr(m, attr), width if src in ('x', 'pool') else units['%s.%s' % (name, src)].cout_pad)
                width = self._block_width(kind, m, width)
            self._head = _ResUnit('conv', net.conv, None, 1.0, ('conv.weight', None, None))
            self._units = units
        return self._units

    @staticmethod
    def _block_width(kind, m, cin):
        return {'A': lambda: 224 + m.branch_pool.conv.out_channels, 'B': lambda: 480 + cin, 'C': lambda: 768, 'D': lambda: 512 + cin,
                'E': lambda: 2048}[kind]()

    def block_units(self, name):
        """The units of block `name` (a Mixed_* name or 'stem') in forward order."""
        units = self._plan()
        if name == 'stem':
            return [units[n] for n in _INCEPTION_STEM]
        return [units['%s.%s' % (name, attr)] for attr, _, _ in _INCEPTION_BLOCKS[_INCEPTION_KIND[name]]]

    def grad_order(self):
        names = ['conv.bias', 'conv.weight']
        for name in list(reversed(list(_INCEPTION_KIND))) + ['stem']:
            for u in reversed(self.block_units(name)):
                names += [u.pnames[1], u.pnames[2], u.pnames[0]]
        return names

    def _head_unit(self):
        return self._head.key, self._head, 'conv.bias'

    def _repack(self, device):
        """Forward and data-gradient fp16 operands of every conv after the stem's first and of the head, re-derived from the fp32 weights in
        ONE launch (KhwPackPlan; the optimizer just changed the weights).  The stem conv reads its fp32 weights in place."""
        units = [u for name, u in self._plan().items() if name != 'Conv2d_1a_3x3']
        head = self._head
        cpad = (head.cout + 31) // 32 * 32            # the head's filters are padded to the width of its dz buffer
        entries = [(u.key, u.conv.weight.detach(), u.cout_pad, u.cin_pad) for u in units] + [(head.key, head.conv.weight.detach(), cpad, head.cin)]
        plan = self._pack_plan
        wdev = entries[0][1].device                    # the weights' device, with its index ('cuda' alone would never compare equal)
        if plan is None or plan.key != tuple(w.data_ptr() for _, w, _, _ in entries) or plan.table.device != wdev:
            plan = self._pack_plan = KhwPackPlan(entries, wdev)
        plan.run()
        for u in units:
            u.w16, u.wd = plan.fwd[u.key], plan.dgrad[u.key]
        head.w16 = plan.fwd[head.key][:head.cout]      # the forward writes fp32 NCHW with the module's own filter count
        self.wd_cache[head.key] = plan.dgrad[head.key]

    def _wd(self, key, u, cout_pad=0):
        """The head's data-gradient operand, from this step's batched pack (the 1 x 1 layout of yb_pack_weight_dgrad_f16)."""
        return self.wd_cache[key]

    def _check(self, x):
        b, c, h, w = x.shape
        if c != 3:
            raise ValueError('Inception3 expects [B,3,H,W]')
        from model.inception3 import MIN_SIZE
        if h < MIN_SIZE or w < MIN_SIZE:
            raise ValueError('Inception3: a %d x %d input leaves a stage empty (H and W must be >= %d)' % (h, w, MIN_SIZE))
        for u in self._plan().values():
            if u.bn.momentum is None or not u.bn.track_running_stats:
                raise ValueError('Inception3 training: %s needs a BatchNorm with running statistics and a momentum' % u.key)

    # ---- forward -----------------------------------------------------------------------------------------
    def _bn_unit_forward(self, u, z, ain, out=None, a_off=0, **extra):
        """Train-mode BatchNorm + ReLU of a unit's raw output z [B,OH,OW,cout_pad]: batch statistics, running-statistics update, and the
        activation into channels [a_off, a_off + cout) of `out` (default: a new buffer of cout_pad channels, exact zeros beyond cout)."""
        b, oh, ow, ld = z.shape
        dev = z.device
        rows = b * oh * ow
        if out is None:
            out = (torch.zeros if u.cout_pad != u.cout else torch.empty)(b, oh, ow, u.cout_pad, dtype=torch.float16, device=dev)
        bn = u.bn
        mean = torch.empty(u.cout, dtype=torch.float32, device=dev)
        invstd = torch.empty(u.cout, dtype=torch.float32, device=dev)
        gamma, beta = bn.weight.detach(), bn.bias.detach()
        for off, n in _bn_chunks(u.cout):
            sums = self._sums(('f', u.key, off), n, dev)
            ops.call('yb_bn_stats', z[..., off:], ld, rows, n, sums)
            ops.call('yb_bn_finalize', sums, rows, n, float(bn.eps), float(bn.momentum), bn.running_mean[off:], bn.running_var[off:], mean[off:],
                     invstd[off:])
            ops.call('yb_bn_act_apply', z[..., off:], ld, mean[off:], invstd[off:], gamma[off:], beta[off:], 0.0, out, out.shape[-1], a_off + off,
                     b, oh, ow, n, 0)
        if bn.num_batches_tracked is not None:
            self._tracked.append(bn.num_batches_tracked)
        return out, self._saved_unit(u, ain, z, mean, invstd, oh, ow, a_off=a_off, **extra)

    def _unit_forward(self, u, src, out=None, a_off=0):
        one, zero = self._ones(u.cout_pad, src.device)
        z = ops.conv2d_bn_act(src, u.w16, one, zero, 1.0, stride=u.stride, pad=u.pad)
        return self._bn_unit_forward(u, z, src, out, a_off, in_h=src.shape[1], in_w=src.shape[2])

    def stem_forward(self, x):
        """Conv2d_1a_3x3 .. the second max-pool on the fp32 image x [B,3,H,W]: (Mixed_5b's input [B,H5,W5,192], saved stem)."""
        u1, u2a, u2b, u3b, u4a = self.block_units('stem')
        z = ops.stem3x3_s2_raw(x, u1.conv.weight.detach().contiguous(), pad=0)
        a, s1 = self._bn_unit_forward(u1, z, None)
        a, s2a = self._unit_forward(u2a, a)
        a3, s2b = self._unit_forward(u2b, a)
        p1 = ops.maxpool3x3_s2_valid(a3)
        a, s3b = self._unit_forward(u3b, p1)
        a5, s4a = self._unit_forward(u4a, a)
        p2 = ops.maxpool3x3_s2_valid(a5)
        st = _Saved()
        st.x, st.units, st.a3, st.a5 = x, [s1, s2a, s2b, s3b, s4a], a3, a5
        return p2, st

    def block_forward(self, name, x):
        """Mixed block `name` on x (fp16 NHWC): (its concatenated output, saved block)."""
        kind = _INCEPTION_KIND[name]
        m = getattr(self.dnn, name)
        b, h, w, c = x.shape
        oh, ow = ((h - 3) // 2 + 1, (w - 3) // 2 + 1) if kind in _INCEPTION_MAXPOOL else (h, w)
        out = torch.empty(b, oh, ow, self._block_width(kind, m, c), dtype=torch.float16, device=x.device)
        vals = {'x': x}
        if kind in ('A', 'C', 'E'):
            vals['pool'] = ops.avgpool3x3_s1(x)          # kept: the branch_pool weight gradient reads it
        recs = []
        for (attr, src, off), u in zip(_INCEPTION_BLOCKS[kind], self.block_units(name)):
            a, s = self._unit_forward(u, vals[src], out if off is not None else None, off or 0)
            s.src, s.name, s.to_out = src, attr, off is not None
            vals[attr] = a
            recs.append(s)
        if kind in _INCEPTION_MAXPOOL:
            ops.maxpool3x3_s2_valid(x, out, _INCEPTION_MAXPOOL[kind])
        blk = _Saved()
        blk.name, blk.kind, blk.x, blk.units = name, kind, x, recs
        return out, blk

    def forward(self, x):
        x = self._start_forward(x)
        self._check(x)
        if self.dnn.transform_input:
            raise NotImplementedError('Inception3: transform_input=True has no kernel path (the reference never sets it)')
        dev = x.device
        self._plan()
        self._repack(dev)
        saved = _Saved()
        saved.b = x.shape[0]
        cur, saved.stem = self.stem_forward(x)
        saved.blocks = []
        for name in _INCEPTION_KIND:
            cur, blk = self.block_forward(name, cur)
            saved.blocks.append(blk)
        head = self._head
        one, _ = self._ones(head.cout, dev)
        feature = ops.conv2d_bn_act(cur, head.w16, one, head.conv.bias.detach(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, cur.shape[1], cur.shape[2]
        self._bump_tracked()
        return feature, saved

    # ---- backward ----------------------------------------------------------------------------------------
    def _bn_unit_backward(self, s, da, da_off, grads):
        """BatchNorm + ReLU backward of a saved unit from channels [da_off, da_off + cout) of da: dz [B,OH,OW,cout_pad] (exact zeros beyond
        cout), dgamma and dbeta."""
        u = s.u
        b = s.z.shape[0]
        dev = s.z.device
        dz = (torch.zeros if u.cout_pad != u.cout else torch.empty)(b, s.h, s.w, u.cout_pad, dtype=torch.float16, device=dev)
        _, gname, bname = u.pnames
        dgamma, dbeta = self.arena.views[gname], self.arena.views[bname]
        gamma, beta = u.bn.weight.detach(), u.bn.bias.detach()
        for off, n in _bn_chunks(u.cout):
            sums = self._sums(('b', u.key, off), n, dev)
            args = (s.z[..., off:], s.z.shape[-1], s.mean[off:], s.invstd[off:], gamma[off:], beta[off:], 0.0, da, da.shape[-1], da_off + off,
                    None, 0, 0, b, s.h, s.w, n, 0, sums)
            ops.call('yb_bn_act_bwd', 0, *args, None, 0, 1)
            ops.call('yb_bn_act_bwd', 1, *args, dz[..., off:], dz.shape[-1], 1)
            ops.call('yb_bn_param_grad', sums, n, dgamma[off:], dbeta[off:], 1, self._unscale)
        grads[gname], grads[bname] = dgamma, dbeta
        self._emit(gname, grads)
        self._emit(bname, grads)
        return dz

    def _wgrad_khw(self, s, dz, grads):
        """Weight gradient of a unit from its input and dz, on the weight-gradient stream while a graph is captured (as TrainerBase._wgrad)."""
        u, ain = s.u, s.ain
        dev = dz.device
        side = self._side(dev)
        if side is not None:
            fork = torch.cuda.Event()
            fork.record(torch.cuda.current_stream(dev))
            side.wait_event(fork)
            dz.record_stream(side)
            ain.record_stream(side)
            self._side_busy = True
        with torch.cuda.stream(side) if side is not None else _NullCtx():
            b, h, w, ld = ain.shape
            dw_krsc = torch.empty(u.cout, u.kh, u.kw, ld, dtype=torch.float32, device=dev)
            ops.call('yb_conv2d_wgrad', ain, dz, dw_krsc, b, h, w, ld, u.cout, u.kh, u.kw, u.stride, u.pad[0], u.pad[1], ld, dz.shape[-1])
            wname = u.pnames[0]
            dw = self.arena.views[wname]
            ops.call('yb_unpack_wgrad_khw', dw_krsc, dw, u.cout, u.cin, u.kh, u.kw, ld, self._unscale)
            grads[wname] = dw
            self._emit(wname, grads)

    def _dgrad_khw(self, s, dz):
        """Gradient at a unit's input [B,H,W,cin_pad]: the forward conv on dz (zero-inserted for stride 2) with the rotated, transposed
        weights at padding (k - 1 - pad); zero channels beyond Cin."""
        u = s.u
        if u.stride == 2:
            fh, fw = s.in_h + 2 * u.pad[0] - u.kh + 1, s.in_w + 2 * u.pad[1] - u.kw + 1      # the stride-1 output grid
            dzf = torch.empty(dz.shape[0], fh, fw, dz.shape[-1], dtype=torch.float16, device=dz.device)
            ops.call('yb_upsample2_zero_f16', dz, dzf, dz.shape[0], fh, fw, dz.shape[-1])
            dz = dzf
        one, zero = self._ones(u.cin_pad, dz.device)
        return ops.conv2d_bn_act(dz, u.wd, one, zero, 1.0, pad=(u.kh - 1 - u.pad[0], u.kw - 1 - u.pad[1]))

    def _unit_backward(self, s, da, da_off, grads, need_dgrad=True):
        dz = self._bn_unit_backward(s, da, da_off, grads)
        self._wgrad_khw(s, dz, grads)
        return self._dgrad_khw(s, dz) if need_dgrad else None

    @staticmethod
    def _sum(terms):
        return terms[0] if len(terms) == 1 else ops.join(terms)

    def block_backward(self, blk, g, grads):
        """Backward of a saved Mixed block from g, the gradient of its output: the parameter gradients of its units, and the gradient at its
        input.  Every branch's data gradient at a shared tensor is collected and joined once."""
        terms = {}
        for s in reversed(blk.units):
            if s.to_out:
                gi = self._unit_backward(s, g, s.a_off, grads)
            else:
                gi = self._unit_backward(s, self._sum(terms.pop(s.name)), 0, grads)
            terms.setdefault(s.src, []).append(gi)
        if 'pool' in terms:
            terms['x'].append(ops.avgpool3x3_s1(self._sum(terms.pop('pool'))))
        if blk.kind in _INCEPTION_MAXPOOL:
            terms['x'].append(ops.maxpool3x3_s2_valid_bwd(blk.x, g, _INCEPTION_MAXPOOL[blk.kind]))
        return self._sum(terms['x'])

    def stem_backward(self, st, g, grads):
        """Stem backward from g, the gradient at Mixed_5b's input: returns the gradient at Conv2d_1a_3x3's activation."""
        s1, s2a, s2b, s3b, s4a = st.units
        g = self._unit_backward(s4a, ops.maxpool3x3_s2_valid_bwd(st.a5, g), 0, grads)
        g = self._unit_backward(s3b, g, 0, grads)
        g = self._unit_backward(s2b, ops.maxpool3x3_s2_valid_bwd(st.a3, g), 0, grads)
        g = self._unit_backward(s2a, g, 0, grads)
        dz = self._bn_unit_backward(s1, g, 0, grads)
        x = st.x
        wname = s1.u.pnames[0]
        dw = self.arena.views[wname]
        ops.call('yb_stem3x3_s2_wgrad', x, dz, dw, x.shape[0], x.shape[2], x.shape[3], 0)
        grads[wname] = dw.mul_(self._unscale)
        self._emit(wname, grads)
        return g

    def backward(self, saved, dfeature):
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        g = self._head_backward(saved.a_last, saved.hh, saved.ww, dfeature, grads)
        for blk in reversed(saved.blocks):
            g = self.block_backward(blk, g, grads)
        self.stem_backward(saved.stem, g, grads)
        self._finish_backward(dev)
        return grads


class Inception4Trainer(InceptionTrainer):
    """Training-mode forward / backward of the full-width `model.inception4.Inception4` (reference model/inception4.py), with BatchNorm on or
    off, for any input side >= 75.  The blocks come from the model's own tables (`Block.UNITS / POOLS / CAT`, `Block.chain`, the plan of
    `Inception4._plan`); at full width every width is a multiple of 32 and every channel layout the identity.

    BatchNorm on: every unit is InceptionTrainer's (raw conv -> batch statistics in power-of-two channel chunks -> running-statistics update
    with the module's eps 1e-3 and momentum 0.1 -> normalise + ReLU into the unit's channel range of its block's buffer); features.0 is the
    raw stride-2 stem kernel on the fp32 image.  BatchNorm off (conv with bias -> ReLU): the inference epilogue (scale 1, shift = bias, ReLU)
    writes the activation straight into the block buffer and is kept as the ReLU mask; its backward is yb_bn_act_bwd with has_bn = 0 in the
    same channel chunks, and the reduce pass's per-channel sum is the bias gradient (as VGGTrainer's plain units).

    Backward of a block runs its units in reverse; the gradient at a tensor read by several units (the block input: up to three branch heads
    plus the pool term; Inception_C's branch1_0 and branch2_2, each read by two convs) is joined once (yb_join_f16).  The branch3 term is
    yb_avgpool3x3_s1_excl_bwd_f16 of that conv's data gradient: the count-exclusive pool is not its own transpose (each output divides by
    its own count, 4, 6 or 9); the max-pool term is yb_maxpool3x3_s2_valid_bwd_f16 from the block gradient's channel slice.  The stem runs
    last: features.2 and features.1, then features.0's BatchNorm (or ReLU) backward and its weight gradient from the fp32 image.

    The static loss scale is 32, not Inception-v3's 1024.  With BatchNorm the largest stored |gradient| grows 2100- to 3800-fold from the
    last block to features.0's dz (measured on the synthetic steps of the tests: peaks of 4708 at 4 x 107 x 139 and 2934 at 2 x 416^2 at
    scale 32); 1024 overflowed fp16 on the first step and 64 left less than 8-fold headroom below 65504.  Without BatchNorm the gradient
    does not grow (peaks of 0.3 to 0.8 at scale 32) and part of the stem's gradient underflows; the same scale is used for both modes."""
    NAME = 'Inception4'

    def __init__(self, dnn, grad_scale=32.0):
        InceptionTrainer.__init__(self, dnn, grad_scale)
        self._blocks = None
        self._scratch = {}

    # ---- plan --------------------------------------------------------------------------------------------
    def _plan(self):
        """{unit key: _IncUnit} of every conv in forward order (the stem, then each block's units in `Block.UNITS` order), and the per-block
        plan `self._blocks`: [(block index, module, [(unit key, path, source, output channel offset or None)], max-pool offset or None)].
        `source` is 'x' (the block input), 'pool' (its count-exclusive average pool) or the path of the producing unit."""
        if self._units is None:
            net = self.dnn
            f = net.features
            names = {m: n for n, m in net.named_modules()}
            units = {}
            for i in range(3):
                lay = net.layouts[f[i]]
                units['features.%d' % i] = _IncUnit('features.%d' % i, f[i], 3 if lay is None else lay.width)
            blocks = []
            for m, segs, _ in net.blocks:
                index = int(names[m].split('.')[1])
                out_off = {seg_units[-1]: off for kind, seg_units, off in segs if kind != 'max'}
                maxpool = [off for kind, _, off in segs if kind == 'max']
                recs = []
                for path, _, _, _, _, src in m.UNITS:
                    mod = m.get_submodule(path)
                    key = '%s.%s' % (names[m], path)
                    units[key] = _IncUnit(key, mod, net.layouts[mod].width)
                    recs.append((key, path, {None: 'x', 'avg': 'pool'}.get(src, src), out_off.get(mod)))
                blocks.append((index, m, recs, maxpool[0] if maxpool else None))
            for u in units.values():
                u.bias_name = u.key + '.conv.bias' if u.bn is None else None
            head = f[-1]
            self._head = _ResUnit(names[head], head, None, 1.0, (names[head] + '.weight', None, None))
            self._blocks = blocks
            self._units = units
        return self._units

    def block_plan(self):
        self._plan()
        return self._blocks

    def block_units(self, name):
        """The units of the stem ('stem') or of block features.`name` (an index 3 .. 21) in forward order."""
        units = self._plan()
        if name == 'stem':
            return [units['features.%d' % i] for i in range(3)]
        recs = [r for i, _, r, _ in self._blocks if i == name][0]
        return [units[key] for key, _, _, _ in recs]

    def grad_order(self):
        self._plan()
        names = [self._head.key + '.bias', self._head.pnames[0]]
        for name in [i for i, _, _, _ in reversed(self._blocks)] + ['stem']:
            for u in reversed(self.block_units(name)):
                names += [u.bias_name] if u.bn is None else [u.pnames[1], u.pnames[2]]
                names.append(u.pnames[0])
        return names

    def _head_unit(self):
        return self._head.key, self._head, self._head.key + '.bias'

    def _repack(self, device):
        """Forward and data-gradient fp16 operands of every conv after features.0 and of the head in ONE launch (KhwPackPlan); features.0
        reads its fp32 weights in place."""
        units = [u for key, u in self._plan().items() if key != 'features.0']
        head = self._head
        cpad = (head.cout + 31) // 32 * 32            # the head's filters are padded to the width of its dz buffer
        entries = [(u.key, u.conv.weight.detach(), u.cout_pad, u.cin_pad) for u in units] + [(head.key, head.conv.weight.detach(), cpad, head.cin)]
        plan = self._pack_plan
        wdev = entries[0][1].device
        if plan is None or plan.key != tuple(w.data_ptr() for _, w, _, _ in entries) or plan.table.device != wdev:
            plan = self._pack_plan = KhwPackPlan(entries, wdev)
        plan.run()
        for u in units:
            u.w16, u.wd = plan.fwd[u.key], plan.dgrad[u.key]
        head.w16 = plan.fwd[head.key][:head.cout]
        self.wd_cache[head.key] = plan.dgrad[head.key]

    def _check(self, x):
        """Refuse what the trainer cannot run: a channel-pruned or ratio != 1 model (its padded channel layout would need the gradient
        gathered back out of the scattered channels), a bad shape, a BatchNorm without running statistics."""
        from model.inception4 import MIN_SIZE, STEM_FILTERS
        units = self._plan()
        u0 = units['features.0']
        if u0.cout != STEM_FILTERS:
            raise ValueError('Inception4 training: features.0 has %d filters, the stem needs exactly %d; training needs the full-width model '
                             '(no channel pruning, ratio 1)' % (u0.cout, STEM_FILTERS))
        for u in units.values():          # every tensor is then a multiple of 32 channels wide, and every layout the identity
            if u.cout % 32:
                raise ValueError('Inception4 training: %s has %d filters, not a multiple of 32; training needs the full-width model '
                                 '(no channel pruning, ratio 1)' % (u.key, u.cout))
        b, c, h, w = x.shape
        if c != 3:
            raise ValueError('Inception4 expects [B,3,H,W]')
        if h < MIN_SIZE or w < MIN_SIZE:
            raise ValueError('Inception4: a %d x %d input leaves a stage empty (H and W must be >= %d)' % (h, w, MIN_SIZE))
        for u in units.values():
            if u.bn is not None and (u.bn.momentum is None or not u.bn.track_running_stats):
                raise ValueError('Inception4 training: %s needs a BatchNorm with running statistics and a momentum' % u.key)

    # ---- forward -----------------------------------------------------------------------------------------
    def _unit_forward(self, u, src, out=None, a_off=0):
        """One unit on src: BatchNorm on as InceptionTrainer's; off, conv + bias + ReLU into channels [a_off, a_off + cout) of `out` (or a
        new buffer), that activation kept for the ReLU backward."""
        if u.bn is not None:
            return InceptionTrainer._unit_forward(self, u, src, out, a_off)
        one, _ = self._ones(u.cout_pad, src.device)
        a = ops.conv2d_bn_act(src, u.w16, one, u.conv.bias.detach(), 0.0, stride=u.stride, pad=u.pad, out=out, y_ch_off=a_off)
        return a, self._saved_unit(u, src, None, None, None, a.shape[1], a.shape[2], act=a, a_off=a_off, in_h=src.shape[1], in_w=src.shape[2])

    def stem_forward(self, x):
        """features.0 .. features.2 on the fp32 image x [B,3,H,W]: (Mixed_3a's input [B,H3,W3,64], saved stem)."""
        u0, u1, u2 = self.block_units('stem')
        w0 = u0.conv.weight.detach().contiguous()
        if u0.bn is not None:
            a, s0 = self._bn_unit_forward(u0, ops.stem3x3_s2_raw(x, w0, pad=0), None)
        else:
            one, _ = self._ones(u0.cout, x.device)
            a = ops.stem3x3_s2(x, w0, one, u0.conv.bias.detach(), pad=0)
            s0 = self._saved_unit(u0, None, None, None, None, a.shape[1], a.shape[2], act=a, a_off=0)
        a, s1 = self._unit_forward(u1, a)
        a, s2 = self._unit_forward(u2, a)
        st = _Saved()
        st.x, st.units = x, [s0, s1, s2]
        return a, st

    def block_forward(self, index, x):
        """Block features.`index` on x (fp16 NHWC): (its concatenated output, saved block)."""
        from model.inception4 import Mixed_4a
        _, m, recs, maxpool = [blk for blk in self._blocks if blk[0] == index][0]
        b, h, w, c = x.shape
        if m.POOLS:            # Mixed_3a / 5a, Reduction_A / B: every branch ends in a 3x3 valid stride-2 conv or pool
            oh, ow = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        elif isinstance(m, Mixed_4a):      # two 3x3 valid convs in parallel branches
            oh, ow = h - 2, w - 2
        else:
            oh, ow = h, w
        width = self.dnn.blocks[index - 3][2].width
        out = torch.empty(b, oh, ow, width, dtype=torch.float16, device=x.device)
        vals = {'x': x}
        if any(src == 'pool' for _, _, src, _ in recs):
            vals['pool'] = ops.avgpool3x3_s1_excl(x)          # kept: the branch3 conv's weight gradient reads it
        units = self._plan()
        saved = []
        for key, path, src, off in recs:
            a, s = self._unit_forward(units[key], vals[src], out if off is not None else None, off or 0)
            s.src, s.name, s.to_out = src, path, off is not None
            vals[path] = a
            saved.append(s)
        if maxpool is not None:
            ops.maxpool3x3_s2_valid(x, out, maxpool)
        blk = _Saved()
        blk.index, blk.x, blk.units, blk.maxpool = index, x, saved, maxpool
        return out, blk

    def forward(self, x):
        x = self._start_forward(x)
        self._check(x)
        dev = x.device
        self._repack(dev)
        saved = _Saved()
        saved.b = x.shape[0]
        cur, saved.stem = self.stem_forward(x)
        saved.blocks = []
        for index, _, _, _ in self._blocks:
            cur, blk = self.block_forward(index, cur)
            saved.blocks.append(blk)
        head = self._head
        one, _ = self._ones(head.cout, dev)
        feature = ops.conv2d_bn_act(cur, head.w16, one, head.conv.bias.detach(), 1.0, out_mode=ops.OUT_F32_NCHW)
        saved.a_last, saved.hh, saved.ww = cur, cur.shape[1], cur.shape[2]
        self._bump_tracked()
        return feature, saved

    # ---- backward ----------------------------------------------------------------------------------------
    def _bn_unit_backward(self, s, da, da_off, grads):
        """BatchNorm + ReLU backward as InceptionTrainer's; with BatchNorm off the ReLU backward on the kept activation (yb_bn_act_bwd,
        has_bn = 0, in the BatchNorm's channel chunks) into dz, and the bias gradient from the reduce pass's per-channel sums."""
        u = s.u
        if u.bn is not None:
            return InceptionTrainer._bn_unit_backward(self, s, da, da_off, grads)
        a = s.act
        b, dev = a.shape[0], a.device
        dz = (torch.zeros if u.cout_pad != u.cout else torch.empty)(b, s.h, s.w, u.cout_pad, dtype=torch.float16, device=dev)
        dbias = self.arena.views[u.bias_name]
        dscratch = self._scratch.get((u.cout, dev))
        if dscratch is None:
            dscratch = self._scratch[(u.cout, dev)] = torch.empty(u.cout, dtype=torch.float32, device=dev)
        for off, n in _bn_chunks(u.cout):
            sums = self._sums(('b', u.key, off), n, dev)
            args = (a[..., s.a_off + off:], a.shape[-1], None, None, None, None, 0.0, da, da.shape[-1], da_off + off, None, 0, 0, b, s.h, s.w, n, 0,
                    sums)
            ops.call('yb_bn_act_bwd', 0, *args, None, 0, 0)
            ops.call('yb_bn_act_bwd', 1, *args, dz[..., off:], dz.shape[-1], 0)
            ops.call('yb_bn_param_grad', sums, n, dscratch[off:], dbias[off:], 1, self._unscale)
        grads[u.bias_name] = dbias
        self._emit(u.bias_name, grads)
        return dz

    def block_backward(self, blk, g, grads):
        """Backward of a saved block from g, the gradient of its output: the parameter gradients of its units and the gradient at its input,
        every branch's contribution at a shared tensor joined once."""
        terms = {}
        for s in reversed(blk.units):
            if s.to_out:
                gi = self._unit_backward(s, g, s.a_off, grads)
            else:
                gi = self._unit_backward(s, self._sum(terms.pop(s.name)), 0, grads)
            terms.setdefault(s.src, []).append(gi)
        if 'pool' in terms:
            terms['x'].append(ops.avgpool3x3_s1_excl_bwd(self._sum(terms.pop('pool'))))
        if blk.maxpool is not None:
            terms['x'].append(ops.maxpool3x3_s2_valid_bwd(blk.x, g, blk.maxpool))
        return self._sum(terms['x'])

    def stem_backward(self, st, g, grads):
        """Stem backward from g, the gradient at Mixed_3a's input: features.2, features.1, then features.0's BatchNorm / ReLU backward and its
        weight gradient from the fp32 image (no data gradient)."""
        s0, s1, s2 = st.units
        g = self._unit_backward(s2, g, 0, grads)
        g = self._unit_backward(s1, g, 0, grads)
        dz = self._bn_unit_backward(s0, g, 0, grads)
        x = st.x
        wname = s0.u.pnames[0]
        dw = self.arena.views[wname]
        ops.call('yb_stem3x3_s2_wgrad', x, dz, dw, x.shape[0], x.shape[2], x.shape[3], 0)
        grads[wname] = dw.mul_(self._unscale)
        self._emit(wname, grads)
        return g


class _DenseStats(object):
    """Per-block batch statistics shared by every norm that reads a block channel: double accumulators (the writer of channels [s, s + n)
    owns sums[2s, 2s + 2n) in the [sum | sum of squares] layout of yb_bn_stats), the batch mean / unbiased variance that feed the running
    statistics (zero-initialised: yb_bn_finalize with momentum 1 stores them), and mean / invstd."""

    def __init__(self, width, device):
        self.sums = torch.zeros(2 * width, dtype=torch.float64, device=device)
        self.bmean = torch.zeros(width, dtype=torch.float32, device=device)
        self.bvar = torch.zeros(width, dtype=torch.float32, device=device)
        self.mean = torch.zeros(width, dtype=torch.float32, device=device)
        self.invstd = torch.zeros(width, dtype=torch.float32, device=device)
        self.running = None       # (key, device table of yb_bn_running) of the block's norms

    def seg(self, s, n):
        return self.sums[2 * s:2 * s + 2 * n]


class DenseNetTrainer(TrainerBase):
    """Training-mode forward / backward of `model.densenet.DenseNet` (densenet121 / 169 / 201; reference model/densenet.py over torchvision's
    _DenseLayer / _Transition).  Each dense block lives in one fp16 buffer as wide as its output, as in inference.

    Forward: the stem is ResNet's (`TrainerBase._stem_forward`), pooling into channels [0, 64) of block 1's buffer.  A channel's batch
    statistics are computed once, when it is written (yb_bn_stats on the stem's pool output, the conv2 and transition-conv epilogues), and
    shared by every norm that reads it; each norm folds them with its own gamma / beta (yb_bn_batch_fold), and all norms of a block update
    their running statistics in one launch (yb_bn_running_update_batch).  A dense layer is norm1 + relu1 + conv1 on the block's first Ci
    channels (yb_conv1x1_preact_stats_fwd: raw z1 with norm2's statistics in its epilogue), norm2 + relu2 (the shared unit helpers), then the
    3x3 conv2 writing its 32 channels at channel Ci with their statistics.  A transition pools before its 1x1 conv, as in inference, and keeps
    the pooled activation for its weight gradient; norm5 feeds the head through the identity pre-activation.

    Backward: the gradient of a block buffer is accumulated in fp32 ([B,H,W,C] per block): every pre-activation norm's backward
    (yb_bn_preact_bwd; its reduce pass is yb_bn_act_bwd mode 0 when C / 8 divides 256 and the gradient is unpooled) adds its dx, and rounds to
    fp16 the slice that its contribution completes -- layer j's 32 channels once layer j + 1 has added its part, the block input once layer
    1 has -- which is the next dz: conv2's, the transition conv's (on the pooled grid) or the stem pool's.  The pre-activation convs' weight
    gradients form a = act(norm(x)) on the shared-memory tile (yb_conv1x1_preact_wgrad)."""
    NAME = 'DenseNet'
    GROWTH = 32
    GRAD_SCALE = 1024.0      # static loss scale, chosen on synthetic steps (DESIGN §6)

    def __init__(self, dnn, grad_scale=GRAD_SCALE):
        TrainerBase.__init__(self, dnn, grad_scale, slope=0.0)
        self._blocks = None
        self._stats = {}

    # ---- plan ----------------------------------------------------------------------------------------
    @staticmethod
    def _norm_unit(key, bn, channels):
        u = _BNUnit(bn, channels)
        u.key, u.pnames = key, (None, key + '.weight', key + '.bias')
        return u

    def _plan(self):
        if self._blocks is None:
            net = self.dnn
            f = net.features
            self._stem = _ResUnit('features.conv0', f.conv0, f.norm0, 0.0, ('features.conv0.weight', 'features.norm0.weight', 'features.norm0.bias'))
            self._head = _ResUnit('features.conv', f.conv, None, 1.0, ('features.conv.weight', None, None))
            blocks = []
            for i, n in enumerate(net.block_config):
                name = 'features.denseblock%d' % (i + 1)
                mod = getattr(f, 'denseblock%d' % (i + 1))
                cin0, width = net.block_channels[i]
                layers = []
                for j in range(n):
                    key = '%s.denselayer%d' % (name, j + 1)
                    layer = getattr(mod, 'denselayer%d' % (j + 1))
                    ci = cin0 + j * net.growth_rate
                    layers.append(dict(cin=ci, norm1=self._norm_unit(key + '.norm1', layer.norm1, ci),
                                       conv1=_ResUnit(key + '.conv1', layer.conv1, layer.norm2, 0.0,
                                                      (key + '.conv1.weight', key + '.norm2.weight', key + '.norm2.bias')),
                                       conv2=_ResUnit(key + '.conv2', layer.conv2, None, 1.0, (key + '.conv2.weight', None, None))))
                if i + 1 < len(net.block_config):
                    tname = 'features.transition%d' % (i + 1)
                    t = getattr(f, 'transition%d' % (i + 1))
                    tail = self._norm_unit(tname + '.norm', t.norm, width)
                    tconv = _ResUnit(tname + '.conv', t.conv, None, 1.0, (tname + '.conv.weight', None, None))
                else:
                    tail, tconv = self._norm_unit('features.norm5', f.norm5, width), None
                blocks.append(dict(index=i, cin=cin0, width=width, layers=layers, tail=tail, tconv=tconv))
            self._blocks = blocks
        return self._blocks

    def grad_order(self):
        names = ['features.conv.bias', 'features.conv.weight']
        for blk in reversed(self._plan()):
            if blk['tconv'] is not None:
                names += [blk['tconv'].pnames[0]]
            names += list(blk['tail'].pnames[1:])
            for layer in reversed(blk['layers']):
                c1, c2 = layer['conv1'], layer['conv2']
                names += [c2.pnames[0], c1.pnames[1], c1.pnames[2], c1.pnames[0]] + list(layer['norm1'].pnames[1:])
        return names + ['features.norm0.weight', 'features.norm0.bias', 'features.conv0.weight']

    def _block_norm_settings(self, blk):
        """(eps, momentum) shared by every norm reading the block's channels (each later norm1 and the tail all read channel 0)."""
        norms = [layer['norm1'].bn for layer in blk['layers']] + [blk['tail'].bn]
        eps = set(float(bn.eps) for bn in norms)
        mom = set(bn.momentum for bn in norms)
        if len(eps) != 1 or len(mom) != 1:
            raise ValueError('DenseNet training: the norms reading %s disagree on eps %s or momentum %s; they share one set of batch '
                             'statistics' % ('features.denseblock%d' % (blk['index'] + 1), sorted(eps), sorted(mom, key=str)))
        m = mom.pop()
        if m is None:
            raise ValueError('DenseNet training: momentum=None (cumulative running average) is not supported')
        return eps.pop(), float(m)

    def _repack(self, device):
        """Forward and data-gradient fp16 operands of every conv1, conv2, transition conv and the head in ONE batched launch (the stem reads
        its fp32 weights in place)."""
        entries = []
        for blk in self._plan():
            for layer in blk['layers']:
                entries += [(layer['conv1'].key, layer['conv1'], 0), (layer['conv2'].key, layer['conv2'], 0)]
            if blk['tconv'] is not None:
                entries.append((blk['tconv'].key, blk['tconv'], 0))
        entries.append((self._head.key, self._head, (self._head.cout + 31) // 32 * 32))      # padded to the dz buffer's width
        self._pack(entries, device)

    def _block_stats(self, blk, device):
        key = (blk['index'], str(device))
        st = self._stats.get(key)
        if st is None or st.mean.numel() != blk['width']:
            st = self._stats[key] = _DenseStats(blk['width'], device)
        return st

    # ---- forward -------------------------------------------------------------------------------------
    def _finalize(self, st, s, n, rows, eps):
        """Batch statistics of block channels [s, s + n) from their accumulators: mean / invstd, and the batch mean / unbiased variance for the
        running statistics (yb_bn_finalize with momentum 1 writes exactly those into its running-stat outputs)."""
        ops.call('yb_bn_finalize', st.seg(s, n), rows, n, eps, 1.0, st.bmean[s:s + n], st.bvar[s:s + n], st.mean[s:s + n], st.invstd[s:s + n])

    @staticmethod
    def _fold(st, nu):
        c = nu.cout
        scale = torch.empty(c, dtype=torch.float32, device=st.mean.device)
        shift = torch.empty_like(scale)
        ops.call('yb_bn_batch_fold', st.mean, st.invstd, nu.bn.weight.detach(), nu.bn.bias.detach(), scale, shift, c)
        return scale, shift

    def _running_update(self, blk, st, momentum):
        """Running statistics of every norm of the block (each over its own channels [0, C)) in one launch; num_batches_tracked with the rest."""
        norms = [layer['norm1'] for layer in blk['layers']] + [blk['tail']]
        key = tuple((nu.bn.running_mean.data_ptr(), nu.bn.running_var.data_ptr()) for nu in norms)
        if st.running is None or st.running[0] != key:
            table = np.zeros(len(norms), dtype=np.dtype([('m', '<u8'), ('v', '<u8'), ('c', '<i4'), ('mom', '<f4')]))
            for k, nu in enumerate(norms):
                table[k] = (nu.bn.running_mean.data_ptr(), nu.bn.running_var.data_ptr(), nu.cout, momentum)
            st.running = (key, torch.from_numpy(table.view(np.uint8).copy()).to(st.mean.device))
        ops.call('yb_bn_running_update_batch', st.bmean, st.bvar, st.running[1], len(norms), blk['width'])
        for nu in norms:
            if nu.bn.num_batches_tracked is not None:
                self._tracked.append(nu.bn.num_batches_tracked)
            nu._bver = None

    def _layer_forward(self, layer, buf, st, eps, b, hh, ww):
        """One dense layer on channels [0, Ci) of the block buffer; its 32 new channels (and their statistics) land at channel Ci."""
        ci, c1, c2 = layer['cin'], layer['conv1'], layer['conv2']
        dev = buf.device
        pre = self._fold(st, layer['norm1'])
        one, zero = self._ones(c1.cout, dev)
        z1 = torch.empty(b, hh, ww, c1.cout, dtype=torch.float16, device=dev)
        ops.call('yb_conv1x1_preact_stats_fwd', buf, c1.w16, pre[0], pre[1], 1, one, zero, 1.0, z1, b, hh, ww, ci, c1.cout, buf.shape[-1], c1.cout, 0,
                 self._sums(('f', c1.key), c1.cout, dev))
        mean2, invstd2 = self._bn_forward(c1.key, c1, z1, b * hh * ww, True)
        a2 = self._apply(c1, z1, mean2, invstd2, b, hh, ww, False)
        one, zero = self._ones(c2.cout, dev)
        ops.call('yb_conv_bn_act_stats_fwd', a2, c2.w16, one, zero, 1.0, buf, b, hh, ww, c2.cin, c2.cout, 3, a2.shape[-1], buf.shape[-1], ci, 0,
                 st.seg(ci, c2.cout))
        self._finalize(st, ci, c2.cout, b * hh * ww, eps)
        return self._saved_unit(c1, None, z1, mean2, invstd2, hh, ww, a2=a2, pre=pre)

    def _transition_forward(self, blk, rec, nblk, nst, eps, b):
        """norm + relu + AvgPool2d(2) of the whole block buffer (rec.pre: the norm's fold), kept for the weight gradient, then the 1x1 conv into
        channels [0, C/2) of the next block's new buffer with their statistics (into nst).  Returns (that buffer, nst)."""
        width, hh, ww, dev = blk['width'], rec.h, rec.w, rec.buf.device
        tc = blk['tconv']
        rec.pooled = torch.empty(b, hh // 2, ww // 2, width, dtype=torch.float16, device=dev)
        ops.call('yb_bn_relu_avgpool2x2_f16', rec.buf, width, rec.pre[0], rec.pre[1], rec.pooled, b, hh, ww, width)
        hh, ww = hh // 2, ww // 2
        nbuf = torch.empty(b, hh, ww, nblk['width'], dtype=torch.float16, device=dev)
        one, zero = self._ones(tc.cout, dev)
        ops.call('yb_conv_bn_act_stats_fwd', rec.pooled, tc.w16, one, zero, 1.0, nbuf, b, hh, ww, width, tc.cout, 1, width, nbuf.shape[-1], 0, 0,
                 nst.seg(0, tc.cout))
        self._finalize(nst, 0, tc.cout, b * hh * ww, eps)
        return nbuf, nst

    def _head_forward(self, rec):
        """norm5 (rec.pre, identity activation) + the head conv with bias on the last block's buffer: the fp32 NCHW feature."""
        head = self._head
        one, _ = self._ones(head.cout, rec.buf.device)
        return ops.conv1x1_preact(rec.buf, head.w16, rec.pre[0], rec.pre[1], False, one, head.conv.bias.detach(), 1.0, out_mode=ops.OUT_F32_NCHW)

    def _check(self, x):
        net = self.dnn
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise ValueError('DenseNet expects [B,3,H,W] with H, W multiples of 32')
        why = net.unsupported()
        if why is not None:
            raise NotImplementedError('DenseNet: no kernel path for %s' % why)
        if net.growth_rate != self.GROWTH or net.bn_size * net.growth_rate != 128:
            raise NotImplementedError('DenseNet training: growth rate %d, bn_size %d (the training path is built for 32 and 4)'
                                      % (net.growth_rate, net.bn_size))

    def forward(self, x):
        x = self._start_forward(x)
        self._check(x)
        b, _, h, w = x.shape
        dev = x.device
        blocks = self._plan()
        settings = [self._block_norm_settings(blk) for blk in blocks]
        self._repack(dev)
        saved = _Saved()
        saved.x, saved.b, saved.blocks = x, b, []
        hh, ww = h // 4, w // 4
        buf = torch.empty(b, hh, ww, blocks[0]['width'], dtype=torch.float16, device=dev)
        saved.stem, saved.stem_a, _ = self._stem_forward(x, out=buf)
        st = self._block_stats(blocks[0], dev)
        ops.call('yb_bn_stats', buf, buf.shape[-1], b * hh * ww, 64, st.seg(0, 64))
        self._finalize(st, 0, 64, b * hh * ww, settings[0][0])
        feature = None
        for blk, (eps, momentum) in zip(blocks, settings):
            rec = _Saved()
            rec.buf, rec.st, rec.h, rec.w = buf, st, hh, ww
            rec.layers = [self._layer_forward(layer, buf, st, eps, b, hh, ww) for layer in blk['layers']]
            self._running_update(blk, st, momentum)
            rec.pre = self._fold(st, blk['tail'])
            if blk['tconv'] is not None:
                nblk = blocks[blk['index'] + 1]
                buf, st = self._transition_forward(blk, rec, nblk, self._block_stats(nblk, dev), settings[blk['index'] + 1][0], b)
                hh, ww = hh // 2, ww // 2
            else:
                feature = self._head_forward(rec)
            saved.blocks.append(rec)
        self._bump_tracked()
        return feature, saved

    # ---- backward ------------------------------------------------------------------------------------
    def _preact_wgrad(self, u, x, pre, relu, dz, b, hh, ww, grads):
        """Weight gradient of a pre-activation 1x1 conv (conv1, the head) into its arena slot."""
        dev = dz.device
        dw_krsc = torch.empty(u.cout, 1, 1, u.cin, dtype=torch.float32, device=dev)
        ops.call('yb_conv1x1_preact_wgrad', x, pre[0], pre[1], int(relu), dz, dw_krsc, b, hh, ww, u.cin, u.cout, x.shape[-1], dz.shape[-1])
        wname = u.pnames[0]
        dw = self.arena.views[wname]
        ops.call('yb_unpack_wgrad', dw_krsc, dw, u.cout, u.cin, 1, self._unscale)
        grads[wname] = dw
        self._emit(wname, grads)

    def _preact_bn_backward(self, nu, rec, da, relu, pool, gbuf, out16, out16_ch0, b, grads):
        """Backward of a pre-activation norm over channels [0, C) of the block buffer: reduce (dgamma, dbeta), then dx added into the fp32 block
        gradient with channels [out16_ch0, C) also rounded into out16."""
        c = nu.cout
        buf, st = rec.buf, rec.st
        sums = self._sums(('b', nu.key), c, buf.device)
        gamma, beta = nu.bn.weight.detach(), nu.bn.bias.detach()
        if not pool and 256 % (c // 8) == 0:         # yb_bn_act_bwd's kernels need C / 8 to divide their 256 threads
            ops.call('yb_bn_act_bwd', 0, buf, buf.shape[-1], st.mean, st.invstd, gamma, beta, 0.0 if relu else 1.0, da, da.shape[-1], 0, None, 0, 0,
                     b, rec.h, rec.w, c, 0, sums, None, 0, 1)
        else:
            ops.call('yb_bn_preact_bwd', 0, buf, buf.shape[-1], st.mean, st.invstd, gamma, beta, int(relu), da, da.shape[-1], int(pool), b, rec.h, rec.w, c,
                     sums, None, 0, None, 0, 0)
        ops.call('yb_bn_preact_bwd', 1, buf, buf.shape[-1], st.mean, st.invstd, gamma, beta, int(relu), da, da.shape[-1], int(pool), b, rec.h, rec.w, c,
                 sums, gbuf, gbuf.shape[-1], out16, out16.shape[-1], out16_ch0)
        self._bn_param_grad(nu.key, nu, sums, grads)

    def _tail_backward(self, blk, rec, g, gbuf, b, grads):
        """Backward of the block's tail into its fp32 gradient gbuf: norm5 + head from dfeature g (fp32 NCHW), or the transition from g, the
        fp16 gradient of its conv's output.  Returns the fp16 gradient of the block's last 32 channels (the last conv2's dz)."""
        hh, ww, width = rec.h, rec.w, blk['width']
        dz2 = torch.empty(b, hh, ww, self.GROWTH, dtype=torch.float16, device=g.device)
        if blk['tconv'] is None:
            head = self._head
            dzh = self._head_grad('features.conv.bias', head.cout, rec.buf, hh, ww, g, grads)
            self._preact_wgrad(head, rec.buf, rec.pre, 0, dzh, b, hh, ww, grads)
            da = self._dgrad(head.key, head, dzh, dzh.shape[-1])
            self._preact_bn_backward(blk['tail'], rec, da, 0, 0, gbuf, dz2, width - self.GROWTH, b, grads)
        else:
            tc = blk['tconv']
            self._wgrad(tc, rec.pooled, g, b, hh // 2, ww // 2, grads, tc.key)
            dpool = self._dgrad(tc.key, tc, g)
            self._preact_bn_backward(blk['tail'], rec, dpool, 1, 1, gbuf, dz2, width - self.GROWTH, b, grads)
        return dz2

    def _layer_backward(self, layer, rec, s, dz2, gbuf, b, grads, first):
        """Backward of one dense layer from dz2, the fp16 gradient of its 32 channels: conv2, norm2 + relu2, conv1 and norm1 + relu1, whose dx
        is added into gbuf.  Returns the fp16 slice that contribution completes: the previous layer's 32 channels, or the block input when
        `first`."""
        hh, ww, dev = rec.h, rec.w, dz2.device
        ci, c1, c2 = layer['cin'], layer['conv1'], layer['conv2']
        self._wgrad(c2, s.a2, dz2, b, hh, ww, grads, c2.key)
        da2 = self._dgrad(c2.key, c2, dz2)
        dz1 = torch.empty(b, hh, ww, c1.cout, dtype=torch.float16, device=dev)
        self._bn_backward(c1.key, s, b, grads, dz1, da=da2)
        self._preact_wgrad(c1, rec.buf, s.pre, 1, dz1, b, hh, ww, grads)
        da1 = self._dgrad(c1.key, c1, dz1)
        n16 = ci if first else self.GROWTH
        out16 = torch.empty(b, hh, ww, n16, dtype=torch.float16, device=dev)
        self._preact_bn_backward(layer['norm1'], rec, da1, 1, 0, gbuf, out16, ci - n16, b, grads)
        return out16

    def backward(self, saved, dfeature):
        b = saved.b
        grads = {}
        dev = dfeature.device
        self._start_backward(dev)
        g = dfeature         # the gradient arriving at the current block's tail
        for blk, rec in reversed(list(zip(self._plan(), saved.blocks))):
            gbuf = torch.zeros(b, rec.h, rec.w, blk['width'], dtype=torch.float32, device=dev)
            dz2 = self._tail_backward(blk, rec, g, gbuf, b, grads)
            for j in reversed(range(len(blk['layers']))):
                dz2 = self._layer_backward(blk['layers'][j], rec, rec.layers[j], dz2, gbuf, b, grads, j == 0)
            g = dz2          # the block input's gradient: the previous transition conv's dz, or the stem pool's
        self._stem_backward(saved.x, saved.stem, saved.stem_a, g, grads)
        self._finish_backward(dev)
        return grads
