"""train -- the training step of the reference (train.py:57-71,338-362) on the GPU path.

`norm_data`, `ensure_model` and `iterate` keep the reference's meaning:
  iterate: forward (train-mode Darknet: batch-statistics BatchNorm) -> region loss -> hparam-weighted sum ->
           zero_grad -> backward (explicit kernel chain + optional NCCL gradient all-reduce) -> optional clip ->
           optimizer.step().
The optimizer / scheduler objects are torch.optim's, built from the same `train/optimizer` lambda strings as the
reference (train.py:270,368).  TensorBoard summaries, checkpoint timers and the data loader are host glue outside the
hot path.  Multi-GPU is one process per GPU (torch.distributed, NCCL) instead of the reference's nn.DataParallel.
"""
import configparser
import warnings

import torch
import torch.distributed as dist
import torch.nn as nn

import model
from b200 import ddp as _ddp


def norm_data(data, height, width, rows, cols, keys='yx_min, yx_max'):
    """GT pixel coordinates -> grid units (reference train.py:57-62)."""
    out = {key: data[key] for key in data}
    sy, sx = rows / height, cols / width
    for key in keys.split(', '):
        t = out[key]
        # Python-scalar multiplies only: no host tensor is created, so the step stays CUDA-graph capturable
        out[key] = torch.stack([t[..., 0] * sy, t[..., 1] * sx], -1)
    return out


def ensure_model(module):
    """reference train.py:65-71: move to the GPU; with more than one GPU the reference wraps the module in nn.DataParallel,
    which re-replicates GPU 0's parameters and buffers on every step.  Here replication is one process per GPU
    (torch.distributed): nothing is wrapped, every rank's parameters and buffers are made equal to rank 0's once, and the
    gradient exchange (b200.ddp) is attached by `iterate`."""
    if not torch.cuda.is_available():
        raise RuntimeError('train: a CUDA device is required; there is no CPU fallback')
    module = module.cuda()
    reducer = _ddp.default_reducer()
    if reducer is not None:
        sync_replicas(module, reducer)
    return module


def sync_replicas(module, reducer):
    """Broadcast rank 0's parameters and buffers (once per module per reducer)."""
    if getattr(module, '_yb_synced_with', None) is not reducer:
        reducer.broadcast_module(module)
        module._yb_synced_with = reducer


def build_optimizer(config, params, lr):
    """`train/optimizer` is a Python lambda in the INI, exactly as in the reference (config.ini:72, train.py:270)."""
    return eval(config.get('train', 'optimizer'))(params, lr)


def loss_scale_config(config):
    """(mode, growth_interval) from `[train] loss_scale` ('static' when absent, or 'dynamic') and `[train] loss_scale_growth_interval`
    (default 2000, a positive integer).  A bad value raises ValueError naming its key."""
    def get(key, default):
        return config.get('train', key).strip() if config.has_option('train', key) else default

    mode = get('loss_scale', 'static')
    if mode not in ('static', 'dynamic'):
        raise ValueError('[train] loss_scale must be static or dynamic, got %r' % mode)
    interval = get('loss_scale_growth_interval', '2000')
    try:
        interval = int(interval)
    except ValueError:
        raise ValueError('[train] loss_scale_growth_interval must be a positive integer, got %r' % interval) from None
    if interval <= 0:
        raise ValueError('[train] loss_scale_growth_interval must be a positive integer, got %d' % interval)
    return mode, interval


def iterate(inference, optimizer, anchors, config, data, reducer=None):
    """One training step (reference Train.iterate, train.py:338-362).  `data`: dict with `tensor` [B,3,H,W] fp32 (or uint8 frames
    [B,H,W,3], put through the backbone's input_transform, else ToTensor), `yx_min`/`yx_max` [B,G,2] in pixels, `cls` [B,G].  Returns the same kind of dict as the reference; with `[train] loss_scale =
    dynamic` it also holds `loss_scale`, the device scale (the trainer's static scale times its dynamic factor) the next step runs at."""
    dev = torch.device('cuda', torch.cuda.current_device())
    data = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) else v) for k, v in data.items()}
    tensor = data['tensor']
    dnn = inference.dnn
    if tensor.dtype == torch.uint8:                 # uint8 NHWC frames from utils.data.Collate: the input transform on the device
        if getattr(dnn, 'input_transform', None) is not None:
            tensor = dnn.input_transform(tensor)
        else:
            import transform
            tensor = transform.to_tensor(tensor)
    height, width = tensor.shape[-2:]
    if reducer is False:                           # this rank alone, no collective (compute-only timing of a data-parallel step)
        with _ddp.local_only():
            return iterate(inference, optimizer, anchors, config, data, None)
    if reducer is None:
        reducer = _ddp.default_reducer()          # torch.distributed initialised with world > 1: data parallel
    elif _ddp.default_reducer(create=False) is None:
        _ddp.set_default_reducer(reducer)          # model.loss normalises the class term through the same communicator
    if reducer is not None:
        sync_replicas(inference, reducer)          # unseeded ranks would otherwise train different models on averaged gradients
    trainer = dnn.trainer
    trainer.reducer = reducer
    trainer.set_loss_scale(*loss_scale_config(config))
    pred = model._inference(inference, tensor)
    rows, cols = pred['feature'].shape[-2:]
    cross_entropy = config.getboolean('train', 'cross_entropy') if config.has_option('train', 'cross_entropy') else True
    loss, debug = model.loss(anchors, norm_data(data, height, width, rows, cols), pred, config.getfloat('model', 'threshold'), cross_entropy)
    loss_hparam = {key: loss[key] * config.getfloat('hparam', key) for key in loss}
    loss_total = sum(loss_hparam.values())
    optimizer.zero_grad()
    loss_total.backward()          # ends with the main stream joined to the gradient all-reduces (b200.train_engine.backward)
    try:
        clip = config.getfloat('train', 'clip')
        nn.utils.clip_grad_norm_(inference.parameters(), clip)
    except (configparser.NoOptionError, configparser.NoSectionError):
        pass
    if getattr(optimizer, '_step_supports_amp_scaling', False):
        # fused torch.optim optimizers skip the update (state untouched) when found_inf is raised -- the overflow guard of the fp16
        # backward (b200.train_engine.backward); the others step on the zeroed gradients
        optimizer.found_inf = trainer.found_inf
        optimizer.grad_scale = None
    elif trainer.loss_scale == 'dynamic' and not getattr(trainer, '_warned_found_inf', False):
        trainer._warned_found_inf = True
        warnings.warn('[train] loss_scale = dynamic: %s cannot skip a step on found_inf, so each overflowed step (routine while the scale '
                      'backs off) is a step on zeroed gradients; a fused optimizer (e.g. torch.optim.Adam(..., fused=True)) skips it'
                      % type(optimizer).__name__, RuntimeWarning)
    optimizer.step()
    # What is returned is for summaries / logging only (the reference reads .data / float() of it, train.py:353-362), so it is detached:
    # a caller that keeps the dict must not keep the autograd graph -- and with it the parameters' AccumulateGrad nodes, which remember
    # the stream they were created on -- alive: a later CUDA-graph capture of the step would then have to synchronise with that
    # uncaptured stream (cudaErrorStreamCaptureIsolation; found with tests/test_ddp_nccl.py).
    def _d(v):
        return v.detach() if torch.is_tensor(v) else v

    out = dict(height=height, width=width, rows=rows, cols=cols, data=data, pred={k: _d(v) for k, v in pred.items()}, debug=debug,
               loss_total=loss_total.detach(), loss={k: _d(v) for k, v in loss.items()}, loss_hparam={k: _d(v) for k, v in loss_hparam.items()})
    if trainer.loss_scale == 'dynamic':
        out['loss_scale'] = trainer.loss_scale_state(dev)[0] * trainer.grad_scale
    return out


class GraphedStep(object):
    """`iterate` captured once per input shape into a CUDA graph and replayed: the ~300 kernel launches, the autograd
    bookkeeping and the optimizer step of one training iteration cost one graph launch, which removes the host
    launch overhead that dominates the eager step (wgmma kernels of 20-100 us each).

        step = train.GraphedStep(inference, optimizer, anchors, config)
        out = step(dict(tensor=..., yx_min=..., yx_max=..., cls=...))      # same dict as iterate()

    * Inputs (host-pinned or device tensors) are copied into static device buffers, then the graph is replayed; the
      returned tensors are static too (overwritten by the next call with the same shapes).
    * One graph per distinct set of input shapes (multi-scale training, `data/sizes`: one per size).
    * Capture needs two eager warm-up iterations (lazy optimizer state, kernel attribute setup).  Parameters, buffers,
      optimizer state and the dynamic loss scale's factor and growth tracker are restored afterwards, so the first replay
      is the first real update.
    * The optimizer must be capture-safe: torch.optim.SGD as is, Adam/AdamW with `capturable=True`.  The learning
      rate is baked into the graph unless it is a tensor (`lr=torch.tensor(...)`).
    * Operand caches keyed by parameter version (packed fp16 weights) are refreshed inside the graph; call
      `finish()` before switching the model to eval() so the inference engine re-packs from the final parameters.
    """

    def __init__(self, inference, optimizer, anchors, config, reducer=None, warmup=2):
        self.inference, self.optimizer, self.anchors, self.config, self.reducer = inference, optimizer, anchors, config, reducer
        self.warmup = int(warmup)
        self.graphs = {}
        self.launches = 0          # library kernels replayed so far (bench.py's gpu_launches)
        self.keys = ('tensor', 'yx_min', 'yx_max', 'cls')

    def _snapshot(self, dev):
        mod = self.inference
        tensors = [p.data for p in mod.parameters()] + [b for b in mod.buffers()]
        mode, interval = loss_scale_config(self.config)
        if mode == 'dynamic':
            trainer = mod.dnn.trainer
            trainer.set_loss_scale(mode, interval)
            tensors += trainer.loss_scale_state(dev)          # the factor and tracker, created here at 1 and 0 if new
        saved = [(t, t.clone()) for t in tensors]
        state = {}
        for p, st in self.optimizer.state.items():
            for k, v in st.items():
                if torch.is_tensor(v):
                    state[(id(p), k)] = v.clone()
        return saved, state

    def _restore(self, snap):
        saved, state = snap
        for t, c in saved:
            t.copy_(c)
        for p, st in self.optimizer.state.items():
            for k, v in st.items():
                if torch.is_tensor(v):
                    c = state.get((id(p), k))
                    if c is not None:
                        v.copy_(c)
                    else:
                        v.zero_()      # state created lazily by the warm-up steps: back to its initial value

    def _capture(self, key, data, dev):
        from b200 import ops as _ops
        static = {k: data[k].to(dev).clone() for k in self.keys}
        self.anchors = self.anchors.detach().to(device=dev, dtype=torch.float32).contiguous()   # no host->device copy inside the capture
        red = None if self.reducer is False else (self.reducer if self.reducer is not None else _ddp.default_reducer())
        if red is not None:
            sync_replicas(self.inference, red)      # before the snapshot: the restore below must not undo rank 0's broadcast
        snap = self._snapshot(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                iterate(self.inference, self.optimizer, self.anchors, self.config, static, self.reducer)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self._restore(snap)
        self.optimizer.zero_grad(set_to_none=True)
        graph = torch.cuda.CUDAGraph()
        n0 = _ops.launch_count
        with torch.cuda.graph(graph):
            out = iterate(self.inference, self.optimizer, self.anchors, self.config, static, self.reducer)
        entry = (static, graph, out, _ops.launch_count - n0)
        self.graphs[key] = entry
        return entry

    def __call__(self, data):
        dev = torch.device('cuda', torch.cuda.current_device())
        key = tuple(tuple(data[k].shape) for k in self.keys)
        entry = self.graphs.get(key)
        if entry is None:
            entry = self._capture(key, data, dev)
        static, graph, out, launches = entry
        for k in self.keys:
            static[k].copy_(data[k], non_blocking=True)
        graph.replay()
        self.launches += launches
        return out

    def finish(self):
        """Drop operand caches that the graph kept current on its own buffers (see the class docstring)."""
        self.inference.dnn.drop_operands()

    def close(self):
        """Destroy the captured graphs (required before the NCCL communicator whose collectives they captured is destroyed)."""
        self.finish()
        self.graphs.clear()
