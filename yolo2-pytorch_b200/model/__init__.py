"""model -- detection head helpers of the plugin surface, H100-native.

Mirrors the public names of ruiminshen/yolo2-pytorch `model/__init__.py` (reference file:line per
item) so `detect.py`/`train.py`-style callers keep working: `ConfigChannels` (:29-43),
`output_channels` (:46-50), `meshgrid` (:53-56), `Inference` (:110-135), `_inference` (:170-179),
`loss` (:138-167).  The decode (sigmoid xy/objectness, exp wh * anchors, class softmax) is ONE CUDA
kernel (yb_decode_fwd); nothing here computes on the CPU.
"""
import logging

import torch
import torch.nn as nn

import torch.distributed as _dist

from b200 import ddp as _ddp
from b200 import engine as _engine
from b200 import ops as _ops
import transform as _transform


class _TrainFunction(torch.autograd.Function):
    """Training-mode forward/backward of a whole backbone as one autograd node: forward runs the plugin's train-mode kernel chain
    (batch-statistics BatchNorm, running-stat update), backward its explicit backward chain (b200.train_engine) and hands every parameter
    its fp32 gradient."""

    @staticmethod
    def forward(ctx, dnn, x, *params):
        feature, saved = dnn.trainer.forward(x)
        ctx.dnn, ctx.saved = dnn, saved
        return feature

    @staticmethod
    def backward(ctx, dfeature):
        dnn = ctx.dnn
        grads = dnn.trainer.backward(ctx.saved, dfeature)
        ctx.saved = None
        # The gradients live in the trainer's persistent arena (b200.ddp.GradArena; in data-parallel runs its buckets are being
        # all-reduced in place right now).  `.grad` is bound to those views directly -- handing them to autograd instead would let
        # AccumulateGrad clone them whenever it cannot steal the tensor, silently detaching `.grad` from the reduced buffer.
        # Like the reference (zero_grad before every backward, train.py:350), gradients are not accumulated across calls.
        params = list(dnn.named_parameters())
        for name, p in params:
            p.grad = grads[name]
        return (None, None) + (None,) * len(params)


class Backbone(nn.Module):
    """Base of the backbone plugins.  Holds the kernel operands cached per parameter version (`_cache`), the lazily built trainer (an
    instance of the b200.train_engine class `TRAINER`) and the train-mode entry through it.

    In eval mode every backbone takes either the fp32 NCHW image [B,3,H,W], taken as already transformed (as the reference's model takes
    it), or a uint8 NHWC frame batch [B,H,W,3], which its first-layer kernel reads through `input_transform`'s table."""
    TRAINER = None
    input_transform = None

    def __init__(self):
        nn.Module.__init__(self)
        self._cache = _engine.OperandCache()
        self._trainer = None

    @property
    def trainer(self):
        if self._trainer is None:
            self._trainer = self.TRAINER(self)
        return self._trainer

    def drop_operands(self):
        """Forget every cached kernel operand."""
        self._cache.clear()

    def set_input_transform(self, t):
        """The tensor transform (transform.TensorTransform, e.g. the reference's `[transform] tensor` chain) that uint8 frame batches go
        through: in the first-layer kernel in eval mode, and in train.iterate before a training step.  None (the default): ToTensor alone
        (Darknet's uint8 path then scales by 1/255 in its kernel, as it always has).  Set it before capturing a CUDA graph.  Returns self."""
        if t is not None and not isinstance(t, _transform.TensorTransform):
            raise TypeError('set_input_transform expects a transform.TensorTransform or None, not %r' % (t,))
        self.input_transform = t
        return self

    def input_lut(self, device):
        """The table fp32 [3, 256] on `device` that a uint8 frame batch goes through: input_transform's, else ToTensor's."""
        t = self.input_transform if self.input_transform is not None else _transform.to_tensor_transform()
        return t.lut(device)

    def eval_input(self, x):
        """An eval-mode input -> (x, lut, (B, C, H, W)): a uint8 frame batch [B,H,W,C] with its table, or the fp32 image [B,C,H,W] with None."""
        if x.dtype == torch.uint8:
            if x.dim() != 4:
                raise ValueError('%s expects uint8 frames [B,H,W,3], got %s' % (type(self).__name__, tuple(x.shape)))
            b, h, w, c = x.shape
            return x.contiguous(), self.input_lut(x.device), (b, c, h, w)
        b, c, h, w = x.shape
        return x.contiguous().float(), None, (b, c, h, w)

    def train(self, mode=True):
        """nn.Module.train + drop cached kernel operands on a mode switch: fused optimizers and CUDA-graph replays update parameters without
        advancing torch's version counters, so inference after training re-packs from the trained state."""
        if bool(mode) != self.training:
            self.drop_operands()
        return nn.Module.train(self, mode)

    def train_forward(self, x):
        """Batch-statistics BatchNorm + autograd through the explicit backward chain of `TRAINER`."""
        return _TrainFunction.apply(self, x, *[p for _, p in self.named_parameters()])


class ConfigChannels(object):
    """Plugin constructor contract (reference model/__init__.py:29-43): tracks the current channel
    count; `cc(default, key)` returns the layer's output channels -- `state_dict[key].size(0)` when a
    checkpoint is supplied (channel-pruned models), else `default`."""

    def __init__(self, config, state_dict=None, channels=3):
        self.config = config
        self.state_dict = state_dict
        self.channels = channels

    def __call__(self, default, name, fn=lambda var: var.size(0)):
        if self.state_dict is None:
            self.channels = default
            return default
        found = fn(self.state_dict[name])
        if found != default:
            logging.warning('%s: change number of output channels from %d to %d' % (name, default, found))
        self.channels = found
        return found


def output_channels(num_anchors, num_cls):
    """Head width A*(5+C), or A*5 for single-class models (reference model/__init__.py:46-50)."""
    return num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5


def meshgrid(rows, cols, swap=False):
    """Cell coordinates exactly as the reference builds them (model/__init__.py:53-56): row k is
    (k // rows, k % rows) -- a true (row, col) grid only when rows == cols.  Host helper; the decode
    kernel derives the same pair from the cell index."""
    k = torch.arange(0, rows * cols)
    a, b = k // rows, k % rows
    return torch.stack([b, a] if swap else [a, b], 1)


class Inference(nn.Module):
    """backbone + anchor-box decode (reference model/__init__.py:110-135).  forward(x) returns the
    same 7-tuple: (feature, iou, center_offset, size_norm, yx_min, yx_max, logits)."""

    def __init__(self, config, dnn, anchors):
        nn.Module.__init__(self)
        self.config = config
        self.dnn = dnn
        self.anchors = anchors
        self._anchors_dev = None
        self.last_prob = None

    def _anchors_on(self, device):
        if self._anchors_dev is None or self._anchors_dev.device != device:
            self._anchors_dev = self.anchors.detach().to(device=device, dtype=torch.float32).contiguous()
        return self._anchors_dev

    def forward(self, x):
        feature = self.dnn(x)
        if not feature.is_cuda:
            raise RuntimeError('model.Inference: the backbone must return a CUDA tensor; there is no CPU fallback')
        anchors = self._anchors_on(feature.device)
        a = anchors.size(0)
        per = feature.size(1) // a
        num_cls = per - 5 if per > 5 else 1
        out = _ops.decode(feature.contiguous().float(), anchors, num_cls, with_prob=True)
        self.last_prob = out['prob']
        return feature, out['iou'], out['center_offset'], out['size_norm'], out['yx_min'], out['yx_max'], out.get('logits')


def _inference(inference, tensor):
    """Tuple -> dict (reference model/__init__.py:170-179).  One extra key, `prob`, carries the
    class softmax the decode kernel already produced (the reference recomputes it at detect.py:152)."""
    feature, iou, center_offset, size_norm, yx_min, yx_max, logits = inference(tensor)
    pred = dict(feature=feature, iou=iou, center_offset=center_offset, size_norm=size_norm, yx_min=yx_min, yx_max=yx_max)
    if logits is not None:
        pred['logits'] = logits
    prob = getattr(inference, 'last_prob', None)
    if prob is None and hasattr(inference, 'module'):
        prob = getattr(inference.module, 'last_prob', None)
    if prob is not None:
        pred['prob'] = prob
    return pred


class _RegionLoss(torch.autograd.Function):
    """feature -> the five region-loss scalars; backward = one kernel combining the stored per-term
    gradients with the upstream weights (no host sync)."""

    @staticmethod
    def forward(ctx, feature, anchors, yx_min, yx_max, cls, threshold, cross_entropy, holder):
        out = _ops.region_loss_forward(feature.detach().contiguous().float(), anchors, yx_min, yx_max, cls, threshold, cross_entropy)
        ctx.save_for_backward(out['grad_terms'], out['grad_bg'])
        ctx.num_anchors = anchors.size(0)
        holder.update(out)
        losses = out['losses']
        return losses[0], losses[1], losses[2], losses[3], losses[4]

    @staticmethod
    def backward(ctx, g0, g1, g2, g3, g4):
        grad_terms, grad_bg = ctx.saved_tensors
        zero = torch.zeros((), dtype=torch.float32, device=grad_terms.device)
        w = torch.stack([zero if g is None else g.float() for g in (g0, g1, g2, g3, g4)])
        return _ops.region_loss_backward(grad_terms, grad_bg, w.contiguous(), ctx.num_anchors), None, None, None, None, None, None, None


def loss(anchors, data, pred, threshold, cross_entropy=True):
    """Region loss (reference model/__init__.py:138-167) as fused CUDA kernels: target assignment
    (iou_match :59-73, fit_positive :76-95, fill_norm :98-103), the five terms and the closed-form
    gradient w.r.t. the head feature map.  `data` holds yx_min / yx_max [B,G,2] in GRID units
    (train.norm_data) and cls [B,G]; zero-padded slots are allowed.  Returns (dict of 5 scalars that
    back-propagate into pred['feature'], debug dict) like the reference.  `cross_entropy` mirrors
    train/cross_entropy (config.ini:77; the reference infers it from the rank of data['cls'])."""
    feature = pred['feature']
    if not feature.is_cuda:
        raise RuntimeError('model.loss: tensors must be on the GPU; there is no CPU fallback')
    dev = feature.device
    anchors = anchors.detach().to(device=dev, dtype=torch.float32).contiguous()
    yx_min = data['yx_min'].to(device=dev, dtype=torch.float32).contiguous()
    yx_max = data['yx_max'].to(device=dev, dtype=torch.float32).contiguous()
    cls = data['cls'].to(device=dev, dtype=torch.int64).contiguous()
    aux = {}
    values = _RegionLoss.apply(feature, anchors, yx_min, yx_max, cls, float(threshold), bool(cross_entropy), aux)
    names = ('foreground', 'background', 'center', 'size', 'cls')
    per = feature.size(1) // anchors.size(0)
    losses = {k: v for k, v in zip(names, values) if k != 'cls' or per > 5}
    if 'cls' in losses and cross_entropy and _dist.is_available() and _dist.is_initialized() and _dist.get_world_size() > 1:
        # data parallel: the class term is a mean over the positives of the WHOLE batch in the reference (loss on the
        # gathered batch, train.py:344-347); re-weight this rank's mean so that the rank-averaged gradient matches it
        losses['cls'] = losses['cls'] * _ddp.global_mean_factor(aux['pos_count'].sum())
    debug = dict(iou=aux['best_iou'], positive=aux['positive'], negative=aux['negative'], pos_count=aux['pos_count'])
    return losses, debug
