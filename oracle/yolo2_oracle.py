"""CPU oracle for the YOLOv2 hot path -- TEST INFRASTRUCTURE ONLY.

This file is a CPU restatement (torch fp32 on CPU + numpy) of the algorithm on the hot path of
ruiminshen/yolo2-pytorch.  It is the checker for the CUDA kernels: only `tests/`,
`__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference` legs of `bench.py` may
import it.  Nothing under `yolo2-pytorch_b200/` (the product) imports this module.

Parity status
-------------
* backbone / reorg / decode / softmax / filter / NMS / IoU: PINNED -- every function below is
  checked in `tests/test_oracle_golden.py` against fixtures in `tests/golden/*.npz` that were
  produced by executing the *reference's own code* (`/root/reference`, imported with the one-line
  `async` rename that Python >= 3.7 needs) by `tests/golden/make_golden.py`, plus the reference's
  embedded IoU known-answer tests (`utils/iou/torch.py:79-113,179-213`).
* region loss (`loss`, `iou_match`, `fit_positive`, `fill_norm`): PINNED BY EXECUTION UNDER TWO SHIMS.
  The reference's `model.loss` does not run on torch >= 0.4 as is (IndexError at
  `model/__init__.py:154`, and `fit_positive` silently mis-masks because `torch.prod` of a
  comparison is no longer a mask).  `tests/golden/make_golden_loss.py` executes the reference's
  unmodified loss source with the two torch-0.3.1 behaviours supplied from outside (masks stay masks
  under `prod`; `x[mask]` broadcasts the mask) and stores losses, masks, matched IoU and the gradient
  w.r.t. the head feature map for four cases (13x13, 19x19, one ground-truth slot, the one-hot branch);
  `tests/test_oracle_golden.py::test_region_loss_oracle_matches_executed_reference` checks the
  restatement below against them (terms 1e-5, masks exact, gradient 1e-4).  The restatement writes the
  same 0.3.1 semantics out explicitly; each deviation is commented.
* one whole training step (train-mode backbone + loss + autograd + running statistics): PINNED against the step executed
  with the reference's own modules (`tests/golden/make_golden_train.py`).
* Tiny backbone, evaluation matching / VOC AP, Darknet head permutation, cv2-exact resize: PINNED by
  fixtures made with the reference's functions (and cv2) -- see the generators under `tests/golden/`.

The conv / BN / pooling / softmax / sort arithmetic of the reference lives in its third-party
dependency torch (`requirements.txt:5`, `torch<=0.3.1`, not vendored); the restatement calls the
same library ops (`F.conv2d`, `F.batch_norm`, ...) in fp32 on CPU, which is what "the reference's
CPU PyTorch path" is.

All citations are `file:line` into /root/reference (ruiminshen/yolo2-pytorch @ 146ebdf).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

EPS32 = float(np.finfo(np.float32).eps)  # utils/iou/torch.py:47 default `min`

# ----------------------------------------------------------------------------------------------
# Topology (model/yolo2.py:69-115)
# ----------------------------------------------------------------------------------------------

def darknet19_layers(num_anchors=5, num_cls=20, ratio=1):
    """Return the Darknet-19 layer list as dicts in module-registration order.

    Follows model/yolo2.py:76-113.  Each conv entry: key (state_dict prefix), cin, cout, k, bn, act;
    `pool_after` says a MaxPool2d(2) follows (yolo2.py:79,86), `group` is the nn.Sequential name.
    """
    L = []
    cin = 3
    ch = int(32 * ratio)
    idx = 0

    def add(group, i, cout, k, bn=True, act=True):
        nonlocal cin
        L.append(dict(key='%s.%d' % (group, i), group=group, cin=cin, cout=cout, k=k, bn=bn, act=act, pool_after=False))
        cin = cout

    # layers1 (yolo2.py:77-93)
    for _ in range(2):
        add('layers1', idx, ch, 3); idx += 1
        L[-1]['pool_after'] = True; idx += 1
        ch *= 2
    for _ in range(2):
        add('layers1', idx, ch, 3); idx += 1
        add('layers1', idx, ch // 2, 1); idx += 1
        add('layers1', idx, ch, 3); idx += 1
        L[-1]['pool_after'] = True; idx += 1
        ch *= 2
    for _ in range(2):
        add('layers1', idx, ch, 3); idx += 1
        add('layers1', idx, ch // 2, 1); idx += 1
    add('layers1', idx, ch, 3); idx += 1
    c_l1 = cin
    # layers2 (yolo2.py:96-105): index 0 is the MaxPool
    idx = 1
    ch *= 2
    for _ in range(2):
        add('layers2', idx, ch, 3); idx += 1
        add('layers2', idx, ch // 2, 1); idx += 1
    for _ in range(3):
        add('layers2', idx, ch, 3); idx += 1
    c_l2 = cin
    # passthrough (yolo2.py:107)
    c_pt = int(64 * ratio)
    L.append(dict(key='passthrough', group='passthrough', cin=c_l1, cout=c_pt, k=1, bn=True, act=True, pool_after=False))
    # layers3 (yolo2.py:110-113)
    cin = c_pt * 4 + c_l2
    add('layers3', 0, int(1024 * ratio), 3)
    cout_head = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5  # model/__init__.py:46-50
    add('layers3', 1, cout_head, 1, bn=False, act=False)
    return L


def make_state_dict(seed=0, num_anchors=5, num_cls=20, ratio=1, bn_random=True):
    """Deterministic synthetic Darknet-19 state_dict (SURVEY section 8d).

    Conv weights: kaiming-normal (fan_in, gain sqrt(2)) as `Darknet.init` does (yolo2.py:117-123);
    BN tensors randomised so that BN folding is actually exercised (at init BN is the identity);
    head bias ~ N(0, 0.1).  Keys are exactly the reference module's state_dict keys.
    """
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for l in darknet19_layers(num_anchors, num_cls, ratio):
        fan_in = l['cin'] * l['k'] * l['k']
        std = math.sqrt(2.0 / fan_in)
        sd[l['key'] + '.conv.weight'] = torch.randn(l['cout'], l['cin'], l['k'], l['k'], generator=g) * std
        if l['bn']:
            c = l['cout']
            if bn_random:
                sd[l['key'] + '.bn.weight'] = torch.rand(c, generator=g) + 0.5
                sd[l['key'] + '.bn.bias'] = torch.randn(c, generator=g) * 0.1
                sd[l['key'] + '.bn.running_mean'] = torch.randn(c, generator=g) * 0.1
                sd[l['key'] + '.bn.running_var'] = torch.rand(c, generator=g) + 0.5
            else:
                sd[l['key'] + '.bn.weight'] = torch.ones(c)
                sd[l['key'] + '.bn.bias'] = torch.zeros(c)
                sd[l['key'] + '.bn.running_mean'] = torch.zeros(c)
                sd[l['key'] + '.bn.running_var'] = torch.ones(c)
        else:
            sd[l['key'] + '.conv.bias'] = torch.randn(l['cout'], generator=g) * 0.1
    return sd


ANCHORS_YOLO_VOC_WH = [  # config/anchors/yolo-voc.tsv:1-6 (columns: width, height; grid units)
    (1.3221, 1.73145), (3.19275, 4.00944), (5.05587, 8.09892), (9.47112, 4.84053), (11.2364, 10.0071)]


def anchors_yolo_voc():
    """[A,2] float32 tensor in (height, width) order, as utils/__init__.py:78-81 loads it."""
    return torch.tensor([[h, w] for (w, h) in ANCHORS_YOLO_VOC_WH], dtype=torch.float32)


# ----------------------------------------------------------------------------------------------
# Backbone (model/yolo2.py:33-65,125-130)
# ----------------------------------------------------------------------------------------------

def reorg(x, stride_h=2, stride_w=2):
    """model/yolo2.py:33-46 (branch `if 1`): out[b,(sh*sw_n+sw)*C+c,h',w'] = x[b,c,sh_n*h'+sh,...]."""
    b, c, h, w = x.shape
    _h, _w = h // stride_h, w // stride_w
    x = x.reshape(b, c, _h, stride_h, _w, stride_w)
    x = x.permute(0, 3, 5, 1, 2, 4)  # b, sh, sw, c, _h, _w
    return x.reshape(b, stride_h * stride_w * c, _h, _w).contiguous()


def conv_unit(x, sd, key, k, bn, act, train=False, stats=None):
    """model/yolo2.py:49-65: conv(k, stride 1, pad (k-1)//2, bias=not bn) -> BN(eps 1e-5) -> LeakyReLU(0.1)."""
    bias = None if bn else sd.get(key + '.conv.bias')
    y = F.conv2d(x, sd[key + '.conv.weight'], bias, stride=1, padding=(k - 1) // 2)
    if bn:
        if train:
            mean = y.mean(dim=(0, 2, 3))
            var = y.var(dim=(0, 2, 3), unbiased=False)
            if stats is not None:
                stats[key] = (mean, var)
            y = F.batch_norm(y, None, None, sd[key + '.bn.weight'], sd[key + '.bn.bias'], True, 0.0, 1e-5)
        else:
            y = F.batch_norm(y, sd[key + '.bn.running_mean'], sd[key + '.bn.running_var'],
                             sd[key + '.bn.weight'], sd[key + '.bn.bias'], False, 0.0, 1e-5)
    if act:
        y = F.leaky_relu(y, 0.1)
    return y


def darknet_forward(sd, x, num_anchors=5, num_cls=20, collect=None, train=False, stats=None):
    """model/yolo2.py:125-130.  `collect` (dict) receives every conv unit's output (pre-pool)."""
    layers = darknet19_layers(num_anchors, num_cls)
    by_group = {}
    for l in layers:
        by_group.setdefault(l['group'], []).append(l)

    def run(group, x, pre_pool=False):
        if pre_pool:
            x = F.max_pool2d(x, 2)
        for l in by_group[group]:
            x = conv_unit(x, sd, l['key'], l['k'], l['bn'], l['act'], train, stats)
            if collect is not None:
                collect[l['key']] = x
            if l['pool_after']:
                x = F.max_pool2d(x, 2)
        return x

    x1 = run('layers1', x)
    _x = reorg(run('passthrough', x1), 2, 2)
    x2 = run('layers2', x1, pre_pool=True)
    return run('layers3', torch.cat([_x, x2], 1))


# ----------------------------------------------------------------------------------------------
# Head decode (model/__init__.py:53-56,110-135,170-179)
# ----------------------------------------------------------------------------------------------

def meshgrid(rows, cols):
    """model/__init__.py:53-56 with swap=False: row k -> (k // rows ... ) exactly as the reference
    builds it (only a true (row, col) grid when rows == cols)."""
    i = torch.arange(0, rows).repeat(cols).view(-1, 1)
    j = torch.arange(0, cols).view(-1, 1).repeat(1, rows).view(-1, 1)
    return torch.cat([j, i], 1)


def decode(feature, anchors):
    """model/__init__.py:117-135 + 170-179: feature [B,A*(5+C),S,S] -> pred dict."""
    b = feature.size(0)
    rows, cols = feature.shape[-2:]
    cells = rows * cols
    a = anchors.size(0)
    _f = feature.permute(0, 2, 3, 1).contiguous().view(b, cells, a, -1)
    sig = torch.sigmoid(_f[:, :, :, :3])
    iou = sig[:, :, :, 0]
    ij = meshgrid(rows, cols).view(1, -1, 1, 2).to(feature.dtype)
    center_offset = sig[:, :, :, 1:3]
    center = ij + center_offset
    size_norm = _f[:, :, :, 3:5]
    size = torch.exp(size_norm) * anchors.view(1, 1, -1, 2)
    size2 = size / 2
    pred = dict(feature=feature, iou=iou, center_offset=center_offset, size_norm=size_norm,
                yx_min=center - size2, yx_max=center + size2)
    if _f.size(-1) > 5:
        pred['logits'] = _f[:, :, :, 5:].contiguous()
    return pred


def class_prob(pred):
    """detect.py:43-48,152: softmax over classes of the logits (ones if single-class)."""
    if 'logits' in pred:
        return F.softmax(pred['logits'], -1)
    return torch.ones(*pred['iou'].shape, 1)


# ----------------------------------------------------------------------------------------------
# IoU (utils/iou/torch.py:24-61,116-153)
# ----------------------------------------------------------------------------------------------

def iou_matrix(yx_min1, yx_max1, yx_min2, yx_max2, min=EPS32):
    """[N1,2]x2 vs [N2,2]x2 -> [N1,N2]; operation order of utils/iou/torch.py:24-61."""
    ymin1, xmin1 = yx_min1[:, 0:1], yx_min1[:, 1:2]
    ymax1, xmax1 = yx_max1[:, 0:1], yx_max1[:, 1:2]
    ymin2, xmin2 = yx_min2[:, 0:1].t(), yx_min2[:, 1:2].t()
    ymax2, xmax2 = yx_max2[:, 0:1].t(), yx_max2[:, 1:2].t()
    height = torch.clamp(torch.min(ymax1, ymax2) - torch.max(ymin1, ymin2), min=0)
    width = torch.clamp(torch.min(xmax1, xmax2) - torch.max(xmin1, xmin2), min=0)
    inter = height * width
    area1 = torch.prod(yx_max1 - yx_min1, -1).unsqueeze(-1)
    area2 = torch.prod(yx_max2 - yx_min2, -1).unsqueeze(-2)
    union = torch.clamp(area1 + area2 - inter, min=min)
    return inter / union


def batch_iou_matrix(yx_min1, yx_max1, yx_min2, yx_max2, min=EPS32):
    """[B,N1,2]x2 vs [B,N2,2]x2 -> [B,N1,N2]; utils/iou/torch.py:116-153."""
    ymin1, xmin1 = yx_min1[..., 0:1], yx_min1[..., 1:2]
    ymax1, xmax1 = yx_max1[..., 0:1], yx_max1[..., 1:2]
    ymin2, xmin2 = yx_min2[..., 0:1].transpose(1, 2), yx_min2[..., 1:2].transpose(1, 2)
    ymax2, xmax2 = yx_max2[..., 0:1].transpose(1, 2), yx_max2[..., 1:2].transpose(1, 2)
    height = torch.clamp(torch.min(ymax1, ymax2) - torch.max(ymin1, ymin2), min=0)
    width = torch.clamp(torch.min(xmax1, xmax2) - torch.max(xmin1, xmin2), min=0)
    inter = height * width
    area1 = torch.prod(yx_max1 - yx_min1, -1).unsqueeze(-1)
    area2 = torch.prod(yx_max2 - yx_min2, -1).unsqueeze(-2)
    union = torch.clamp(area1 + area2 - inter, min=min)
    return inter / union


# ----------------------------------------------------------------------------------------------
# NMS + detection post-filter (utils/postprocess.py:23-49, detect.py:51-80)
# ----------------------------------------------------------------------------------------------

def nms(score, yx_min, yx_max, overlap=0.5, limit=200):
    """Greedy class-agnostic NMS, utils/postprocess.py:23-49.  Returns list[int] (indices into the
    inputs, descending score).  numpy float32 arithmetic in the order of iou_matrix above."""
    score = np.asarray(score, dtype=np.float32)
    a = np.asarray(yx_min, dtype=np.float32)
    b = np.asarray(yx_max, dtype=np.float32)
    keep = []
    if score.size == 0:
        return keep
    index = np.argsort(-score, kind='stable')[:limit]
    thr = np.float32(overlap)
    eps = np.float32(EPS32)
    area = (b[:, 0] - a[:, 0]) * (b[:, 1] - a[:, 1])
    while index.size > 0:
        i = int(index[0])
        keep.append(i)
        if index.size == 1:
            break
        index = index[1:]
        h = np.maximum(np.minimum(b[i, 0], b[index, 0]) - np.maximum(a[i, 0], a[index, 0]), np.float32(0))
        w = np.maximum(np.minimum(b[i, 1], b[index, 1]) - np.maximum(a[i, 1], a[index, 1]), np.float32(0))
        inter = h * w
        union = np.maximum(area[i] + area[index] - inter, eps)
        iou = inter / union
        index = index[iou <= thr]
    return keep


def filter_visible(iou, yx_min, yx_max, prob, fix, threshold, threshold_cls):
    """detect.py:51-63 for ONE image: iou [N], yx_* [N,2], prob [N,C] (flattened cells*anchors)."""
    prob_cls, cls = torch.max(prob, -1)
    mask = (iou * prob_cls) > threshold_cls if fix else iou > threshold
    return iou[mask], yx_min[mask], yx_max[mask], prob[mask], prob_cls[mask], cls[mask], mask


def postprocess(iou, yx_min, yx_max, prob, fix, threshold, threshold_cls, overlap):
    """detect.py:66-80 for ONE image.  Returns None when nothing is kept (as the reference's
    implicit fall-through does), else (iou[k], yx_min[m,2], yx_max[m,2], cls[m], score[m])."""
    iou, yx_min, yx_max, prob, prob_cls, cls, _ = filter_visible(iou, yx_min, yx_max, prob, fix, threshold, threshold_cls)
    keep = nms(iou.numpy(), yx_min.numpy(), yx_max.numpy(), overlap)
    if not keep:
        return None
    keep = torch.tensor(keep, dtype=torch.long)
    iou, yx_min, yx_max, prob, prob_cls, cls = (t[keep] for t in (iou, yx_min, yx_max, prob, prob_cls, cls))
    if fix:
        score = iou.unsqueeze(-1) * prob
        mask = score > threshold_cls
        nz = mask.nonzero()
        indices, cls = nz[:, 0], nz[:, 1]
        yx_min, yx_max = yx_min[indices], yx_max[indices]
        score = score[mask]
    else:
        score = iou
    return iou, yx_min, yx_max, cls, score


# ----------------------------------------------------------------------------------------------
# Region loss (model/__init__.py:59-107,138-167; train.py:57-62,347-349) -- restated, see header
# ----------------------------------------------------------------------------------------------

def norm_data(data, height, width, rows, cols):
    """train.py:57-62: GT pixel coordinates -> grid units."""
    scale = torch.tensor([rows / height, cols / width], dtype=torch.float32).view(1, 1, 2)
    out = dict(data)
    out['yx_min'] = data['yx_min'] * scale
    out['yx_max'] = data['yx_max'] * scale
    return out


def iou_match(yx_min, yx_max, data):
    """model/__init__.py:59-73: best GT per (cell, anchor); ties -> lowest GT index."""
    b, cells, a, _ = yx_min.shape
    m = batch_iou_matrix(yx_min.reshape(b, -1, 2), yx_max.reshape(b, -1, 2), data['yx_min'], data['yx_max'])
    m = m.view(b, cells, a, -1)
    iou, index = m.max(-1)
    flat = index.view(b, -1)
    g = {}
    for key in ('yx_min', 'yx_max', 'cls'):
        t = data[key]
        if t.dim() == 2:
            g[key] = torch.stack([d[i] for d, i in zip(t, flat)]).view(b, cells, a)
        else:
            g[key] = torch.stack([d[i] for d, i in zip(t, flat)]).view(b, cells, a, -1)
    return m, iou, index, g


def fit_positive(rows, cols, yx_min, yx_max, anchors):
    """model/__init__.py:76-95.  torch-0.3.1 semantics: `prod(yx_min < yx_max, -1)` is a byte MASK
    (restated as .all(-1)); duplicates collapse; padded (all-zero) GT slots are invalid."""
    b, num, _ = yx_min.shape
    a = anchors.size(0)
    valid = (yx_min < yx_max).all(-1)
    center = (yx_min + yx_max) / 2
    ij = torch.floor(center).long()
    index = ij[..., 0] * cols + ij[..., 1]
    anchors2 = anchors / 2
    m = iou_matrix((yx_min - center).view(-1, 2), (yx_max - center).view(-1, 2), -anchors2, anchors2).view(b, -1, a)
    _, index_anchor = m.max(-1)
    pos = torch.zeros(b, rows * cols, a, dtype=torch.bool)
    for bi in range(b):
        v = valid[bi]
        pos[bi, index[bi][v], index_anchor[bi][v]] = True
    return pos


def fill_norm(yx_min, yx_max, anchors):
    """model/__init__.py:98-103."""
    center = (yx_min + yx_max) / 2
    center_offset = center - torch.floor(center)
    size = yx_max - yx_min
    return center_offset, torch.log(size / anchors.view(1, -1, 2))


def loss(anchors, data, pred, threshold, cross_entropy=True):
    """model/__init__.py:138-167 with `train/cross_entropy=1` (config.ini:77) by default.

    0.3.1 semantics written out: broadcastable-mask indexing == masked_select with expand
    (:148,154,155,160,162); `~byte` is logical not (:145); size_average=False == sum; the CE term is
    a MEAN over positives (:162) and every term is then divided by cnt = B*cells*A (:164-166).
    `data` is already in grid units (train.py:347 applies norm_data first).
    Returns (dict of 5 scalars, debug dict).
    """
    iou = pred['iou']
    rows, cols = pred['feature'].shape[-2:]
    _, _iou, _, _data = iou_match(pred['yx_min'].detach(), pred['yx_max'].detach(), data)
    positive = fit_positive(rows, cols, data['yx_min'], data['yx_max'], anchors)
    negative = (~positive) & (_iou < threshold)
    _center_offset, _size_norm = fill_norm(_data['yx_min'], _data['yx_max'], anchors)
    pos2 = positive.unsqueeze(-1).expand_as(pred['center_offset'])
    out = {}
    out['foreground'] = ((iou[positive] - _iou[positive]) ** 2).sum()
    out['background'] = (iou[negative] ** 2).sum()
    out['center'] = ((pred['center_offset'][pos2] - _center_offset[pos2]) ** 2).sum()
    out['size'] = ((pred['size_norm'][pos2] - _size_norm[pos2]) ** 2).sum()
    if 'logits' in pred:
        logits = pred['logits']
        sel = logits[positive]  # [Npos, C]
        tgt = _data['cls'][positive].view(-1)
        if cross_entropy:
            out['cls'] = F.cross_entropy(sel, tgt)
        else:
            onehot = F.one_hot(tgt, logits.size(-1)).to(sel.dtype)
            out['cls'] = ((F.softmax(sel, -1) - onehot) ** 2).sum()
    cnt = float(np.multiply.reduce(positive.shape))
    for k in out:
        out[k] = out[k] / cnt
    return out, dict(iou=_iou, data=_data, positive=positive, negative=negative)


HPARAM_DEFAULT = dict(foreground=5.0, background=1.0, center=1.0, size=1.0, cls=1.0)  # config.ini:100-105


def loss_total(losses, hparam=HPARAM_DEFAULT):
    """train.py:348-349."""
    return sum(losses[k] * hparam[k] for k in losses)


# ----------------------------------------------------------------------------------------------
# Synthetic inputs (SURVEY section 8d)
# ----------------------------------------------------------------------------------------------

def synth_images(batch, height=416, width=416, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(batch, 3, height, width, generator=g)


def synth_feature(batch, size, seed, channels=125, cols=None):
    """Head feature map [B, channels, size, cols or size] the region-loss fixtures start from (tests/golden/make_golden_loss.py,
    make_golden_head.py), regenerated from its seed."""
    g = torch.Generator().manual_seed(100 + seed)
    return torch.randn(batch, channels, size, size if cols is None else cols, generator=g) * 1.5


def synth_anchors(num_anchors):
    """[A,2] (height, width) anchors: yolo-voc's five, or for any other count a ladder of distinct aspect ratios."""
    if num_anchors == 5:
        return anchors_yolo_voc()
    k = torch.arange(num_anchors, dtype=torch.float32)
    return torch.stack([1.0 + 1.75 * k, 0.75 + 1.25 * k + (k % 2) * 1.5], 1)


# Cases of tests/golden/head.npz (the head and tail executed by the reference off the square 20-class 5-anchor family):
# tag -> rows, cols, anchors, classes, batch, ground-truth slots, seed, one-hot class branch, empty images
# ('one': image 1 has only padding slots, 'all': no image has a ground-truth box).
HEAD_CASES = dict(
    wide=dict(rows=10, cols=19, a=5, c=20, batch=2, slots=12, seed=40),
    tall=dict(rows=19, cols=10, a=5, c=20, batch=2, slots=12, seed=41, one_hot=True),
    strip_h=dict(rows=1, cols=13, a=5, c=20, batch=2, slots=4, seed=42),
    strip_v=dict(rows=13, cols=1, a=5, c=20, batch=2, slots=4, seed=43),
    coco=dict(rows=13, cols=13, a=5, c=80, batch=1, slots=16, seed=44),
    c3a3=dict(rows=13, cols=17, a=3, c=3, batch=2, slots=8, seed=45),
    c1a9=dict(rows=11, cols=13, a=9, c=1, batch=2, slots=8, seed=46),
    nopos_one=dict(rows=13, cols=13, a=5, c=20, batch=3, slots=6, seed=47, empty='one'),
    nopos_all=dict(rows=13, cols=13, a=5, c=20, batch=2, slots=6, seed=48, empty='all'),
)


def head_case_inputs(tag):
    """(feature [B, A*(5+C), rows, cols], anchors [A,2], data in grid units) of one HEAD_CASES entry, from its seed."""
    k = HEAD_CASES[tag]
    rows, cols, a, c = k['rows'], k['cols'], k['a'], k['c']
    channels = a * (5 + c) if c > 1 else a * 5
    feature = synth_feature(k['batch'], rows, k['seed'], channels, cols)
    height, width = rows * 32, cols * 32
    tgt = synth_targets(k['batch'], height, width, slots=k['slots'], num_cls=c, seed=20 + k['seed'])
    empty = k.get('empty')
    if empty:
        for key in tgt:
            if empty == 'all':
                tgt[key].zero_()
            else:
                tgt[key][1].zero_()
    return feature, synth_anchors(a), norm_data(tgt, height, width, rows, cols)


def synth_detections(n, num_cls, seed, extent=13.0):
    """Post-filter input (iou [n], yx_min / yx_max [n,2], prob [n,C]) made with exactly rounded elementwise operations only, so
    that every machine regenerates it bit for bit: boxes jittered around 24 cluster centres (so NMS suppresses), objectness
    uniform, class scores a product of three uniforms (most are small, a few per box pass 0.005)."""
    g = torch.Generator().manual_seed(seed)
    centres = torch.rand(24, 2, generator=g) * extent
    c = centres[torch.randint(0, 24, (n,), generator=g)] + (torch.rand(n, 2, generator=g) - 0.5) * 1.5
    s = torch.rand(n, 2, generator=g) * (extent / 4) + 0.25
    iou = torch.rand(n, generator=g)
    if num_cls > 1:
        prob = torch.rand(n, num_cls, generator=g) * torch.rand(n, num_cls, generator=g) * torch.rand(n, num_cls, generator=g)
    else:
        prob = torch.ones(n, 1)
    return iou, c - s / 2, c + s / 2, prob


def synth_lattice_boxes(n, seed, extent=6):
    """NMS input on an integer lattice: corners and sizes are small integers, so coordinates repeat and many pairwise IoUs are
    exactly 1/2, 1/4 or 1 in fp32 -- the `iou <= overlap` boundary is hit when overlap is one of those.  Distinct scores."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.randint(0, extent, (n, 2), generator=g).float()
    size = torch.randint(1, 4, (n, 2), generator=g).float()
    score = (torch.randperm(n, generator=g).float() + 0.5) / n
    return score, lo, lo + size


# Fixture activations larger than SAMPLE_MIN_ELEMS are stored as a seeded sample of SAMPLE_FRACTION of their elements (name + '_sample'),
# next to their full max|.| and L2 norm, so that the fixtures stay small; sample_index() regenerates which elements were kept.
SAMPLE_MIN_ELEMS = 16384
SAMPLE_FRACTION = 4


def sample_index(numel, seed=0):
    """Sorted flat indices of the stored sample of a `numel`-element fixture tensor (numpy's legacy generator: stable across machines)."""
    return np.sort(np.random.RandomState(seed).choice(numel, numel // SAMPLE_FRACTION, replace=False))


def store_sampled(out, name, a):
    """Put array `a` into the fixture dict `out` under `name`, sampled when large (see SAMPLE_MIN_ELEMS)."""
    a = np.ascontiguousarray(a)
    if a.size <= SAMPLE_MIN_ELEMS:
        out[name] = a
        return
    out[name + '_sample'] = a.reshape(-1)[sample_index(a.size)]
    out[name + '_shape'] = np.array(a.shape)
    out[name + '_absmax'] = np.float64(np.abs(a).max())


def load_sampled(g, name):
    """(flat indices or None, reference values, max|.| of the full tensor) of a fixture stored by store_sampled()."""
    if name in g.files:
        a = g[name]
        return None, a, float(np.abs(a).max())
    shape = tuple(int(v) for v in g[name + '_shape'])
    return sample_index(int(np.prod(shape))), g[name + '_sample'], float(g[name + '_absmax'])


def has_sampled(g, name):
    return name in g.files or name + '_sample' in g.files


def synth_targets(batch, height=416, width=416, slots=16, num_cls=20, seed=2):
    """G=`slots` GT slots per image, 1..slots real boxes, rest zero rows (utils/data.py:38-41);
    boxes in PIXELS (y, x), centres chosen so floor(centre*S/H) < S."""
    g = torch.Generator().manual_seed(seed)
    yx_min = torch.zeros(batch, slots, 2)
    yx_max = torch.zeros(batch, slots, 2)
    cls = torch.zeros(batch, slots, dtype=torch.long)
    for b in range(batch):
        n = int(torch.randint(1, slots + 1, (1,), generator=g))
        hw = torch.rand(n, 2, generator=g) * (torch.tensor([height / 2 - 16.0, width / 2 - 16.0])) + 16.0
        lo = hw / 2
        hi = torch.tensor([float(height), float(width)]) - hw / 2
        c = lo + torch.rand(n, 2, generator=g) * (hi - lo)
        yx_min[b, :n] = c - hw / 2
        yx_max[b, :n] = c + hw / 2
        cls[b, :n] = torch.randint(0, num_cls, (n,), generator=g)
    return dict(yx_min=yx_min, yx_max=yx_max, cls=cls)


def synth_boxes(n, seed=3, extent=13.0):
    """NMS stress input: n random boxes with DISTINCT scores (a random permutation / n)."""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, 2, generator=g) * extent
    s = torch.rand(n, 2, generator=g) * (extent / 3) + 0.2
    score = (torch.randperm(n, generator=g).float() + 0.5) / n
    return score, c - s / 2, c + s / 2


# ----------------------------------------------------------------------------------------------
# MobileNet backbone (model/mobilenet.py:25-85), eval mode -- BASELINE configs[4]
# ----------------------------------------------------------------------------------------------
MOBILENET_UNITS = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1), (1024, 2), (1024, 1)]


def make_mobilenet_state_dict(seed=0, num_anchors=5, num_cls=20):
    """Deterministic synthetic MobileNet state_dict with the reference's key names (model/mobilenet.py:59-75)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def bn(prefix, c):
        sd[prefix + '.weight'] = torch.rand(c, generator=g) + 0.5
        sd[prefix + '.bias'] = torch.randn(c, generator=g) * 0.1
        sd[prefix + '.running_mean'] = torch.randn(c, generator=g) * 0.1
        sd[prefix + '.running_var'] = torch.rand(c, generator=g) + 0.5

    sd['layers.0.conv.weight'] = torch.randn(32, 3, 3, 3, generator=g) * math.sqrt(2.0 / 27)
    bn('layers.0.bn', 32)
    cin = 32
    for i, (cout, _) in enumerate(MOBILENET_UNITS, 1):
        sd['layers.%d.dw.conv.weight' % i] = torch.randn(cin, 1, 3, 3, generator=g) * math.sqrt(2.0 / 9)
        bn('layers.%d.dw.bn' % i, cin)
        sd['layers.%d.pw.conv.weight' % i] = torch.randn(cout, cin, 1, 1, generator=g) * math.sqrt(2.0 / cin)
        bn('layers.%d.pw.bn' % i, cout)
        cin = cout
    ch = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    sd['layers.14.weight'] = torch.randn(ch, cin, 1, 1, generator=g) * math.sqrt(1.0 / cin)
    sd['layers.14.bias'] = torch.randn(ch, generator=g) * 0.1
    return sd


def mobilenet_forward(sd, x, collect=None, train=False, stats=None):
    """model/mobilenet.py:84-85: conv_bn (:25-30) -> 13 x [conv_dw (:33-38), conv_pw (:41-46)] -> 1x1 head with bias; eval mode by default,
    `train=True` uses batch statistics (and records them in `stats`), as nn.BatchNorm2d does in train()."""
    def bn_relu(y, prefix):
        if train:
            if stats is not None:
                stats[prefix] = (y.mean(dim=(0, 2, 3)), y.var(dim=(0, 2, 3), unbiased=False))
            y = F.batch_norm(y, None, None, sd[prefix + '.weight'], sd[prefix + '.bias'], True, 0.0, 1e-5)
        else:
            y = F.batch_norm(y, sd[prefix + '.running_mean'], sd[prefix + '.running_var'], sd[prefix + '.weight'], sd[prefix + '.bias'], False, 0.0, 1e-5)
        return F.relu(y)

    x = bn_relu(F.conv2d(x, sd['layers.0.conv.weight'], None, 2, 1), 'layers.0.bn')
    if collect is not None:
        collect['layers.0'] = x
    for i, (_, stride) in enumerate(MOBILENET_UNITS, 1):
        c = x.size(1)
        x = bn_relu(F.conv2d(x, sd['layers.%d.dw.conv.weight' % i], None, stride, 1, groups=c), 'layers.%d.dw.bn' % i)
        x = bn_relu(F.conv2d(x, sd['layers.%d.pw.conv.weight' % i]), 'layers.%d.pw.bn' % i)
        if collect is not None:
            collect['layers.%d' % i] = x
    return F.conv2d(x, sd['layers.14.weight'], sd['layers.14.bias'])


# ----------------------------------------------------------------------------------------------
# ResNet plugin (model/resnet.py:28-178), eval mode -- SURVEY 8f rank 4
# ----------------------------------------------------------------------------------------------
RESNET_LAYERS = {'resnet18': ('basic', (2, 2, 2, 2)), 'resnet34': ('basic', (3, 4, 6, 3)), 'resnet50': ('bottleneck', (3, 4, 6, 3))}


def resnet_blocks(name='resnet18'):
    """(prefix, kind, cin, width, stride, downsample) per block in forward order (model/resnet.py:111-114,124-129)."""
    kind, counts = RESNET_LAYERS[name]
    expansion = 4 if kind == 'bottleneck' else 1
    out, cin = [], 64
    for li, (width, n) in enumerate(zip((64, 128, 256, 512), counts), 1):
        for bi in range(n):
            stride = 2 if (bi == 0 and li > 1) else 1
            cout = width * expansion
            out.append(dict(prefix='layer%d.%d' % (li, bi), kind=kind, cin=cin, width=width, cout=cout, stride=stride,
                            downsample=(stride > 1 or cin != cout)))
            cin = cout
    return out


def make_resnet_state_dict(name='resnet18', seed=0, num_anchors=5, num_cls=20):
    """Deterministic synthetic ResNet state_dict with the reference's (torchvision's) key names: kaiming-normal convs as
    model/resnet.py:117-119, BatchNorm tensors randomised so folding is exercised; the last BN of every block gets a small
    gamma so the residual sums stay O(1) through the stack."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def conv(key, cout, cin, k):
        sd[key + '.weight'] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cin * k * k))

    def bn(prefix, c, gain=1.0):
        sd[prefix + '.weight'] = (torch.rand(c, generator=g) + 0.5) * gain
        sd[prefix + '.bias'] = torch.randn(c, generator=g) * 0.1
        sd[prefix + '.running_mean'] = torch.randn(c, generator=g) * 0.1
        sd[prefix + '.running_var'] = torch.rand(c, generator=g) + 0.5

    conv('conv1', 64, 3, 7)
    bn('bn1', 64)
    cin = 64
    for b in resnet_blocks(name):
        p = b['prefix']
        if b['kind'] == 'basic':
            conv(p + '.conv1', b['width'], b['cin'], 3); bn(p + '.bn1', b['width'])
            conv(p + '.conv2', b['width'], b['width'], 3); bn(p + '.bn2', b['width'], 0.5)
        else:
            conv(p + '.conv1', b['width'], b['cin'], 1); bn(p + '.bn1', b['width'])
            conv(p + '.conv2', b['width'], b['width'], 3); bn(p + '.bn2', b['width'])
            conv(p + '.conv3', b['cout'], b['width'], 1); bn(p + '.bn3', b['cout'], 0.5)
        if b['downsample']:
            conv(p + '.downsample.0', b['cout'], b['cin'], 1); bn(p + '.downsample.1', b['cout'], 0.5)
        cin = b['cout']
    ch = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    sd['conv.weight'] = torch.randn(ch, cin, 1, 1, generator=g) * math.sqrt(1.0 / cin)
    sd['conv.bias'] = torch.randn(ch, generator=g) * 0.1
    return sd


def resnet_forward(sd, x, name='resnet18', collect=None):
    """model/resnet.py:131-142 (stem :107-110, BasicBlock.forward :44-61, Bottleneck.forward :82-103), eval mode."""
    def bn(y, prefix):
        return F.batch_norm(y, sd[prefix + '.running_mean'], sd[prefix + '.running_var'], sd[prefix + '.weight'], sd[prefix + '.bias'], False, 0.0, 1e-5)

    x = F.relu(bn(F.conv2d(x, sd['conv1.weight'], None, 2, 3), 'bn1'))
    if collect is not None:
        collect['stem'] = x
    x = F.max_pool2d(x, 3, 2, 1)
    if collect is not None:
        collect['maxpool'] = x
    for b in resnet_blocks(name):
        p = b['prefix']
        residual = x
        if b['kind'] == 'basic':
            out = F.relu(bn(F.conv2d(x, sd[p + '.conv1.weight'], None, b['stride'], 1), p + '.bn1'))
            out = bn(F.conv2d(out, sd[p + '.conv2.weight'], None, 1, 1), p + '.bn2')
        else:
            out = F.relu(bn(F.conv2d(x, sd[p + '.conv1.weight']), p + '.bn1'))
            out = F.relu(bn(F.conv2d(out, sd[p + '.conv2.weight'], None, b['stride'], 1), p + '.bn2'))
            out = bn(F.conv2d(out, sd[p + '.conv3.weight']), p + '.bn3')
        if b['downsample']:
            residual = bn(F.conv2d(x, sd[p + '.downsample.0.weight'], None, b['stride']), p + '.downsample.1')
        x = F.relu(out + residual)
        if collect is not None:
            collect[p] = x
    return F.conv2d(x, sd['conv.weight'], sd['conv.bias'])


# ----------------------------------------------------------------------------------------------
# Tiny YOLOv2 backbone (model/yolo2.py:140-173) -- SURVEY 8f rank 4
# ----------------------------------------------------------------------------------------------
FLOAT32_MIN = -3.4028234663852886e+38          # np.finfo(np.float32).min, the ConstantPad2d value (yolo2.py:150)


def tiny_layers(num_anchors=5, num_cls=20, channels=16):
    """Tiny's conv units in nn.Sequential order (yolo2.py:145-156): (index, cin, cout, k, bn, act, after) with
    after in {None, 'pool', 'pool_s1'}."""
    L, cin, idx = [], 3, 0
    for _ in range(5):
        L.append(dict(key='layers.%d' % idx, cin=cin, cout=channels, k=3, bn=True, act=True, after='pool'))
        cin, channels, idx = channels, channels * 2, idx + 2
    L.append(dict(key='layers.%d' % idx, cin=cin, cout=channels, k=3, bn=True, act=True, after='pool_s1'))
    cin, channels, idx = channels, channels * 2, idx + 3
    for _ in range(2):
        L.append(dict(key='layers.%d' % idx, cin=cin, cout=channels, k=3, bn=True, act=True, after=None))
        cin, idx = channels, idx + 1
    cout_head = num_anchors * (5 + num_cls) if num_cls > 1 else num_anchors * 5
    L.append(dict(key='layers.%d' % idx, cin=cin, cout=cout_head, k=1, bn=False, act=False, after=None))
    return L


def make_tiny_state_dict(seed=0, num_anchors=5, num_cls=20):
    """Deterministic synthetic Tiny state_dict: xavier-normal convs as `Tiny.init` (yolo2.py:159-165), randomised BN
    tensors so the folding is exercised, head bias ~ N(0, 0.1)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for l in tiny_layers(num_anchors, num_cls):
        fan_in, fan_out = l['cin'] * l['k'] ** 2, l['cout'] * l['k'] ** 2
        std = math.sqrt(2.0 / (fan_in + fan_out))
        sd[l['key'] + '.conv.weight'] = torch.randn(l['cout'], l['cin'], l['k'], l['k'], generator=g) * std * 2.0
        if l['bn']:
            c = l['cout']
            sd[l['key'] + '.bn.weight'] = torch.rand(c, generator=g) + 0.5
            sd[l['key'] + '.bn.bias'] = torch.randn(c, generator=g) * 0.1
            sd[l['key'] + '.bn.running_mean'] = torch.randn(c, generator=g) * 0.1
            sd[l['key'] + '.bn.running_var'] = torch.rand(c, generator=g) + 0.5
        else:
            sd[l['key'] + '.conv.bias'] = torch.randn(l['cout'], generator=g) * 0.1
    return sd


def tiny_forward(sd, x, num_anchors=5, num_cls=20, collect=None, train=False, stats=None):
    """model/yolo2.py:167-168 (`self.layers(x)`): conv units, MaxPool2d(2) x5, then ConstantPad2d((0,1,0,1), float32
    min) + MaxPool2d(2, stride=1) after the sixth conv.  `collect` receives every conv unit's (pre-pool) output."""
    for l in tiny_layers(num_anchors, num_cls):
        x = conv_unit(x, sd, l['key'], l['k'], l['bn'], l['act'], train, stats)
        if collect is not None:
            collect[l['key']] = x
        if l['after'] == 'pool':
            x = F.max_pool2d(x, 2)
        elif l['after'] == 'pool_s1':
            x = F.max_pool2d(F.pad(x, (0, 1, 0, 1), value=FLOAT32_MIN), 2, stride=1)
    return x


# ----------------------------------------------------------------------------------------------
# Evaluation matching + VOC AP (eval.py:57-121) -- SURVEY 8f rank 3
# ----------------------------------------------------------------------------------------------
def eval_matching(data_yx_min, data_yx_max, yx_min, yx_max, threshold):
    """eval.py:57-75: detections (descending score) vs the ground truth of the same class -> bool[N]."""
    n = yx_min.shape[0]
    tp = np.zeros([n], dtype=bool)
    if data_yx_min.numel() == 0 or n == 0:
        return tp
    m = iou_matrix(yx_min, yx_max, data_yx_min, data_yx_max)
    iou, index = torch.max(m, -1)
    detected = set()
    for i in range(n):
        if bool(iou[i] > threshold) and int(index[i]) not in detected:
            tp[i] = True
            detected.add(int(index[i]))
    return tp


def voc_ap(rec, prec, use_07_metric=False):
    """eval.py:78-108."""
    if use_07_metric:
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            p = 0 if np.sum(rec >= t) == 0 else np.max(prec[rec >= t])
            ap = ap + p / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    for i in range(mpre.size - 1, 0, -1):
        mpre[i - 1] = np.maximum(mpre[i - 1], mpre[i])
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def average_precision(tp, num, metric07=False):
    """eval.py:111-120."""
    tp = np.asarray(tp, dtype=bool)
    fp = np.cumsum(~tp)
    tp = np.cumsum(tp)
    rec = tp / num if num > 0 else np.zeros(len(tp))
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return voc_ap(rec, prec, metric07)


def synth_eval_case(seed, n_det=60, n_gt=12, num_cls=4, extent=13.0):
    """Detections (descending score) and ground truth of one image with many overlaps: jittered copies of the ground truth
    plus random boxes, so that matched / duplicate / unmatched detections all occur."""
    g = torch.Generator().manual_seed(seed)
    gt_min = torch.rand(n_gt, 2, generator=g) * (extent - 4)
    gt_max = gt_min + 1.0 + torch.rand(n_gt, 2, generator=g) * 3
    gt_cls = torch.randint(0, num_cls, (n_gt,), generator=g)
    src = torch.randint(0, n_gt, (n_det,), generator=g)
    jitter = (torch.rand(n_det, 2, generator=g) - 0.5) * 1.2
    det_min = gt_min[src] + jitter
    det_max = gt_max[src] + jitter * 0.5
    rnd = torch.rand(n_det, generator=g) < 0.3
    det_min[rnd] = torch.rand(int(rnd.sum()), 2, generator=g) * (extent - 3)
    det_max[rnd] = det_min[rnd] + 0.5 + torch.rand(int(rnd.sum()), 2, generator=g) * 3
    det_cls = torch.where(torch.rand(n_det, generator=g) < 0.8, gt_cls[src], torch.randint(0, num_cls, (n_det,), generator=g))
    score = torch.sort(torch.rand(n_det, generator=g), descending=True)[0]
    return dict(gt_min=gt_min, gt_max=gt_max, gt_cls=gt_cls, det_min=det_min, det_max=det_max, det_cls=det_cls, score=score)


# head.npz: post-filter, lattice-NMS and evaluation-matching cases (tests/golden/make_golden_head.py)
HEAD_POST_MODES = dict(wide=(1,), tall=(1,), coco=(1, 0), c3a3=(1, 0), c1a9=(0,))     # detect/fix values run per case
HEAD_NMS_CASES = dict(half=(300, 50, 0.5, 200), quarter=(300, 51, 0.25, 200), one=(120, 52, 1.0, 200), zero=(120, 53, 0.0, 200),
                 limit33=(400, 54, 0.5, 33))                                     # tag -> n, seed, overlap, limit (lattice boxes)
HEAD_EVAL_CASES = dict(c80=(60, 200, 40, 80, False), one_cls=(61, 120, 40, 80, True), dup=(62, 90, 24, 20, True))
#                                                      tag -> seed, detections, ground truth, classes, all of one class + duplicated boxes


def head_eval_case(tag):
    seed, n_det, n_gt, num_cls, crowd = HEAD_EVAL_CASES[tag]
    case = synth_eval_case(seed, n_det, n_gt, num_cls)
    if crowd:                                        # > 32 boxes of one class, every other one a copy of its neighbour
        case['gt_cls'] = torch.full_like(case['gt_cls'], 3)
        case['det_cls'] = torch.full_like(case['det_cls'], 3)
        case['gt_min'][1::2] = case['gt_min'][0::2]
        case['gt_max'][1::2] = case['gt_max'][0::2]
    return case, num_cls


# ----------------------------------------------------------------------------------------------
# Input pipeline: cv2.resize (8-bit INTER_LINEAR) + box scaling (transform/resize/label.py:25-31) -- SURVEY 8f rank 2
# ----------------------------------------------------------------------------------------------
def _resize_axis(n_dst, n_src):
    """OpenCV's linear-resize source index / fraction for one axis (imgproc resize.cpp): fx = float((d + 0.5) * scale - 0.5)."""
    d = np.arange(n_dst)
    f = ((d + 0.5) * (n_src / n_dst) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int32)
    return s, (f - s).astype(np.float32)


def resize_u8(src, height, width):
    """cv2.resize(src, (width, height)) for uint8 HWC images, restated from OpenCV's 8-bit fixed-point path: 11-bit
    coefficients rounded half-to-even; horizontally the fraction is dropped at the borders, vertically the rows are
    clamped but the fraction kept; column pass (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2."""
    h0, w0 = src.shape[:2]
    sx, fx = _resize_axis(width, w0)
    lo, hi = sx < 0, sx >= w0 - 1
    fx[lo] = 0; sx[lo] = 0
    fx[hi] = 0; sx[hi] = w0 - 1
    ax0 = np.rint((np.float32(1.0) - fx) * np.float32(2048)).astype(np.int32)
    ax1 = np.rint(fx * np.float32(2048)).astype(np.int32)
    sx1 = np.minimum(sx + 1, w0 - 1)
    sy, fy = _resize_axis(height, h0)
    ay0 = np.rint((np.float32(1.0) - fy) * np.float32(2048)).astype(np.int32)
    ay1 = np.rint(fy * np.float32(2048)).astype(np.int32)
    r0, r1 = np.clip(sy, 0, h0 - 1), np.clip(sy + 1, 0, h0 - 1)
    s = src.astype(np.int32)
    rows = s[:, sx, :] * ax0[None, :, None] + s[:, sx1, :] * ax1[None, :, None]
    out = (((ay0[:, None, None] * (rows[r0] >> 4)) >> 16) + ((ay1[:, None, None] * (rows[r1] >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def rescale_label(image, yx_min, yx_max, height, width):
    """transform/resize/label.py:25-31."""
    _height, _width = image.shape[:2]
    scale = np.array([height / _height, width / _width], np.float32)
    return resize_u8(image, height, width), yx_min * scale, yx_max * scale


def synth_frame(seed, h, w):
    """Deterministic uint8 BGR frame with smooth structure + noise (so interpolation is exercised at all phases)."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([127 + 120 * np.sin(yy / (5.0 + c) + xx / (9.0 - c)) for c in range(3)], -1)
    return np.clip(base + rng.randint(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)
