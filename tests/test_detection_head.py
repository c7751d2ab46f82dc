"""The detection head and tail -- anchor decode + class softmax, region loss, filter + NMS + per-class expansion, IoU matrices,
evaluation matching -- away from the square 20-class 5-anchor family: rows != cols, other class and anchor counts, the capacity
limits and the degenerate inputs, against the executed reference (tests/golden/head.npz) and against the oracle
(oracle/yolo2_oracle.py) evaluated in float64 on the same fp32 inputs.

Comparison rules (helpers below):
  * real-valued outputs, element by element: |got - ref| <= atol + rtol * |ref| with per-quantity constants derived next to each use
    (`assert_close`); never max|d| / max|ref|, which hides every element much smaller than the largest.  The worst distance in fp32
    ulps of the reference is recorded per quantity (`record`, written to $YB_PARITY_OUT/head_measured.json when that is set);
  * decisions (masks, index lists, classes, true-positive flags) exactly against the fp32 oracle (`assert_same`); where a decision
    hangs on a transcendental, elements whose float64 margin is below a stated epsilon are excluded and counted, and more than
    MAX_EXCLUDED of them fail the test;
  * data moves bit for bit.

The unmarked tests run without a GPU: the oracle reproduces every case of head.npz, and the helpers reject deliberately wrong
restatements on the very inputs the GPU tests use (so those inputs are known to separate right from wrong).
"""
import configparser
import json
import os

import numpy as np
import pytest
import torch

from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu
ULP = 2.0 ** -23            # fp32 spacing at 1
TINY = 1e-37                # absolute slack in the fp32 denormal range, where relative accuracy is lost by construction
MAX_EXCLUDED = 4
MEASURED = {}


def make_config(fix, metric07=0):
    config = configparser.ConfigParser()
    config.read_dict({'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': str(int(fix)), 'overlap': '0.45'},
                      'eval': {'metric07': str(metric07)}})
    return config


def record(name, value):
    """Keep the worst measured figure per quantity; mirror them to $YB_PARITY_OUT/head_measured.json."""
    MEASURED[name] = max(float(value), MEASURED.get(name, 0.0))
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'head_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def _np64(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def assert_close(name, got, ref, rtol, atol=0.0):
    """Element-wise |got - ref| <= atol + rtol * |ref| (atol may be an array).  `ref` is float64; where it overflows fp32 the result
    must be the same infinity, and a NaN is accepted only where the reference is NaN too."""
    got, ref = _np64(got), _np64(ref)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    with np.errstate(over='ignore', invalid='ignore'):
        ref32 = ref.astype(np.float32).astype(np.float64)
        same = (got == ref32) | (np.isnan(got) & np.isnan(ref))
        err = np.abs(got - ref)
        ok = same | (err <= atol + rtol * np.abs(ref))
        finite = np.isfinite(got) & np.isfinite(ref32) & ~same
        if finite.any():
            record(name + ' [ulp]', (err[finite] / np.spacing(np.abs(ref32[finite]).astype(np.float32)).astype(np.float64)).max())
    if not ok.all():
        i = np.unravel_index(np.argmax(~ok), ok.shape)
        raise AssertionError('%s: %d of %d elements differ, first at %s: got %r, reference %r' % (name, (~ok).sum(), ok.size, i, got[i], ref[i]))


def assert_same(name, got, ref, margin=None, eps=0.0):
    """Exact equality of decisions; elements with |margin| < eps (float64 distance from the deciding threshold) are left out."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    diff = got != ref
    if margin is not None:
        near = np.abs(_np64(margin)) < eps
        excluded = int((diff & near).sum())
        record(name + ' [excluded]', excluded)
        assert excluded <= MAX_EXCLUDED, '%s: %d elements within %g of the threshold differ' % (name, excluded, eps)
        diff = diff & ~near
    if diff.any():
        i = np.unravel_index(np.argmax(diff), diff.shape)
        raise AssertionError('%s: %d of %d decisions differ, first at %s: got %r, reference %r' % (name, diff.sum(), diff.size, i, got[i], ref[i]))


def channels(a, c):
    return a * (5 + c) if c > 1 else a * 5


# ------------------------------------------------------------------------------------------------------------------------------------
# decode
# ------------------------------------------------------------------------------------------------------------------------------------
GRIDS = [(13, 13), (10, 19), (19, 10), (1, 33), (33, 1), (7, 5)]
HEADS = [(5, 20), (5, 80), (3, 3), (9, 1), (1, 2), (5, 36)]
SATURATING = (30.0, -30.0, 88.0, -88.0)


def decode_input(batch, rows, cols, a, c, seed):
    """Feature map ~ N(0, 2) whose first cells carry a band of saturating values: +-30 / +-88 in the sigmoid and exp channels (fp32
    exp(88) * anchor overflows for the larger anchors, exp(-88) is a denormal) and class logits spread by 60."""
    per = 5 + c if c > 1 else 5
    f = torch.randn(batch, a * per, rows, cols, generator=torch.Generator().manual_seed(seed)) * 2
    flat = f.view(batch, a, per, rows * cols)
    for cell in range(min(rows * cols, 8)):
        for k in range(a):
            flat[0, k, (cell + k) % 5, cell] = SATURATING[cell % 4]
        if c > 1:
            flat[0, :, 5:, cell] = (torch.arange(c) % 3).float() * 60 * (1 if cell % 2 else -1)
    return f


def decode_parts64(feature, anchors):
    """The oracle's decode in float64, with |centre| + |half size| per box coordinate (the scale of the rounding error of yx_*)."""
    ref = O.decode(feature.double(), anchors.double())
    ref['prob'] = O.class_prob(ref)
    half = (ref['yx_max'] - ref['yx_min']) / 2
    ref['yx_scale'] = ((ref['yx_max'] + ref['yx_min']) / 2).abs() + half.abs()
    return ref


def check_decode(got, feature, anchors, c, tag=''):
    """Decode outputs against float64.
    iou, center_offset: 1 / (1 + expf(-v)) -- expf is within 2 ulp, the add and the divide round once each: 4 ulp, plus TINY.
    yx_min / yx_max: (cell + sigmoid) -+ expf(n) * anchor / 2 -- every term is within 4 ulp of ITS OWN magnitude, so the error is
        bounded by 4 ulp of |centre| + |half size|, not of the (possibly cancelled) result.
    prob: expf(v - max) / sum -- 2 ulp per expf, the fp32 sum of C positive terms within (C - 1) / 2 ulp, one divide: (C + 7) / 2 ulp;
        on top of that the fp32 difference v - max is rounded to an ulp of ITS magnitude, an absolute error that exp turns into a
        relative one: (max - v) ulp more for the classes far below the maximum.
    logits, size_norm: copies, bit for bit."""
    ref = decode_parts64(feature, anchors)
    b, cells, a = ref['iou'].shape
    assert_close(tag + 'decode iou', got['iou'], ref['iou'], 4 * ULP, TINY)
    assert_close(tag + 'decode center_offset', got['center_offset'], ref['center_offset'], 4 * ULP, TINY)
    with np.errstate(invalid='ignore'):
        scale = np.nan_to_num(_np64(ref['yx_scale']), nan=0.0, posinf=0.0)
    ref32 = O.decode(feature, anchors)
    for k in ('yx_min', 'yx_max'):
        # exp(n) * anchor overflows fp32 before it is halved, so the fp32 formula gives an infinity up to a factor 2 below the
        # float64 value's own overflow: an infinity is right exactly where the fp32 oracle has one, and is compared with it
        over = torch.isinf(ref32[k])
        x = torch.as_tensor(got[k]).cpu()
        assert torch.equal(torch.isinf(x), over) and torch.equal(x[over], ref32[k][over]), k + ': infinities differ from the fp32 oracle'
        assert_close(tag + 'decode ' + k, x.masked_fill(over, 0), ref[k].masked_fill(over, 0), 0.0, 4 * ULP * scale + TINY)
    moved = feature.permute(0, 2, 3, 1).reshape(b, cells, a, -1)
    assert torch.equal(torch.as_tensor(got['size_norm']).cpu(), moved[..., 3:5]), 'size_norm is a copy'
    if c > 1:
        assert torch.equal(torch.as_tensor(got['logits']).cpu(), moved[..., 5:]), 'logits is a copy'
    if 'prob' in got:
        below = (ref['logits'].max(-1, keepdim=True)[0] - ref['logits']) if c > 1 else torch.zeros_like(ref['prob'])
        assert_close(tag + 'decode prob', got['prob'], ref['prob'], (c + 7) / 2 * ULP, TINY + _np64(ref['prob'] * below) * ULP)


def oracle32_decode(feature, anchors):
    out = O.decode(feature, anchors)
    out['prob'] = O.class_prob(out)
    return out


# ------------------------------------------------------------------------------------------------------------------------------------
# region loss
# ------------------------------------------------------------------------------------------------------------------------------------
TERMS = ('foreground', 'background', 'center', 'size', 'cls')
WEIGHTS = dict(foreground=5.0, background=0.75, center=1.5, size=2.5, cls=0.5)      # five distinct values
GROUPS = dict(objectness=(0, 1), center=(1, 3), size=(3, 5), cls=(5, None))


def loss_input(batch, rows, cols, a, c, slots, seed):
    f = torch.randn(batch, channels(a, c), rows, cols, generator=torch.Generator().manual_seed(seed)) * 1.2
    tgt = O.synth_targets(batch, rows * 32, cols * 32, slots=slots, num_cls=c, seed=seed + 5)
    return f, O.synth_anchors(a), O.norm_data(tgt, rows * 32, cols * 32, rows, cols)


def loss_reference(feature, anchors, data, threshold, cross_entropy, weights):
    """(fp32 oracle debug dict, float64 oracle: losses, debug, d(sum_k w_k loss_k)/dfeature, top-2 IoU gap of every box).  The class
    term is left out when the batch has no positive (the reference's mean over zero rows is NaN, DESIGN.md)."""
    _, dbg32 = O.loss(anchors, data, O.decode(feature, anchors), threshold, cross_entropy)
    f64 = feature.double().requires_grad_(True)
    a64 = anchors.double()
    d64 = dict(yx_min=data['yx_min'].double(), yx_max=data['yx_max'].double(), cls=data['cls'])
    pred = O.decode(f64, a64)
    if not bool(dbg32['positive'].any()):
        pred.pop('logits', None)
    l64, dbg64 = O.loss(a64, d64, pred, threshold, cross_entropy)
    sum(l64[k] * weights[k] for k in l64).backward()
    m = O.iou_match(pred['yx_min'].detach(), pred['yx_max'].detach(), d64)[0]
    top = torch.topk(m, min(2, m.size(-1)), -1)[0]
    gap = (top[..., 0] - top[..., -1]) if m.size(-1) > 1 else torch.ones_like(top[..., 0])
    return dbg32, l64, dbg64, f64.grad, gap


def check_loss(got, feature, anchors, data, threshold, cross_entropy, weights, tag=''):
    """`got`: dict(losses [5], positive, negative, best_iou, dfeature) of the implementation under test.

    positive depends on the ground truth alone (no transcendental): exact.  negative = !positive & best_iou < threshold hangs on the
    decoded box: elements within 1e-5 of the threshold are excluded.  A positive whose two best ground-truth IoUs are closer than
    1e-5 (and not exactly tied: ties go to the lowest slot everywhere) has an ambiguous regression target: its gradient is excluded,
    and the scalars are compared only when there is no such box (with 128 slots a case or two of the sweep has one).
    best_iou: the decoded corners are within 4 ulp of |centre| + |half size| (< 1e-4 cell at these sizes); an IoU moves by at most
        (overlap height + width) * that / union: atol 2e-6, rtol 1e-5.
    the five scalars: fp32 sums of up to 2e4 non-negative terms, rtol 2e-5.
    gradient, in units of w / cnt: objectness 2 (s - iou) s (1 - s) inherits best_iou's error (4e-6); centre 2 (s - t) s (1 - s) and
        size 2 (n - log(size / anchor)) a few ulp of O(1) operands (2e-6); class (softmax - onehot) / npos the softmax's (C + 7) / 2 ulp
        (1e-5 at C = 80); rtol 2e-5 throughout."""
    dbg32, l64, dbg64, grad64, gap = loss_reference(feature, anchors, data, threshold, cross_entropy, weights)
    b, ch, rows, cols = feature.shape
    a = anchors.size(0)
    per = ch // a
    pos32 = dbg32['positive'].numpy()
    assert np.array_equal(pos32, dbg64['positive'].numpy()), 'input: fp32 and float64 disagree on a positive'
    ambiguous = (dbg64['positive'] & (gap > 0) & (gap < 1e-5)).numpy()
    record(tag + 'loss matched slot [excluded]', ambiguous.sum())
    assert ambiguous.sum() <= MAX_EXCLUDED, 'input: %d positives whose two best ground truths are within 1e-5 in IoU' % ambiguous.sum()
    assert_same(tag + 'loss positive', np.asarray(got['positive']).astype(bool), pos32)
    margin = dbg64['iou'] - threshold
    assert_same(tag + 'loss negative', np.asarray(got['negative']).astype(bool), dbg32['negative'].numpy(), margin, 1e-5)
    assert_close(tag + 'loss best_iou', got['best_iou'], dbg64['iou'], 1e-5, 2e-6)
    near = np.abs(_np64(margin)) < 1e-5
    flipped = (np.asarray(got['negative']).astype(bool) != dbg32['negative'].numpy()) & near
    for i, k in enumerate(TERMS):
        if k in l64 and not (flipped.any() if k == 'background' else ambiguous.any()):
            assert_close(tag + 'loss ' + k, np.asarray(got['losses'])[i], l64[k].item(), 2e-5, 1e-12)
        elif k not in l64:
            assert k == 'cls' and float(np.asarray(got['losses'])[i]) == 0.0, 'class term without logits or without a positive is 0'
    cnt = float(b * rows * cols * a)
    g_got = _np64(got['dfeature']).reshape(b, a, per, rows * cols)
    g_ref = _np64(grad64).reshape(b, a, per, rows * cols)
    npos = max(int(pos32.sum()), 1)
    near, skip = (m.reshape(b, rows * cols, a).transpose(0, 2, 1)[:, :, None] for m in (near, ambiguous))      # -> [B, A, 1, cells]
    units = dict(objectness=4e-6 * max(weights['foreground'], weights['background']), center=2e-6 * weights['center'],
                 size=2e-6 * weights['size'], cls=1e-5 * weights['cls'] / npos)
    for name, (lo, hi) in GROUPS.items():
        if lo >= per:
            continue
        x, r = g_got[:, :, lo:hi], g_ref[:, :, lo:hi]
        drop = (near | skip) if name == 'objectness' else skip
        x, r = np.where(drop, 0.0, x), np.where(drop, 0.0, r)
        if name == 'cls' and not pos32.any():
            r = np.zeros_like(r)
        assert_close(tag + 'loss grad ' + name, x, r, 2e-5, units[name] / cnt)


def oracle32_loss(feature, anchors, data, threshold, cross_entropy, weights):
    """The fp32 oracle in the shape check_loss takes (the stand-in for the kernels in the tests that run without a GPU)."""
    f = feature.clone().requires_grad_(True)
    pred = O.decode(f, anchors)
    losses, dbg = O.loss(anchors, data, pred, threshold, cross_entropy)
    sum(losses[k] * weights[k] for k in losses).backward()
    return dict(losses=np.array([losses[k].item() if k in losses else 0.0 for k in TERMS]), positive=dbg['positive'].numpy(),
                negative=dbg['negative'].numpy(), best_iou=dbg['iou'], dfeature=f.grad)


def gpu_loss(ops, feature, anchors, data, threshold, cross_entropy, weights):
    out = ops.region_loss_forward(feature.to(DEV), anchors.to(DEV), data['yx_min'].to(DEV), data['yx_max'].to(DEV), data['cls'].to(DEV),
                                  threshold, cross_entropy)
    w = torch.tensor([weights[k] for k in TERMS], dtype=torch.float32, device=DEV)
    df = ops.region_loss_backward(out['grad_terms'], out['grad_bg'], w, anchors.size(0))
    return dict(losses=out['losses'].cpu().numpy(), positive=out['positive'].cpu().numpy(), negative=out['negative'].cpu().numpy(),
                best_iou=out['best_iou'].cpu(), dfeature=df.cpu(), pos_count=out['pos_count'].cpu().numpy())


def edge_targets(rows, cols, c):
    """[3, 8] ground truth in grid units on a rows x cols grid: image 0 -- centres exactly on cell edges, in the last row and the last
    column, in the first cell; image 1 -- padding only; image 2 -- three boxes on one (cell, anchor), two of them identical with
    different classes, and class ids outside [0, C) (which the kernels clamp into range)."""
    lo, hi, cls = torch.zeros(3, 8, 2), torch.zeros(3, 8, 2), torch.zeros(3, 8, dtype=torch.long)

    def put(b, g, cy, cx, h, w, k):
        lo[b, g] = torch.tensor([cy - h / 2, cx - w / 2]); hi[b, g] = torch.tensor([cy + h / 2, cx + w / 2]); cls[b, g] = k

    put(0, 0, 2.0, 3.0, 1.0, 1.0, 1 % c)                       # centre on the corner of four cells: floor -> cell (2, 3), offset 0
    put(0, 1, rows - 0.5, 1.5, 0.5, 3.0, 2 % c)                # last row
    put(0, 2, 0.5, cols - 0.5, 3.0, 0.5, 3 % c)                # last column
    put(0, 3, rows - 0.25, cols - 0.25, 0.5, 0.5, 4 % c)       # last cell, box reaching outside the grid
    put(0, 4, 0.25, 0.25, 4.0, 9.0, 5 % c)                     # first cell
    put(2, 0, 3.5, 2.5, 1.5, 1.25, 0)
    put(2, 1, 3.5, 2.5, 1.5, 1.25, c - 1)                      # identical box, other class: the tie goes to slot 0
    put(2, 2, 3.25, 2.75, 1.75, 1.5, 1 % c)                    # same cell, same anchor, different box
    put(2, 5, 1.5, 1.5, 2.0, 2.0, c + 3)                       # class id above the range
    put(2, 7, 5.5, 3.5, 2.0, 5.0, -1)                          # class id below the range
    return dict(yx_min=lo, yx_max=hi, cls=cls)


def clamp_cls(data, c):
    return dict(data, cls=data['cls'].clamp(0, max(c - 1, 0)))


# ------------------------------------------------------------------------------------------------------------------------------------
# filter + NMS + expansion
# ------------------------------------------------------------------------------------------------------------------------------------
THRESHOLD, THRESHOLD_CLS = 0.25, 1.0 / 64       # exactly representable, and reached exactly by the quantised scores below


def nms_input(n, c, seed, kind):
    """`smooth`: synth_detections (distinct scores, clustered boxes).  `lattice`: scores k / 64 (repeated, and equal to THRESHOLD at
    k = 16), corners on a half-integer lattice (repeated boxes; IoUs of exactly 0, 1/4, 1/2, 1), every eleventh box of zero area, class
    scores j / 16 (tied maxima in most rows; score * prob == THRESHOLD_CLS exactly for k * j == 16)."""
    if kind == 'smooth':
        return O.synth_detections(n, c, seed)
    g = torch.Generator().manual_seed(seed)
    score = torch.randint(0, 65, (n,), generator=g).float() / 64
    lo = torch.randint(0, 8, (n, 2), generator=g).float() / 2
    size = torch.randint(1, 5, (n, 2), generator=g).float() / 2
    size[::11] = 0
    prob = torch.randint(0, 17, (n, c), generator=g).float() / 16 if c > 1 else torch.ones(n, 1)
    return score, lo, lo + size, prob


def oracle_filter_nms(score, yx_min, yx_max, prob, mode, overlap, limit):
    """One image through O.filter_visible, O.nms and the expansion of O.postprocess (detect.py:72-77), keeping every index list."""
    n = score.numel()
    if mode == 2:
        mask = torch.ones(n, dtype=torch.bool)
    else:
        mask = O.filter_visible(score, yx_min, yx_max, prob, mode == 1, THRESHOLD, THRESHOLD_CLS)[6]
    filt = mask.nonzero().view(-1)
    keep = O.nms(score[filt].numpy(), yx_min[filt].numpy(), yx_max[filt].numpy(), overlap, limit)
    out = dict(n_filtered=filt.numel(), filt_box=filt.numpy(), keep_idx=np.array(keep, dtype=np.int64), keep_box=filt.numpy()[keep])
    if prob is not None:
        out['best_prob'], out['best_cls'] = (t.numpy() for t in torch.max(prob, -1))
    if mode == 1:
        s = score[filt][keep].unsqueeze(-1) * prob[filt][keep]
        nz = (s > THRESHOLD_CLS).nonzero()
        out['det_keep'], out['det_cls'], out['det_score'] = nz[:, 0].numpy(), nz[:, 1].numpy(), s[s > THRESHOLD_CLS].numpy()
    return out


def check_filter_nms(got, bi, ref, limit, tag=''):
    """Everything here is a decision or a copy on identical fp32 inputs (score * prob is one correctly rounded product on both
    sides): exact, nothing excluded."""
    nf, nk = int(got['n_filtered'][bi]), int(got['n_keep'][bi])
    assert nf == ref['n_filtered'], (tag, 'n_filtered', nf, ref['n_filtered'])
    assert_same(tag + 'keep_idx', got['keep_idx'][bi, :nk], ref['keep_idx'])
    assert_same(tag + 'keep_box', got['keep_box'][bi, :nk], ref['keep_box'])
    assert nk <= limit
    if 'filt_box' in got:
        assert_same(tag + 'filt_box', got['filt_box'][bi, :nf], ref['filt_box'])
    if 'best_cls' in got:
        assert_same(tag + 'best_cls', got['best_cls'][bi], ref['best_cls'])
        assert_same(tag + 'best_prob', got['best_prob'][bi], ref['best_prob'])
    if 'n_det' in got:
        nd = int(got['n_det'][bi])
        if 'det_keep' in ref:
            for k in ('det_keep', 'det_cls', 'det_score'):
                assert_same(tag + k, got[k][bi, :nd], ref[k])
        else:
            assert nd == 0


def gpu_filter_nms(ops, score, yx_min, yx_max, prob, mode, overlap, limit, expand=True, details=True):
    res = ops.filter_nms(score.to(DEV), yx_min.to(DEV), yx_max.to(DEV), None if prob is None else prob.to(DEV), mode, THRESHOLD,
                         THRESHOLD_CLS, overlap, limit, expand=expand, details=details)
    return {k: v.cpu().numpy() for k, v in res.items()}


# ------------------------------------------------------------------------------------------------------------------------------------
# evaluation matching
# ------------------------------------------------------------------------------------------------------------------------------------
def oracle_tp(case, num_cls, threshold):
    tp = np.zeros(case['det_cls'].numel(), dtype=bool)
    for c in range(num_cls):
        dm, gm = case['det_cls'] == c, case['gt_cls'] == c
        if bool(dm.any()):
            tp[dm.numpy()] = O.eval_matching(case['gt_min'][gm], case['gt_max'][gm], case['det_min'][dm], case['det_max'][dm], threshold)
    return tp


def eval_image(seed, n_det, n_gt, num_cls, crowd=False):
    """One image: n_gt == 0 / n_det == 0 give empty arrays; `crowd` puts every box in class 1, duplicates every other ground-truth box
    and lets all detections compete for them."""
    case = O.synth_eval_case(seed, max(n_det, 1), max(n_gt, 1), num_cls)
    if n_gt == 0:
        for k in ('gt_min', 'gt_max', 'gt_cls'):
            case[k] = case[k][:0]
    if n_det == 0:
        for k in ('det_min', 'det_max', 'det_cls', 'score'):
            case[k] = case[k][:0]
    if crowd:
        case['gt_cls'] = torch.full_like(case['gt_cls'], min(1, num_cls - 1))
        case['det_cls'] = torch.full_like(case['det_cls'], min(1, num_cls - 1))
        case['gt_min'][1::2] = case['gt_min'][0:case['gt_min'].size(0) - 1:2]
        case['gt_max'][1::2] = case['gt_max'][0:case['gt_max'].size(0) - 1:2]
    return case


def eval_batch(num_cls):
    """Ragged batch: 0, 1, 40 (> 32 of one class, duplicated) and 1024 ground-truth boxes, images without detections and without ground
    truth in the middle."""
    spec = [(30, 5, False), (0, 7, False), (25, 0, False), (300, 40, True), (9, 1, False), (0, 0, False), (200, 1024, False), (64, 40, False)]
    return [eval_image(900 + 10 * num_cls + i, d, g, num_cls, crowd) for i, (d, g, crowd) in enumerate(spec)]


# ====================================================================================================================================
# without a GPU: the oracle reproduces head.npz, and the helpers reject wrong restatements
# ====================================================================================================================================
@pytest.fixture(scope='module')
def head(golden_dir):
    return np.load(os.path.join(golden_dir, 'head.npz'))


def _sampled(g, name, full):
    idx, ref, _ = O.load_sampled(g, name)
    full = _np64(full)
    return (full.reshape(-1)[idx] if idx is not None else full), ref


def check_against_head_npz(head, tag, dec, loss, exact_masks):
    """Decode outputs and loss results of one HEAD_CASES entry against what the reference returned.  Both sides are fp32 evaluations
    of the same formula by different exp / sigmoid implementations, so the element-wise tolerances are those of check_decode /
    check_loss doubled (each side is within them of the exact value)."""
    k = O.HEAD_CASES[tag]
    for name in ('iou', 'center_offset', 'prob'):
        got, ref = _sampled(head, '%s_dec_%s' % (tag, name), dec[name])
        assert_close('%s vs reference: %s' % (tag, name), got, ref, (8 if name != 'prob' else k['c'] + 7 + 16) * ULP, TINY)      # logits ~ N(0, 1.5): max - v < 16
    for name in ('yx_min', 'yx_max'):
        got, ref = _sampled(head, '%s_dec_%s' % (tag, name), dec[name])
        scale, _ = _sampled(head, '%s_dec_%s' % (tag, name), dec['yx_scale'])
        assert_close('%s vs reference: %s' % (tag, name), got, ref, 0.0, 8 * ULP * scale)
    n = k['batch'] * k['rows'] * k['cols'] * k['a']
    iou_got, iou_ref = _sampled(head, tag + '_iou', loss['best_iou'])
    assert_close(tag + ' vs reference: best_iou', iou_got, iou_ref, 2e-5, 4e-6)
    full_iou = _np64(loss['best_iou']).reshape(-1)
    for name in ('positive', 'negative'):
        ref = np.unpackbits(head['%s_%s' % (tag, name)])[:n].astype(bool)
        got = np.asarray(loss[name]).astype(bool).reshape(-1)
        if name == 'positive' or exact_masks:
            assert_same('%s vs reference: %s' % (tag, name), got, ref)
        else:
            assert_same('%s vs reference: %s' % (tag, name), got, ref, full_iou - 0.6, 1e-5)
    for i, name in enumerate(TERMS):
        key = '%s_loss_%s' % (tag, name)
        if key not in head.files:
            assert name == 'cls' and k['c'] == 1
        elif np.isnan(head[key]):
            assert tag == 'nopos_all' and name == 'cls' and float(np.asarray(loss['losses'])[i]) == 0.0     # DESIGN.md: 0 where the reference has NaN
        else:
            assert_close('%s vs reference: %s' % (tag, name), np.asarray(loss['losses'])[i], float(head[key]), 4e-5, 1e-12)
    got, ref = _sampled(head, tag + '_grad', loss['dfeature'])
    cnt = float(n)
    finite = np.isfinite(ref)
    assert finite.all() or tag == 'nopos_all'
    assert_close(tag + ' vs reference: gradient', got[finite], ref[finite], 4e-5, 5.0 * 8e-6 / cnt)
    if not finite.all():
        assert (got[~finite] == 0).all()


def head_case_results(tag, decode_fn, loss_fn):
    k = O.HEAD_CASES[tag]
    feature, anchors, data = O.head_case_inputs(tag)
    dec = dict(decode_fn(feature, anchors, k['c']))
    dec['yx_scale'] = decode_parts64(feature, anchors)['yx_scale']
    return dec, loss_fn(feature, anchors, data, 0.6, not k.get('one_hot'), O.HPARAM_DEFAULT)


def _oracle32_loss_safe(feature, anchors, data, threshold, cross_entropy, weights):
    """oracle32_loss with the class term dropped when nothing is positive (NaN in the reference; the kernels give 0)."""
    if not bool(O.fit_positive(feature.size(2), feature.size(3), data['yx_min'], data['yx_max'], anchors).any()):
        f = feature.clone().requires_grad_(True)
        pred = O.decode(f, anchors)
        pred.pop('logits', None)
        losses, dbg = O.loss(anchors, data, pred, threshold, cross_entropy)
        sum(losses[k] * weights[k] for k in losses).backward()
        return dict(losses=np.array([losses[k].item() if k in losses else 0.0 for k in TERMS]), positive=dbg['positive'].numpy(),
                    negative=dbg['negative'].numpy(), best_iou=dbg['iou'], dfeature=f.grad)
    return oracle32_loss(feature, anchors, data, threshold, cross_entropy, weights)


@pytest.mark.parametrize('tag', list(O.HEAD_CASES))
def test_oracle_decode_and_loss_reproduce_executed_reference(head, tag):
    dec, loss = head_case_results(tag, lambda f, a, c: oracle32_decode(f, a), _oracle32_loss_safe)
    check_against_head_npz(head, tag, dec, loss, exact_masks=False)


def post_case(head, tag, fix):
    k = O.HEAD_CASES[tag]
    inputs = O.synth_detections(k['rows'] * k['cols'] * k['a'], k['c'], 300 + k['seed'])
    pre = '%s_fix%d_' % (tag, fix)
    return inputs, {name[len(pre):]: head[name] for name in head.files if name.startswith(pre)}


def check_post_case(ref, inputs, fv, res):
    """filter_visible / postprocess results (reference-shaped tuples) against the stored index lists: gathers of the inputs are bit
    exact, classes exact, score = iou * prob one rounded product: exact."""
    iou, yx_min, yx_max, prob = (t.cpu() for t in inputs)
    box = torch.from_numpy(ref['fv_box'].astype(np.int64))
    for got, want in zip(fv, (iou[box], yx_min[box], yx_max[box], prob[box], torch.from_numpy(ref['fv_prob_cls']), torch.from_numpy(ref['fv_cls']).long())):
        assert torch.equal(got.cpu(), want)
    keep, det = torch.from_numpy(ref['keep_box'].astype(np.int64)), torch.from_numpy(ref['det_box'].astype(np.int64))
    assert np.array_equal(iou[keep].numpy(), ref['iou'])
    for got, want in zip(res, (iou[keep], yx_min[det], yx_max[det], torch.from_numpy(ref['cls']).long(), torch.from_numpy(ref['score']))):
        assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize('tag,fix', [(t, f) for t, modes in O.HEAD_POST_MODES.items() for f in modes])
def test_oracle_postprocess_reproduces_executed_reference(head, tag, fix):
    inputs, ref = post_case(head, tag, fix)
    fv = O.filter_visible(*inputs, bool(fix), 0.3, 0.005)[:6]
    res = O.postprocess(*inputs, bool(fix), 0.3, 0.005, 0.45)
    check_post_case(ref, inputs, fv, res)


@pytest.mark.parametrize('tag', list(O.HEAD_NMS_CASES))
def test_oracle_nms_reproduces_executed_reference(head, tag):
    n, seed, overlap, limit = O.HEAD_NMS_CASES[tag]
    score, a, b = O.synth_lattice_boxes(n, seed)
    assert O.nms(score.numpy(), a.numpy(), b.numpy(), overlap, limit) == head['nms_%s_keep' % tag].tolist()


@pytest.mark.parametrize('tag', list(O.HEAD_EVAL_CASES))
def test_oracle_eval_matching_reproduces_executed_reference(head, tag):
    case, num_cls = O.head_eval_case(tag)
    ref = np.unpackbits(head['eval_%s_tp' % tag])[:case['det_cls'].numel()].astype(bool)
    assert np.array_equal(oracle_tp(case, num_cls, 0.5), ref) and ref.any() and not ref.all()


# ---- the helpers have teeth: a wrong restatement is rejected on the inputs the GPU tests use ----
def test_fp32_oracle_passes_the_gpu_checks():
    """The fp32 oracle itself passes check_decode / check_loss / check_filter_nms (so a rejection below is due to the planted error)."""
    f = decode_input(2, 10, 19, 5, 36, 7)
    check_decode(oracle32_decode(f, O.synth_anchors(5)), f, O.synth_anchors(5), 36, 'cpu ')
    f, anchors, data = loss_input(2, 19, 10, 3, 3, 16, 11)
    check_loss(oracle32_loss(f, anchors, data, 0.6, True, WEIGHTS), f, anchors, data, 0.6, True, WEIGHTS, 'cpu ')


def test_wrong_meshgrid_is_rejected(monkeypatch):
    """cols in place of rows: invisible on a square grid, caught on every other one -- in the decode and in the loss."""
    right = O.meshgrid

    def wrong(rows, cols):
        k = torch.arange(0, rows * cols)
        return torch.stack([k // cols, k % cols], 1)

    assert torch.equal(wrong(13, 13), right(13, 13))
    for rows, cols in GRIDS:
        if rows == cols:
            continue
        assert not torch.equal(wrong(rows, cols), right(rows, cols))
        f, anchors = decode_input(1, rows, cols, 3, 3, 5), O.synth_anchors(3)
        monkeypatch.setattr(O, 'meshgrid', wrong)
        bad = oracle32_decode(f, anchors)
        fl, al, data = loss_input(2, rows, cols, 5, 20, 16, 13)
        bad_loss = oracle32_loss(fl, al, data, 0.6, True, WEIGHTS)
        monkeypatch.setattr(O, 'meshgrid', right)
        with pytest.raises(AssertionError):
            check_decode(bad, f, anchors, 3, 'cpu ')
        with pytest.raises(AssertionError):
            check_loss(bad_loss, fl, al, data, 0.6, True, WEIGHTS, 'cpu ')


def test_softmax_without_max_subtraction_is_rejected():
    f, anchors = decode_input(1, 7, 5, 5, 20, 3), O.synth_anchors(5)
    bad = oracle32_decode(f, anchors)
    e = torch.exp(bad['logits'])
    bad['prob'] = e / e.sum(-1, keepdim=True)
    with pytest.raises(AssertionError):
        check_decode(bad, f, anchors, 20, 'cpu ')
    f2 = torch.randn(1, 125, 7, 5, generator=torch.Generator().manual_seed(3))       # without the spread-60 band the two agree
    ok = oracle32_decode(f2, anchors)
    e = torch.exp(ok['logits'])
    ok['prob'] = e / e.sum(-1, keepdim=True)
    check_decode(ok, f2, anchors, 20, 'cpu ')


def test_small_probabilities_are_seen():
    """A 10 % error on a probability below 1e-4 -- which max|d| / max|ref| <= 1e-5 lets through -- is rejected."""
    f, anchors = decode_input(1, 7, 5, 5, 20, 3), O.synth_anchors(5)
    bad = oracle32_decode(f, anchors)
    p = bad['prob'].view(-1)
    i = int(((p > 5e-5) & (p < 9e-5)).nonzero()[0])
    p[i] *= 1.1
    assert (bad['prob'] - O.class_prob(O.decode(f, anchors))).abs().max() / 1.0 <= 1e-5
    with pytest.raises(AssertionError):
        check_decode(bad, f, anchors, 20, 'cpu ')


def test_swapped_loss_weights_are_rejected():
    f, anchors, data = loss_input(2, 10, 19, 5, 20, 16, 17)
    swapped = dict(WEIGHTS, center=WEIGHTS['size'], size=WEIGHTS['center'])
    with pytest.raises(AssertionError):
        check_loss(oracle32_loss(f, anchors, data, 0.6, True, swapped), f, anchors, data, 0.6, True, WEIGHTS, 'cpu ')
    zero = dict(WEIGHTS, size=0.0)                    # a weight of 0 removes the term's gradient: both sides must agree on which
    check_loss(oracle32_loss(f, anchors, data, 0.6, True, zero), f, anchors, data, 0.6, True, zero, 'cpu ')
    with pytest.raises(AssertionError):
        check_loss(oracle32_loss(f, anchors, data, 0.6, True, dict(WEIGHTS, center=0.0)), f, anchors, data, 0.6, True, zero, 'cpu ')


def test_wrong_nms_and_argmax_are_rejected():
    """NMS with `<` for `<=` (the lattice input has IoUs exactly equal to the overlap), arg-max taking the last maximum (the
    lattice class scores tie), `>=` for `>` at the thresholds (scores reach them exactly)."""
    score, lo, hi, prob = nms_input(845, 20, 21, 'lattice')
    ref = oracle_filter_nms(score, lo, hi, prob, 1, 0.5, 200)
    below = float(np.nextafter(np.float32(0.5), np.float32(0)))
    wrong = oracle_filter_nms(score, lo, hi, prob, 1, below, 200)               # iou <= just-below-0.5  ==  iou < 0.5
    got = dict(n_filtered=np.array([wrong['n_filtered']]), n_keep=np.array([len(wrong['keep_idx'])]),
               keep_idx=wrong['keep_idx'][None], keep_box=wrong['keep_box'][None])
    with pytest.raises(AssertionError):
        check_filter_nms(got, 0, ref, 200, 'cpu ')
    last = prob.size(1) - 1 - prob.flip(-1).argmax(-1)
    with pytest.raises(AssertionError):
        assert_same('cpu best_cls', last.numpy(), ref['best_cls'])
    assert bool((score == THRESHOLD).any()) and bool((score.unsqueeze(-1) * prob == THRESHOLD_CLS).any())
    assert int((score > THRESHOLD).sum()) != int((score >= THRESHOLD).sum())
    area = (hi - lo).prod(-1)
    assert bool((area == 0).any())
    m = O.iou_matrix(lo, hi, lo, hi)
    assert bool((m == 0.5).any()) and bool((m == 1).sum() > 845)


# ====================================================================================================================================
# on the GPU
# ====================================================================================================================================
@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


def gpu_decode(ops, feature, anchors, c, with_prob=True):
    return {k: v.cpu() for k, v in ops.decode(feature.to(DEV), anchors.to(DEV), c, with_prob=with_prob).items()}


@gpu
@pytest.mark.parametrize('tag', list(O.HEAD_CASES))
def test_decode_and_loss_vs_executed_reference(ops, head, tag):
    """Every head.npz case through yb_decode_fwd, yb_region_loss_fwd and yb_region_loss_bwd."""
    dec, loss = head_case_results(tag, lambda f, a, c: gpu_decode(ops, f, a, c), lambda *args: gpu_loss(ops, *args))
    check_against_head_npz(head, tag, dec, loss, exact_masks=False)
    if tag == 'nopos_one':
        assert loss['pos_count'][1] == 0 and loss['pos_count'][0] > 0 and loss['pos_count'][2] > 0
    if tag == 'nopos_all':
        assert not loss['pos_count'].any() and not np.asarray(loss['positive']).any()


@gpu
@pytest.mark.parametrize('head_shape', HEADS, ids=lambda h: 'A%dC%d' % h)
@pytest.mark.parametrize('grid', GRIDS, ids=lambda g: '%dx%d' % g)
@pytest.mark.parametrize('batch', [1, 3])
def test_decode_sweep_vs_float64(ops, batch, grid, head_shape):
    """Ragged last 32-cell block (every grid but none is a multiple of 32), the > 48 KB slab (A5C80), no logits (C = 1)."""
    (rows, cols), (a, c) = grid, head_shape
    f, anchors = decode_input(batch, rows, cols, a, c, 1000 * batch + 10 * rows + cols + a + c), O.synth_anchors(a)
    got = gpu_decode(ops, f, anchors, c)
    check_decode(got, f, anchors, c)
    assert bool(torch.isinf(got['yx_max']).any()) == (a > 1), 'the saturating band overflows exp * anchor for the larger anchors'
    assert ('logits' in got) == (c > 1)


@gpu
def test_decode_batch64_and_without_prob(ops):
    f, anchors = decode_input(64, 19, 19, 5, 20, 77), O.synth_anchors(5)
    got = gpu_decode(ops, f, anchors, 20)
    check_decode(got, f, anchors, 20)
    bare = gpu_decode(ops, f, anchors, 20, with_prob=False)
    assert 'prob' not in bare
    for k in bare:
        assert torch.equal(bare[k], got[k]), k
    f80 = decode_input(2, 10, 19, 5, 80, 78)
    bare = gpu_decode(ops, f80, anchors, 80, with_prob=False)
    check_decode(bare, f80, anchors, 80)


@gpu
def test_decode_refuses_bad_shapes(ops):
    anchors = O.synth_anchors(5).to(DEV)
    with pytest.raises(ValueError):
        ops.decode(torch.zeros(1, 124, 13, 13, device=DEV), anchors, 20)                 # channel count != A * (5 + C)
    a9 = O.synth_anchors(9).to(DEV)
    with pytest.raises(RuntimeError, match='shared-memory slab'):                        # 9 * 180 * 33 * 4 bytes > 200 KB
        ops.decode(torch.zeros(1, 9 * 180, 2, 2, device=DEV), a9, 175)
    ok = ops.decode(torch.zeros(1, 9 * 170, 2, 2, device=DEV), a9, 165)                  # 197 KB: the largest slab still runs
    assert bool((ok['prob'] == 1.0 / 165).all())


LOSS_SHAPES = [(1, 1), (5, 16), (1, 128), (5, 1), (1, 16), (5, 128)]      # (batch, ground-truth slots), cycled over the sweep


@gpu
@pytest.mark.parametrize('cross_entropy', [True, False], ids=['xent', 'onehot'])
@pytest.mark.parametrize('head_shape', HEADS, ids=lambda h: 'A%dC%d' % h)
@pytest.mark.parametrize('grid', GRIDS, ids=lambda g: '%dx%d' % g)
def test_region_loss_sweep_vs_float64(ops, grid, head_shape, cross_entropy):
    (rows, cols), (a, c) = grid, head_shape
    if c == 1 and not cross_entropy:
        pytest.skip('a single-class head has no class term')
    i = GRIDS.index(grid) * len(HEADS) + HEADS.index(head_shape) + (0 if cross_entropy else 3)
    batch, slots = LOSS_SHAPES[i % len(LOSS_SHAPES)]
    weights = dict(WEIGHTS)
    weights[TERMS[i % 5]] = 0.0 if i % 4 == 3 else weights[TERMS[i % 5]]              # one weight set to 0 in a quarter of the cases
    f, anchors, data = loss_input(batch, rows, cols, a, c, slots, 500 + i)
    check_loss(gpu_loss(ops, f, anchors, data, 0.6, cross_entropy, weights), f, anchors, data, 0.6, cross_entropy, weights)


@gpu
@pytest.mark.parametrize('grid', [(10, 19), (19, 10), (7, 5)], ids=lambda g: '%dx%d' % g)
@pytest.mark.parametrize('head_shape', [(5, 20), (3, 3), (9, 1)], ids=lambda h: 'A%dC%d' % h)
def test_region_loss_edge_targets(ops, grid, head_shape):
    """Centres on cell edges and in the last row / column of a non-square grid, several ground truths on one (cell, anchor), an
    all-padding image between two with positives, class ids outside [0, C) (clamped)."""
    (rows, cols), (a, c) = grid, head_shape
    f = torch.randn(3, channels(a, c), rows, cols, generator=torch.Generator().manual_seed(rows + a)) * 1.2
    anchors, data = O.synth_anchors(a), edge_targets(rows, cols, c)
    got = gpu_loss(ops, f, anchors, data, 0.6, True, WEIGHTS)
    check_loss(got, f, anchors, clamp_cls(data, c), 0.6, True, WEIGHTS)
    pos = got['positive'].reshape(3, rows, cols, a).astype(bool)
    assert pos[0, 2, 3].any() and pos[0, rows - 1, 1].any() and pos[0, 0, cols - 1].any() and pos[0, rows - 1, cols - 1].any() and pos[0, 0, 0].any()
    assert got['pos_count'].tolist() == [5, 0, int(pos[2].sum())] and 3 <= pos[2].sum() <= 4 and pos[2, 3, 2].sum() == 1


@gpu
def test_region_loss_without_any_positive(ops):
    """npos = 0: the four sums are exact zeros apart from the background, the class term and its gradient are 0 (not the NaN of a
    mean over zero rows), the gradient is the background's alone."""
    f, anchors, data = loss_input(2, 13, 17, 5, 20, 4, 9)
    data = {k: torch.zeros_like(v) for k, v in data.items()}
    got = gpu_loss(ops, f, anchors, data, 0.6, True, WEIGHTS)
    check_loss(got, f, anchors, data, 0.6, True, WEIGHTS)
    assert got['losses'][0] == 0 and got['losses'][2] == 0 and got['losses'][3] == 0 and got['losses'][4] == 0 and got['losses'][1] > 0
    g = got['dfeature'].view(2, 5, 25, -1)
    assert bool((g[:, :, 1:] == 0).all()) and bool((g[:, :, 0] != 0).all()) and np.asarray(got['negative']).all()


@gpu
def test_region_loss_refuses_129_slots(ops):
    f, anchors, _ = loss_input(1, 7, 5, 5, 20, 1, 1)
    z = torch.zeros(1, 129, 2, device=DEV)
    with pytest.raises(RuntimeError, match='G <= 128'):
        ops.region_loss_forward(f.to(DEV), anchors.to(DEV), z, z.clone(), torch.zeros(1, 129, dtype=torch.int64, device=DEV), 0.6)


# ---- filter + NMS + expansion ----
@gpu
@pytest.mark.parametrize('kind', ['smooth', 'lattice'])
@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('c', [1, 3, 20, 24, 32, 36, 80])
def test_filter_nms_class_counts(ops, c, mode, kind):
    """Vector / scalar arg-max (C % 4), the partial last group of 20 (24, 36, 80), bit 31 of the class mask (32), scalar expansion
    (C > 32 or C % 4 != 0); two images per launch, overlap 0.5 so that the lattice's IoU == overlap pairs decide."""
    imgs = [nms_input(845, c, 40 + c + i, kind) for i in range(2)]
    score, lo, hi, prob = (torch.stack(t) for t in zip(*imgs))
    got = gpu_filter_nms(ops, score, lo, hi, prob, mode, 0.5, 200)
    for bi in range(2):
        check_filter_nms(got, bi, oracle_filter_nms(*imgs[bi], mode, 0.5, 200), 200)


@gpu
@pytest.mark.parametrize('limit', [1, 31, 32, 33, 200, 1024])
@pytest.mark.parametrize('n', [1, 31, 32, 33, 845, 1805, 16384])
def test_filter_nms_sizes_and_limits(ops, n, limit):
    """limit > n (scratch padded to limit + 1), n_filtered > limit, 32 mask words at limit 1024; n = 16384 with limit 1024 needs more
    shared memory than an SM has and is refused before the launch."""
    kind = 'lattice' if (n + limit) % 2 else 'smooth'
    score, lo, hi, prob = nms_input(n, 20, n + limit, kind)
    args = (score[None], lo[None], hi[None], prob[None], 1, 0.45, limit)
    if n == 16384 and limit == 1024:
        with pytest.raises(RuntimeError, match='shared memory'):
            gpu_filter_nms(ops, *args)
        return
    ref = oracle_filter_nms(score, lo, hi, prob, 1, 0.45, limit)
    check_filter_nms(gpu_filter_nms(ops, *args), 0, ref, limit)
    assert ref['n_filtered'] > limit or n <= 33 or limit == 1024 or kind == 'lattice'


@gpu
@pytest.mark.parametrize('overlap', [0.0, 0.25, 0.45, 1.0])
def test_filter_nms_overlap_extremes_and_plain_nms(ops, overlap):
    """overlap 0 keeps only disjoint (or zero-area) boxes, overlap 1 keeps everything up to the limit; FILTER_NONE without prob."""
    import utils.postprocess
    for kind in ('smooth', 'lattice'):
        score, lo, hi, _ = nms_input(1200, 1, 70, kind)
        ref = O.nms(score.numpy(), lo.numpy(), hi.numpy(), overlap, 200)
        got = gpu_filter_nms(ops, score[None], lo[None], hi[None], None, 2, overlap, 200, expand=False, details=False)
        assert got['keep_idx'][0, :int(got['n_keep'][0])].tolist() == ref
        assert utils.postprocess.nms(score.to(DEV), lo.to(DEV), hi.to(DEV), overlap, 200) == ref
        if overlap == 1.0:
            assert len(ref) == 200


@gpu
def test_filter_nms_mixed_batch_and_optional_outputs(ops):
    """Eight images -- empty (nothing passes), one box, saturated (more than `limit` pass), repeated -- in one launch; `details` and
    `expand` on or off leave the common outputs unchanged."""
    imgs = [list(nms_input(845, 20, 80 + i, 'lattice' if i % 2 else 'smooth')) for i in range(8)]
    for i in (0, 3, 7):
        imgs[i][0] = torch.zeros(845)                         # nothing passes
    imgs[5][0] = torch.zeros(845); imgs[5][0][400] = 1.0     # exactly one box
    imgs[5][3] = imgs[5][3].clone(); imgs[5][3][400, 7] = 1.0
    score, lo, hi, prob = (torch.stack(t) for t in zip(*imgs))
    for mode in (0, 1):
        full = gpu_filter_nms(ops, score, lo, hi, prob, mode, 0.45, 200)
        refs = [oracle_filter_nms(*img, mode, 0.45, 200) for img in imgs]
        for bi in range(8):
            check_filter_nms(full, bi, refs[bi], 200)
        assert [r['n_filtered'] for r in refs][0] == 0 and refs[5]['n_filtered'] == 1 and max(r['n_filtered'] for r in refs) > 200
        for expand, details in ((False, False), (True, False), (False, True)):
            part = gpu_filter_nms(ops, score, lo, hi, prob, mode, 0.45, 200, expand=expand, details=details)
            for bi in range(8):
                check_filter_nms(part, bi, refs[bi], 200)


@gpu
def test_filter_nms_truncates_at_det_cap(ops):
    """A det_cap below the number of (box, class) pairs: n_det == det_cap, the entries are the head of the untruncated list, and the
    memory after each det array is untouched."""
    imgs = [nms_input(845, 20, 90 + i, 'smooth') for i in range(2)]
    score, lo, hi, prob = (torch.stack(t).to(DEV) for t in zip(*imgs))
    refs = [oracle_filter_nms(*img, 1, 0.45, 200) for img in imgs]
    cap = 50
    assert all(len(r['det_keep']) > cap for r in refs)
    i32 = dict(dtype=torch.int32, device=DEV)
    nf, nk, nd = torch.empty(2, **i32), torch.empty(2, **i32), torch.empty(2, **i32)
    kidx, kbox = torch.empty(2, 200, **i32), torch.empty(2, 200, **i32)
    guard = 4096
    ibuf = torch.full((2, 2 * cap + guard), -7, **i32)        # det_keep | guard, det_cls | guard
    fbuf = torch.full((2 * cap + guard,), -7.0, device=DEV)   # det_score | guard
    det_keep, det_cls, det_score = ibuf[0, :2 * cap], ibuf[1, :2 * cap], fbuf[:2 * cap]
    ops.call('yb_filter_nms', score, lo, hi, prob, 2, 845, 20, 1, THRESHOLD, THRESHOLD_CLS, 0.45, 200, nf, nk, kidx, kbox, nd, det_keep,
             det_cls, det_score, cap, None, None, None)
    assert nd.tolist() == [cap, cap]
    for bi in range(2):
        assert det_keep[bi * cap:(bi + 1) * cap].tolist() == refs[bi]['det_keep'][:cap].tolist()
        assert det_cls[bi * cap:(bi + 1) * cap].tolist() == refs[bi]['det_cls'][:cap].tolist()
        assert np.array_equal(det_score[bi * cap:(bi + 1) * cap].cpu().numpy(), refs[bi]['det_score'][:cap])
    assert bool((ibuf[:, 2 * cap:] == -7).all()) and bool((fbuf[2 * cap:] == -7.0).all())


@gpu
def test_filter_nms_refuses_sizes_over_capacity(ops):
    z = lambda *s: torch.zeros(*s, device=DEV)
    with pytest.raises(RuntimeError, match='16384'):
        ops.filter_nms(z(1, 16385), z(1, 16385, 2), z(1, 16385, 2), None, 2, 0.0, 0.0, 0.45, 200)
    with pytest.raises(RuntimeError, match='limit <= 1024'):
        ops.filter_nms(z(1, 64), z(1, 64, 2), z(1, 64, 2), None, 2, 0.0, 0.0, 0.45, 1025)


@gpu
@pytest.mark.parametrize('tag,fix', [(t, f) for t, modes in O.HEAD_POST_MODES.items() for f in modes])
def test_detect_entry_points_vs_executed_reference(head, tag, fix):
    import detect
    inputs, ref = post_case(head, tag, fix)
    dev = tuple(t.to(DEV) for t in inputs)
    cfg = make_config(fix)
    check_post_case(ref, inputs, detect.filter_visible(cfg, *dev), detect.postprocess(cfg, *dev))


@gpu
@pytest.mark.parametrize('tag', list(O.HEAD_NMS_CASES))
def test_nms_entry_point_vs_executed_reference(head, tag):
    import utils.postprocess
    n, seed, overlap, limit = O.HEAD_NMS_CASES[tag]
    score, a, b = O.synth_lattice_boxes(n, seed)
    assert utils.postprocess.nms(score.to(DEV), a.to(DEV), b.to(DEV), overlap, limit) == head['nms_%s_keep' % tag].tolist()


@gpu
@pytest.mark.parametrize('fix', [1, 0])
def test_postprocess_batch_on_nonsquare_80_class_decode(ops, fix):
    """ops.decode -> detect.postprocess_batch on a 10 x 19, 80-class head; image 1 is an empty image between full ones.  The oracle
    runs on the GPU's own decoded tensors, so every comparison is exact."""
    import detect
    f = torch.randn(3, 425, 10, 19, generator=torch.Generator().manual_seed(12)) * 2
    f.view(3, 5, 85, 190)[1, :, 0] = -40.0                    # objectness ~ 0: nothing passes either filter
    pred = ops.decode(f.to(DEV), O.synth_anchors(5).to(DEV), 80)
    results = detect.postprocess_batch(make_config(fix), pred)
    assert results[1] is None and results[0] is not None and results[2] is not None
    for bi, res in enumerate(results):
        exp = O.postprocess(pred['iou'][bi].reshape(-1).cpu(), pred['yx_min'][bi].reshape(-1, 2).cpu(), pred['yx_max'][bi].reshape(-1, 2).cpu(),
                            pred['prob'][bi].reshape(-1, 80).cpu(), bool(fix), 0.3, 0.005, 0.45)
        assert (res is None) == (exp is None)
        if res is not None:
            for got, want in zip(res, exp):
                assert torch.equal(got.cpu(), want)


# ---- IoU matrices ----
def iou_boxes(n, seed):
    """Random, nested, touching, disjoint and zero-area boxes."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(n, 2, generator=g) * 10
    hi = lo + torch.rand(n, 2, generator=g) * 5
    for i in range(0, n - 4, 5):
        lo[i + 1], hi[i + 1] = lo[i] + 0.25, hi[i] - 0.25 * (hi[i] - lo[i])          # nested in box i
        lo[i + 2] = torch.stack([lo[i][0], hi[i][1]]); hi[i + 2] = lo[i + 2] + 1       # touching box i along an edge
        lo[i + 3] = hi[i] + 3; hi[i + 3] = lo[i + 3] + 1                               # disjoint
        hi[i + 4] = torch.stack([lo[i + 4][0], hi[i + 4][1]])                          # zero area
    return lo, hi


@gpu
@pytest.mark.parametrize('batch', [1, 7])
def test_iou_matrix_bit_exact(ops, batch):
    sets = [(iou_boxes(45, 3 * b), iou_boxes(23, 3 * b + 1)) for b in range(batch)]
    a0, a1 = (torch.stack([s[0][k] for s in sets]) for k in (0, 1))
    b0, b1 = (torch.stack([s[1][k] for s in sets]) for k in (0, 1))
    a0[0, :23], a1[0, :23] = b0[0], b1[0]                                            # identical pairs: IoU exactly 1 (or 0 / eps at zero area)
    got = ops.iou_matrix(a0.to(DEV), a1.to(DEV), b0.to(DEV), b1.to(DEV)).cpu()
    ref = O.batch_iou_matrix(a0, a1, b0, b1)
    assert torch.equal(got, ref) and bool((ref == 0).any()) and bool((ref == 1).any())
    got2 = ops.iou_matrix(a0[0].to(DEV), a1[0].to(DEV), b0[0].to(DEV), b1[0].to(DEV)).cpu()
    assert torch.equal(got2, O.iou_matrix(a0[0], a1[0], b0[0], b1[0]))
    e = torch.zeros(batch, 0, 2, device=DEV)
    assert ops.iou_matrix(e, e, b0.to(DEV), b1.to(DEV)).shape == (batch, 0, 23)
    assert ops.iou_matrix(a0.to(DEV), a1.to(DEV), e, e).shape == (batch, 45, 0)


# ---- evaluation matching ----
@gpu
@pytest.mark.parametrize('num_cls', [1, 20, 80])
def test_eval_matching_ragged_batch(num_cls):
    """80 classes iterate the class-stride loop (more than 8 * 4 warps' worth); 40 boxes of one class the lane-stride scan and the
    shuffle tie-break (duplicated boxes -> lowest index); 1024 boxes the whole claimed bitmap."""
    import eval as yb_eval
    rows = eval_batch(num_cls)
    expect = np.concatenate([oracle_tp(r, num_cls, 0.45) for r in rows])
    det_off = torch.from_numpy(np.cumsum([0] + [r['det_cls'].numel() for r in rows]))
    gt_off = torch.from_numpy(np.cumsum([0] + [r['gt_cls'].numel() for r in rows]))
    cat = lambda key: torch.cat([r[key] for r in rows]).to(DEV)
    tp = yb_eval.matching_batch(cat('det_min'), cat('det_max'), cat('det_cls'), det_off, cat('gt_min'), cat('gt_max'), cat('gt_cls'), gt_off,
                                num_cls, 0.45).cpu().numpy().astype(bool)
    assert_same('eval tp', tp, expect)
    crowd = slice(int(det_off[3]), int(det_off[4]))
    assert 0 < expect[crowd].sum() <= 20, 'duplicated ground truth: only the lower index of each pair can be claimed'
    # AP through eval.py's host functions on the kernel's flags == the oracle's on its own
    score = torch.cat([r['score'] for r in rows]).numpy()
    det_cls, gt_cls = torch.cat([r['det_cls'] for r in rows]).numpy(), torch.cat([r['gt_cls'] for r in rows]).numpy()
    for metric07 in (0, 1):
        cfg = make_config(1, metric07)
        for c in range(num_cls):
            m = det_cls == c
            num = int((gt_cls == c).sum())
            if num and m.any():
                order = np.argsort(-score[m], kind='stable')
                assert yb_eval.average_precision(cfg, tp[m][order], num) == O.average_precision(expect[m][order], num, bool(metric07))


@gpu
@pytest.mark.parametrize('tag', list(O.HEAD_EVAL_CASES))
def test_eval_matching_vs_executed_reference(head, tag):
    import eval as yb_eval
    case, num_cls = O.head_eval_case(tag)
    n, g = case['det_cls'].numel(), case['gt_cls'].numel()
    tp = yb_eval.matching_batch(case['det_min'].to(DEV), case['det_max'].to(DEV), case['det_cls'].to(DEV), torch.tensor([0, n]),
                                case['gt_min'].to(DEV), case['gt_max'].to(DEV), case['gt_cls'].to(DEV), torch.tensor([0, g]), num_cls, 0.5)
    assert np.array_equal(tp.cpu().numpy().astype(bool), np.unpackbits(head['eval_%s_tp' % tag])[:n].astype(bool))


@gpu
def test_eval_matching_refuses_1025_ground_truths():
    import eval as yb_eval
    z = lambda n: torch.zeros(n, 2, device=DEV)
    with pytest.raises(RuntimeError, match='1024'):
        yb_eval.matching_batch(z(3), z(3), torch.zeros(3, dtype=torch.int32), torch.tensor([0, 3]), z(1025), z(1025),
                               torch.zeros(1025, dtype=torch.int32), torch.tensor([0, 1025]), 1, 0.5)
