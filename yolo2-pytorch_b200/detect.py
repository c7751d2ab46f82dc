"""detect -- detection post-filter on the GPU (reference detect.py:43-80).

`get_logits`, `filter_visible`, `postprocess` keep the reference's single-image signatures and
return values; `postprocess_batch` is the H100-native entry point that processes every image of a
batch in ONE kernel launch (yb_filter_nms: threshold filter -> stable sort -> greedy NMS ->
per-class expansion, one CTA per image, no host round trips until the results are read).
The cv2 capture/draw loop of the reference's `Detect` class is host glue outside the hot path.
"""
import torch

from b200 import ops as _ops


def get_logits(pred):
    """reference detect.py:43-48."""
    if 'logits' in pred:
        return pred['logits'].contiguous()
    size = pred['iou'].size()
    return torch.ones(*size, 1, device=pred['iou'].device)


def get_prob(pred):
    """Class probabilities: the decode kernel's fused softmax when present (pred['prob'])."""
    if 'prob' in pred:
        return pred['prob']
    raise RuntimeError('pred has no fused `prob`; build it with model._inference on the GPU Inference module')


def _config_filter(config):
    fix = config.getboolean('detect', 'fix')
    mode = _ops.FILTER_FIX if fix else _ops.FILTER_THRESHOLD
    threshold = 0.0 if fix else config.getfloat('detect', 'threshold')
    threshold_cls = config.getfloat('detect', 'threshold_cls') if fix else 0.0
    return fix, mode, threshold, threshold_cls


def _run(config, iou, yx_min, yx_max, prob, expand, details):
    fix, mode, threshold, threshold_cls = _config_filter(config)
    b = iou.size(0)
    n = iou[0].numel()
    num = prob.size(-1)
    return fix, _ops.filter_nms(iou.reshape(b, n).contiguous(), yx_min.reshape(b, n, 2).contiguous(),
                                yx_max.reshape(b, n, 2).contiguous(), prob.reshape(b, n, num).contiguous(), mode, threshold,
                                threshold_cls, config.getfloat('detect', 'overlap'), 200, expand=expand, details=details)


def filter_visible(config, iou, yx_min, yx_max, prob):
    """reference detect.py:51-63, ONE image: iou [N], yx_* [N,2], prob [N,C] ->
    (iou, yx_min, yx_max, prob, prob_cls, cls) of the boxes passing the threshold (ascending index)."""
    n = iou.numel()
    fix, res = _run(config, iou.reshape(1, n), yx_min.reshape(1, n, 2), yx_max.reshape(1, n, 2), prob.reshape(1, n, -1), False, True)
    nf = int(res['n_filtered'][0].item())
    sel = res['filt_box'][0, :nf].long()
    return (iou.reshape(-1)[sel], yx_min.reshape(n, 2)[sel], yx_max.reshape(n, 2)[sel], prob.reshape(n, -1)[sel],
            res['best_prob'][0][sel], res['best_cls'][0][sel].long())


def _unpack(res, bi, fix, iou, yx_min, yx_max):
    nk = int(res['n_keep'][bi])
    if nk == 0:
        return None
    kbox = res['keep_box'][bi, :nk].long()
    k_iou = iou[kbox]
    if fix:
        nd = int(res['n_det'][bi])
        dbox = kbox[res['det_keep'][bi, :nd].long()]
        return k_iou, yx_min[dbox], yx_max[dbox], res['det_cls'][bi, :nd].long(), res['det_score'][bi, :nd]
    # detect.py:71,79: cls is the filtered argmax class of each kept box, score = iou
    return k_iou, yx_min[kbox], yx_max[kbox], res['best_cls'][bi][kbox].long(), k_iou


def postprocess(config, iou, yx_min, yx_max, prob):
    """reference detect.py:66-80, ONE image.  Returns None when nothing is kept, else
    (iou[k], yx_min[m,2], yx_max[m,2], cls[m], score[m])."""
    n = iou.numel()
    iou, yx_min, yx_max, prob = iou.reshape(n), yx_min.reshape(n, 2), yx_max.reshape(n, 2), prob.reshape(n, -1)
    fix, res = _run(config, iou.reshape(1, n), yx_min.reshape(1, n, 2), yx_max.reshape(1, n, 2), prob.reshape(1, n, -1), True, True)
    host = {k: res[k].cpu() for k in ('n_keep', 'n_det')}
    host.update({k: res[k] for k in res if k not in host})
    return _unpack(host, 0, fix, iou, yx_min, yx_max)


def postprocess_batch(config, pred):
    """Batched form: pred is the dict from model._inference.  One launch for the whole batch, one
    device->host copy of the per-image counts; returns a list (len B) of `postprocess` results."""
    iou, yx_min, yx_max = pred['iou'], pred['yx_min'], pred['yx_max']
    prob = get_prob(pred)
    b = iou.size(0)
    n = iou[0].numel()
    fix, res = _run(config, iou, yx_min, yx_max, prob, True, True)
    host = dict(res)
    host['n_keep'] = res['n_keep'].cpu()
    host['n_det'] = res['n_det'].cpu()
    iou, yx_min, yx_max = iou.reshape(b, n), yx_min.reshape(b, n, 2), yx_max.reshape(b, n, 2)
    return [_unpack(host, bi, fix, iou[bi], yx_min[bi], yx_max[bi]) for bi in range(b)]
