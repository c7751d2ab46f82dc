"""eval -- detection-quality bookkeeping immediately downstream of NMS (SURVEY 8f rank 3), H100-native where it is per-image
work: the greedy true-positive matching of reference eval.py:57-75 (`_matching` / `matching`, called per image and per class
from `Eval.filter_cls`, eval.py:210-216) runs as one CUDA launch for a whole batch (`matching_batch`, yb_eval_match); the
per-dataset reductions `voc_ap` / `average_precision` (eval.py:78-121) are the same few numpy lines as in the reference --
they touch one small array per class once per evaluation.  Names and argument meaning follow the reference.
"""
import numpy as np
import torch

from b200 import ops as _ops

EPS32 = 1.1920928955078125e-07


def matching_batch(det_yx_min, det_yx_max, det_cls, det_off, gt_yx_min, gt_yx_max, gt_cls, gt_off, num_cls, threshold):
    """Batched `matching`: image i owns detections [det_off[i], det_off[i+1]) -- in descending-score order, as
    `detect.postprocess` returns them -- and ground-truth boxes [gt_off[i], gt_off[i+1]).  Boxes are float32 [*, 2] (y, x),
    classes and offsets integer tensors, everything on the GPU.  Returns a uint8 device tensor tp[num_detections]."""
    for name, t in (('det_yx_min', det_yx_min), ('det_yx_max', det_yx_max), ('gt_yx_min', gt_yx_min), ('gt_yx_max', gt_yx_max)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RuntimeError('eval.matching_batch: %s must be a CUDA tensor; there is no CPU fallback' % name)
    dev = det_yx_min.device
    i32 = lambda t: t.to(device=dev, dtype=torch.int32).contiguous()
    f32 = lambda t: t.to(dtype=torch.float32).contiguous()
    det_off_h = det_off.detach().cpu().long()
    gt_off_h = gt_off.detach().cpu().long()
    batch = det_off_h.numel() - 1
    n = int(det_off_h[-1])
    tp = torch.zeros(n, dtype=torch.uint8, device=dev)
    if n == 0 or batch <= 0:
        return tp
    max_gt = int((gt_off_h[1:] - gt_off_h[:-1]).max()) if batch > 0 else 0
    _ops.call('yb_eval_match', f32(det_yx_min), f32(det_yx_max), i32(det_cls), i32(det_off), f32(gt_yx_min), f32(gt_yx_max), i32(gt_cls),
              i32(gt_off), batch, int(num_cls), max_gt, float(threshold), EPS32, tp)
    return tp


def matching(data_yx_min, data_yx_max, yx_min, yx_max, threshold):
    """reference eval.py:67-75: ground truth [G,2]x2 and detections [N,2]x2 of ONE class of ONE image -> np.bool_[N]."""
    n = yx_min.size(0)
    if data_yx_min.numel() == 0 or n == 0:
        return np.zeros([n], dtype=bool)
    dev = yx_min.device
    zeros_d = torch.zeros(n, dtype=torch.int32, device=dev)
    zeros_g = torch.zeros(data_yx_min.size(0), dtype=torch.int32, device=dev)
    off_d = torch.tensor([0, n], dtype=torch.int32)
    off_g = torch.tensor([0, data_yx_min.size(0)], dtype=torch.int32)
    tp = matching_batch(yx_min, yx_max, zeros_d, off_d, data_yx_min, data_yx_max, zeros_g, off_g, 1, threshold)
    return tp.cpu().numpy().astype(bool)


def filter_valid(yx_min, yx_max, cls, difficult):
    """reference eval.py:140-145: drop zero-padded (min >= max) and `difficult` ground-truth slots."""
    mask = (yx_min < yx_max).all(-1) & (difficult < 1)
    return yx_min[mask], yx_max[mask], cls[mask]


def voc_ap(rec, prec, use_07_metric=False):
    """reference eval.py:78-108 (VOC devkit AP): 11-point metric or the area under the precision envelope."""
    if use_07_metric:
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            p = 0 if np.sum(rec >= t) == 0 else np.max(prec[rec >= t])
            ap = ap + p / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def average_precision(config, tp, num, dtype=np.float64):
    """reference eval.py:111-120: tp = true-positive flags of one class sorted by descending score, num = ground-truth count."""
    tp = np.asarray(tp, dtype=bool)
    fp = np.cumsum(~tp)
    tp = np.cumsum(tp)
    rec = tp / num if num > 0 else np.zeros(len(tp), dtype=dtype)
    prec = tp / np.maximum(tp + fp, np.finfo(dtype).eps)
    return voc_ap(rec, prec, config.getboolean('eval', 'metric07'))


def merge_ap(config, cls_num, cls_score, cls_tp):
    """reference eval.py:296-303: per-class AP from the accumulated (score, tp) lists."""
    cls_ap = {}
    for c, (num, score, tp) in enumerate(zip(cls_num, cls_score, cls_tp)):
        if num > 0:
            order = np.argsort(-np.asarray(score), kind='stable')
            cls_ap[c] = average_precision(config, np.asarray(tp)[order], num)
    return cls_ap
