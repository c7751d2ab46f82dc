"""utils.postprocess -- greedy NMS on the GPU (reference utils/postprocess.py:23-49)."""
import torch

from b200 import ops as _ops


def nms(score, yx_min, yx_max, overlap=0.5, limit=200):
    """Class-agnostic greedy NMS: sort by score (descending), keep the head, drop every remaining
    box whose IoU with it is > overlap, repeat; only the top-`limit` boxes are considered.
    :param score: [N] scores.  :param yx_min/yx_max: [N, 2] corners (y, x).
    :return: list of indices into the inputs, in descending-score order (bit-identical to the
             reference on the same fp32 inputs).
    The whole loop is one CUDA kernel (yb_filter_nms, one CTA); the only host sync is the final
    read-back that the list-returning API requires."""
    if score.numel() == 0:
        return []
    if not score.is_cuda:
        raise RuntimeError('utils.postprocess.nms: inputs must be CUDA tensors; there is no CPU fallback')
    n = score.numel()
    res = _ops.filter_nms(score.reshape(1, n).contiguous().float(), yx_min.reshape(1, n, 2).contiguous().float(),
                          yx_max.reshape(1, n, 2).contiguous().float(), None, _ops.FILTER_NONE, 0.0, 0.0, overlap, limit)
    k = int(res['n_keep'][0].item())
    return res['keep_idx'][0, :k].tolist()
