#!/usr/bin/env python
"""Golden fixture for the detection head and tail away from the square 20-class 5-anchor family, produced by EXECUTING the
reference's own code on CPU: `model.Inference` with `dnn = lambda t: t` (model/__init__.py:110-135), `model.loss` (:138-167,
under the two torch-0.3.1 shims of make_golden_loss.py), `detect.filter_visible` / `detect.postprocess` (detect.py:51-80),
`utils.postprocess.nms` (utils/postprocess.py:23-49) and eval.py's `matching` (:57-75).

Only the reference's OUTPUTS are stored; the tests regenerate every input from its seed (oracle/yolo2_oracle.py: HEAD_CASES,
head_case_inputs, synth_detections, synth_lattice_boxes, head_eval_case).  Large tensors are stored as the seeded sample of
O.store_sampled.  The post-filter inputs are not decoded feature maps but synth_detections, whose elementwise construction is
bit-identical on every machine, so the exact comparisons do not hang on a CPU's sigmoid.

What the reference does on the cases that are not ordinary (found by running it, kept as fixtures):
  * rows != cols: nothing raises.  The decode grid is the quirked meshgrid (cell k sits at (k // rows, k % rows)) while
    fit_positive marks the true cell i * cols + j, so a positive and the box it is regressed towards can be different cells.
  * `nopos_one` (one image with only padding slots): finite everywhere.
  * `nopos_all` (no ground-truth box in the batch): nothing raises; the four sum terms are 0 or finite, but F.cross_entropy over
    zero rows is NaN and so are the class channels of the gradient.  The fixture stores what the reference returned, NaN included;
    the tests pin the masks, the matched IoU and the four finite terms against it and the class term against the kernels' documented
    0 (DESIGN.md).

    python tests/golden/make_golden_head.py          # build container only (needs /root/reference)
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
warnings.filterwarnings('ignore')
import make_golden as G  # noqa: E402
import make_golden_eval as GE  # noqa: E402
import make_golden_loss as GL  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

def main():
    model, utils, detect = G.import_reference()
    fns = GL.reference_loss_fns(model)
    ev = GE.reference_eval_fns(utils)
    out = {}
    # ---- decode + loss ----
    for tag, k in O.HEAD_CASES.items():
        feature, anchors, data = O.head_case_inputs(tag)
        inference = model.Inference(G.make_config(1), lambda t: t, anchors)
        pred = model._inference(inference, feature.clone().requires_grad_(True))
        for name in ('iou', 'center_offset', 'yx_min', 'yx_max'):
            O.store_sampled(out, '%s_dec_%s' % (tag, name), pred[name].detach().numpy())
        O.store_sampled(out, tag + '_dec_prob', torch.nn.functional.softmax(detect.get_logits(pred).detach(), -1).numpy())
        if k.get('one_hot'):
            data = dict(data, cls=torch.nn.functional.one_hot(data['cls'], k['c']).float())
        losses, debug = fns['loss'](anchors, data, pred, 0.6)
        total = sum(losses[key] * O.HPARAM_DEFAULT[key] for key in losses)
        grad, = torch.autograd.grad(total, pred['feature'])
        for key, v in losses.items():
            out['%s_loss_%s' % (tag, key)] = np.float64(v.item())
        out[tag + '_positive'] = np.packbits(debug['positive'].numpy().astype(bool))
        out[tag + '_negative'] = np.packbits(debug['negative'].numpy().astype(bool))
        O.store_sampled(out, tag + '_iou', debug['iou'].numpy())
        O.store_sampled(out, tag + '_grad', grad.numpy())
    # ---- filter + NMS + expansion ----
    for tag, modes in O.HEAD_POST_MODES.items():
        k = O.HEAD_CASES[tag]
        n = k['rows'] * k['cols'] * k['a']
        iou, yx_min, yx_max, prob = O.synth_detections(n, k['c'], 300 + k['seed'])
        for fix in modes:
            cfg = G.make_config(fix)
            fv = detect.filter_visible(cfg, iou, yx_min, yx_max, prob)
            pre = '%s_fix%d_' % (tag, fix)
            fv_box = G.box_indices(yx_min, yx_max, fv[1], fv[2])
            assert np.array_equal(fv[0].numpy(), iou.numpy()[fv_box])
            out[pre + 'fv_box'] = fv_box.astype(np.int32)
            out[pre + 'fv_prob_cls'] = fv[4].numpy()
            out[pre + 'fv_cls'] = fv[5].numpy().astype(np.int32)
            res = detect.postprocess(cfg, iou, yx_min, yx_max, prob)
            assert res is not None
            keep = [int(i) for i in utils.postprocess.nms(fv[0], fv[1], fv[2], cfg.getfloat('detect', 'overlap'))]
            out[pre + 'keep_box'] = fv_box[keep].astype(np.int32)
            out[pre + 'iou'] = res[0].numpy()
            out[pre + 'det_box'] = G.box_indices(yx_min, yx_max, res[1], res[2]).astype(np.int32)
            out[pre + 'cls'] = res[3].numpy().astype(np.int32)
            out[pre + 'score'] = res[4].numpy()
    # ---- NMS on lattice boxes: IoU exactly equal to the overlap ----
    for tag, (n, seed, overlap, limit) in O.HEAD_NMS_CASES.items():
        score, a, b = O.synth_lattice_boxes(n, seed)
        keep = utils.postprocess.nms(score, a, b, overlap, limit)
        out['nms_%s_keep' % tag] = np.array([int(i) for i in keep], dtype=np.int32)
    # ---- evaluation matching ----
    for tag in O.HEAD_EVAL_CASES:
        case, num_cls = O.head_eval_case(tag)
        tp = np.zeros(case['det_cls'].numel(), dtype=bool)
        for c in range(num_cls):
            dm, gm = case['det_cls'] == c, case['gt_cls'] == c
            tp[dm.numpy()] = ev['matching'](case['gt_min'][gm], case['gt_max'][gm], case['det_min'][dm], case['det_max'][dm], 0.5)
        out['eval_%s_tp' % tag] = np.packbits(tp)
    path = os.path.join(HERE, 'head.npz')
    np.savez_compressed(path, **out)
    print('head.npz %.1f KB' % (os.path.getsize(path) / 1024))
    for tag in O.HEAD_CASES:
        print(tag, {key[len(tag) + 6:]: float(v) for key, v in out.items() if key.startswith(tag + '_loss_')})


if __name__ == '__main__':
    main()
