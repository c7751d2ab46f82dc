#!/usr/bin/env python
"""Golden fixture for the evaluation matching / VOC AP step, produced by EXECUTING the reference's own functions
(eval.py:57-121: `_matching`, `matching`, `voc_ap`, `average_precision`).  eval.py cannot be imported (humanize,
pybenchmark, tinydb, xlsxwriter ... are absent), so the four pure functions are extracted with `ast` and exec'd; the
removed numpy aliases they use (`np.bool`, `np.float`) are supplied in the generator process only.

    python tests/golden/make_golden_eval.py          # build container only (needs /root/reference)
"""
import ast
import configparser
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

REF = '/root/reference'


def reference_eval_fns(utils):
    """The reference's four pure evaluation functions, extracted from eval.py and exec'd."""
    np.bool, np.float = bool, float                  # aliases removed in numpy >= 1.24, used at eval.py:59,73,111
    tree = ast.parse(open(os.path.join(REF, 'eval.py')).read())
    names = ('_matching', 'matching', 'voc_ap', 'average_precision')
    wanted = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    ns = dict(np=np, torch=torch, utils=utils)
    exec(compile(ast.Module(body=wanted, type_ignores=[]), os.path.join(REF, 'eval.py'), 'exec'), ns)
    return ns


def main():
    model, utils, detect = G.import_reference()
    ns = reference_eval_fns(utils)
    out = {}
    cases = [(1, 60, 12, 4), (2, 200, 40, 20), (3, 5, 1, 1), (4, 30, 0, 3), (5, 0, 6, 3)]
    all_tp, all_score, all_num = {}, {}, {}
    for seed, n_det, n_gt, num_cls in cases:
        if n_gt == 0:
            case = O.synth_eval_case(seed, max(n_det, 1), 3, num_cls)
            case['gt_min'], case['gt_max'], case['gt_cls'] = case['gt_min'][:0], case['gt_max'][:0], case['gt_cls'][:0]
        elif n_det == 0:
            case = O.synth_eval_case(seed, 3, n_gt, num_cls)
            for k in ('det_min', 'det_max', 'det_cls', 'score'):
                case[k] = case[k][:0]
        else:
            case = O.synth_eval_case(seed, n_det, n_gt, num_cls)
        tp = np.zeros(case['det_cls'].numel(), dtype=bool)
        for c in range(num_cls):
            dm, gm = case['det_cls'] == c, case['gt_cls'] == c
            t = ns['matching'](case['gt_min'][gm], case['gt_max'][gm], case['det_min'][dm], case['det_max'][dm], 0.5)
            tp[dm.numpy()] = t
            all_tp.setdefault(c, []).append(t)
            all_score.setdefault(c, []).append(case['score'][dm].numpy())
            all_num[c] = all_num.get(c, 0) + int(gm.sum())
        tag = 'case%d_' % seed
        for k, v in case.items():
            out[tag + k] = v.numpy()
        out[tag + 'tp'] = tp
        out[tag + 'num_cls'] = np.int64(num_cls)
    for metric07 in (0, 1):
        config = configparser.ConfigParser()
        config.read_dict({'eval': {'metric07': str(metric07)}})
        for c in sorted(all_tp):
            score, tp = np.concatenate(all_score[c]), np.concatenate(all_tp[c])
            order = np.argsort(-score, kind='stable')
            out['ap%d_cls%d' % (metric07, c)] = np.float64(ns['average_precision'](config, tp[order], all_num[c]))
            out['sorted_tp_cls%d' % c] = tp[order]
            out['num_cls%d' % c] = np.int64(all_num[c])
    path = os.path.join(HERE, 'eval.npz')
    np.savez_compressed(path, **out)
    print('eval.npz %.1f KB' % (os.path.getsize(path) / 1024), {k: float(v) for k, v in out.items() if k.startswith('ap')})


if __name__ == '__main__':
    main()
