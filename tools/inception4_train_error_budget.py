#!/usr/bin/env python
"""Error budget of one Inception-v4 TRAINING step under the GPU path's fp16 storage, with BatchNorm on or off, in float64 arithmetic with
only those roundings added (tests/inception4_train_oracle.Rounding: conv weights -> fp16 except features.0's, every raw conv output z,
activation and count-exclusive pooled tensor -> fp16, every stored gradient -> fp16 at the trainer's loss scale, the pool's gradient
included).  The step (train-mode forward, the synthetic loss sum(feature * R), autograd backward) is compared with the exact float64 step
on the same batch, as tests/test_inception4_train.py::test_training_step_vs_fp64_restatement compares the GPU step: feature, median and
worst gradient relative L2 and cosine, running statistics.

    python tools/inception4_train_error_budget.py 4 107 139 [--nobn]     # batch, H, W (cuda:0 when there is one, else the CPU)

Prints one JSON line; writes nothing.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import inception4_oracle as I  # noqa: E402
import inception4_train_oracle as T4  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

SCALE = 32.0      # b200.train_engine.Inception4Trainer's loss scale


def budget(b, h, w, bn=True, seed=0, image_seed=12, device=None):
    device = device or ('cuda' if torch.cuda.is_available() else 'cpu')
    sd = I.make_state_dict(seed, bn=bn)
    x = O.synth_images(b, h, w, seed=image_seed)
    f_ref, _, g_ref, s_ref = T4.train_step(sd, x, device=device)
    f16, _, g16, s16 = T4.train_step(sd, x, rnd=T4.Rounding(SCALE), device=device)
    if not s_ref:                  # BatchNorm off: no running statistics
        s16 = s_ref = {'-': torch.ones(1)}
    return T4.step_errors(f16, g16, s16, f_ref, g_ref, s_ref, sorted(g_ref))


def main():
    args = [a for a in sys.argv[1:] if not a.startswith('--')]
    bn = '--nobn' not in sys.argv
    b, h, w = (int(v) for v in args[:3]) if len(args) >= 3 else (4, 107, 139)
    torch.set_num_threads(8)
    print(json.dumps(dict(batch=b, size=[h, w], batch_norm=bn, scale=SCALE, **budget(b, h, w, bn))))


if __name__ == '__main__':
    main()
