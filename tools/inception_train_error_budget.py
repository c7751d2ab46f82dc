#!/usr/bin/env python
"""Error budget of one Inception-v3 TRAINING step under the GPU path's fp16 storage, in float64 arithmetic with only those roundings added
(tests/inception_train_oracle.Rounding: conv weights -> fp16 except the stem conv's, every raw conv output z, activation and average-pooled
tensor -> fp16, every stored gradient -> fp16 at the trainer's loss scale, 1024).  The step (train-mode forward, the synthetic loss
sum(feature * R), autograd backward) is compared with the exact float64 step on the same batch, as
tests/test_inception_train.py::test_training_step_vs_fp64_restatement compares the GPU step: feature, median and worst gradient relative L2
and cosine, running statistics.  If the GPU figures are of the same size, the discrepancy is the fp16 roundings amplified by the train-mode
BatchNorm chain (DESIGN §2), not a kernel.

    python tools/inception_train_error_budget.py 4 107 139        # batch, H, W (runs on cuda:0 when there is one, else on the CPU)

Prints one JSON line; writes nothing.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import inception_oracle as I  # noqa: E402
import inception_train_oracle as T  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

SCALE = 1024.0      # b200.train_engine.InceptionTrainer's loss scale


def budget(b, h, w, seed=0, image_seed=12, device=None):
    device = device or ('cuda' if torch.cuda.is_available() else 'cpu')
    sd = I.make_inception_state_dict(seed)
    x = O.synth_images(b, h, w, seed=image_seed)
    f_ref, _, g_ref, s_ref = T.train_step(sd, x, device=device)
    f16, _, g16, s16 = T.train_step(sd, x, rnd=T.Rounding(SCALE), device=device)
    return T.step_errors(f16, g16, s16, f_ref, g_ref, s_ref, sorted(g_ref))


def main():
    b, h, w = (int(v) for v in sys.argv[1:4]) if len(sys.argv) > 3 else (4, 107, 139)
    torch.set_num_threads(8)
    print(json.dumps(dict(batch=b, size=[h, w], scale=SCALE, **budget(b, h, w))))


if __name__ == '__main__':
    main()
