#!/usr/bin/env python
"""Error budget of one DenseNet TRAINING step under the GPU path's fp16 storage, in float64 arithmetic with only those roundings added
(tests/densenet_train_oracle.py, `rnd = Rounding(scale)`: conv weights -> fp16 except conv0's, every stored activation, raw conv output and
pooled tensor -> fp16, every stored gradient -> fp16 at the trainer's loss scale).  The step (train-mode forward, the synthetic loss
sum(feature * R), autograd backward) is compared with the exact float64 step on the same batch, as tests/test_densenet_train.py compares
the GPU step: feature, median and worst gradient relative L2 and cosine, running statistics.

    python tools/densenet_train_error_budget.py densenet121 2 64 96     # network, batch, H, W (cuda:0 when there is one, else the CPU)

Prints one JSON line; writes nothing.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'yolo2-pytorch_b200')]
import densenet_oracle as D  # noqa: E402
import densenet_train_oracle as T  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402


def scale():
    from b200 import train_engine
    return train_engine.DenseNetTrainer.GRAD_SCALE


def budget(name, b, h, w, seed=0, image_seed=4, device=None):
    """(errors of the rounded step against the exact one, the rounded step, the exact step)."""
    device = device or ('cuda' if torch.cuda.is_available() else 'cpu')
    sd = D.make_densenet_state_dict(name, seed)
    x = O.synth_images(b, h, w, seed=image_seed)
    ref = T.step(sd, x, name=name, device=device)
    got = T.step(sd, x, name=name, rnd=T.Rounding(scale()), device=device)
    errs = T.step_errors(got[1], got[2], got[3], ref[1], ref[2], ref[3], sorted(ref[2]))
    return errs, got, ref


def main():
    args = sys.argv[1:]
    name = args[0] if args else 'densenet121'
    b, h, w = (int(v) for v in args[1:4]) if len(args) >= 4 else (2, 64, 96)
    torch.set_num_threads(8)
    print(json.dumps(dict(network=name, batch=b, size=[h, w], scale=scale(), **budget(name, b, h, w)[0])))


if __name__ == '__main__':
    main()
