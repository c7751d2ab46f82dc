#!/usr/bin/env python
"""Golden fixture for training the Inception-v4 plugin, produced by EXECUTING one train()-mode step of the reference's
`model.inception4.Inception4` on CPU with the deterministic synthetic weights of tests/inception4_oracle.py, with BatchNorm on and off:

    python tests/golden/make_golden_inception4_train.py        # build container only (needs the reference checkout)

The step is batch 2 at 107x139 (odd, non-square) on the loss sum(feature * R) (inception_train_oracle.loss_weights).  Stores, per BatchNorm
mode (tag 'bn' on, 'nobn' off), the loss, every parameter gradient's norm and first 16 elements, and every running statistic after the step.
The reference is constructed as make_golden_inception4.py does (the same `pretrainedmodels` shim).  Nothing is copied from the reference.
Asserts that the restatement in inception4_train_oracle.py agrees: loss within 1e-5, gradient norms within 1e-4, running statistics within
1e-5 (relative)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
import make_golden_inception4 as MGI4  # noqa: E402
import inception4_oracle as I  # noqa: E402
import inception4_train_oracle as T4  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

STEP = (2, 107, 139, 11)      # (batch, H, W, image seed)
HEAD = 16
SEEDS = {'bn': 0, 'nobn': 1}  # state_dict seed per BatchNorm mode


def main():
    MGI4.shim_pretrainedmodels()
    model, _, _ = G.import_reference()
    b, h, w, seed = STEP
    x = O.synth_images(b, h, w, seed=seed)
    rec = {'image_seed': np.int64(seed), 'shape': np.array([b, h, w])}
    for tag, sd_seed in SEEDS.items():
        bn = tag == 'bn'
        sd = I.make_state_dict(sd_seed, bn=bn)
        net = MGI4.construct(model, bn)
        res = net.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
        net.train()
        f = net(x)
        loss = (f * T4.loss_weights(tuple(f.shape))).sum()
        loss.backward()
        _, o_loss, o_grads, o_stats = T4.train_step(sd, x, dtype=torch.float32)
        assert abs(o_loss.item() - loss.item()) <= 1e-5 * abs(loss.item()), (tag, o_loss.item(), loss.item())
        rec['loss_' + tag] = np.float64(loss.item())
        rec['seed_' + tag] = np.int64(sd_seed)
        worst = 0.0
        for k, p in net.named_parameters():
            n = p.grad.norm().item()
            rec['gnorm_%s_%s' % (tag, k)] = np.float64(n)
            rec['ghead_%s_%s' % (tag, k)] = p.grad.flatten()[:HEAD].numpy()
            e = abs(o_grads[k].norm().item() - n) / max(n, 1e-30)
            assert e <= 1e-4, (tag, k, e)
            worst = max(worst, e)
        for k, v in net.state_dict().items():
            if 'running' in k:
                rec['stat_%s_%s' % (tag, k)] = v.numpy()
                assert (o_stats[k] - v).abs().max().item() <= 1e-5 * max(v.abs().max().item(), 1.0), (tag, k)
        print('BatchNorm %s: loss %.6f, worst gradient-norm difference of the restatement %.2e' % ('on' if bn else 'off', loss.item(), worst))
    path = os.path.join(HERE, 'inception4_train.npz')
    np.savez_compressed(path, **rec)
    print('inception4_train.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
