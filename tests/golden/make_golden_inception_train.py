#!/usr/bin/env python
"""Golden fixture for training the Inception-v3 plugin, produced by EXECUTING one train()-mode step of the reference's
`model.inception3.Inception3` (model/inception3.py:29-118 over torchvision's BasicConv2d / InceptionA-E) on CPU with the deterministic
synthetic weights of tests/inception_oracle.py:

    python tests/golden/make_golden_inception_train.py        # build container only (needs the reference checkout)

The step is batch 2 at 107x139 (odd, non-square) on the loss sum(feature * R) (inception_train_oracle.loss_weights).  Stores the loss, every
parameter gradient's norm and first 16 elements, and every running statistic after the step.  The reference is constructed as
make_golden_inception.py does (the same shims).  Nothing is copied from the reference.  Asserts that the restatement in
inception_train_oracle.py agrees: loss within 1e-5, gradient norms within 1e-4, running statistics within 1e-5 (relative)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
import make_golden_inception as MGI  # noqa: E402
import inception_oracle as I  # noqa: E402
import inception_train_oracle as T  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

STEP = (2, 107, 139, 11)      # (batch, H, W, image seed)
HEAD = 16


def main():
    model, utils, detect = G.import_reference()
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    net = MGI.construct(model, config, O.anchors_yolo_voc())
    sd = I.make_inception_state_dict(seed=0)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    b, h, w, seed = STEP
    x = O.synth_images(b, h, w, seed=seed)
    net.train()
    f = net(x)
    loss = (f * T.loss_weights(tuple(f.shape))).sum()
    loss.backward()
    _, o_loss, o_grads, o_stats = T.train_step(sd, x, dtype=torch.float32)
    assert abs(o_loss.item() - loss.item()) <= 1e-5 * abs(loss.item()), (o_loss.item(), loss.item())
    rec = {'loss': np.float64(loss.item()), 'image_seed': np.int64(seed), 'shape': np.array([b, h, w])}
    worst = 0.0
    for k, p in net.named_parameters():
        n = p.grad.norm().item()
        rec['gnorm_' + k] = np.float64(n)
        rec['ghead_' + k] = p.grad.flatten()[:HEAD].numpy()
        e = abs(o_grads[k].norm().item() - n) / max(n, 1e-30)
        assert e <= 1e-4, (k, e)
        worst = max(worst, e)
    for k, v in net.state_dict().items():
        if 'running' in k:
            rec['stat_' + k] = v.numpy()
            assert (o_stats[k] - v).abs().max().item() <= 1e-5 * max(v.abs().max().item(), 1.0), k
    path = os.path.join(HERE, 'inception_train.npz')
    np.savez_compressed(path, **rec)
    print('loss %.6f, worst gradient-norm difference of the restatement %.2e' % (loss.item(), worst))
    print('inception_train.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
