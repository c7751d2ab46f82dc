#!/usr/bin/env python
"""Golden fixture for training the DenseNet plugin, produced by EXECUTING one train()-mode step of the reference's `model.densenet.densenet121`
(model/densenet.py over torchvision's _DenseLayer / _Transition) on CPU with the deterministic synthetic weights of tests/densenet_oracle.py:

    python tests/golden/make_golden_densenet_train.py        # build container only (needs the reference checkout)

The step is batch 2 at 64x96 (non-square) on the loss sum(feature * R) (densenet_train_oracle.loss_weights).  Stores the loss, every
parameter gradient's norm and first 16 elements, and every running statistic after the step.  The reference is imported with the shims of
make_golden_densenet.py; nothing is copied from it.  Asserts that the restatement in densenet_train_oracle.py agrees: loss within 1e-5,
gradient norms within 1e-4, running statistics within 1e-5 (relative)."""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
import densenet_oracle as D  # noqa: E402
import densenet_train_oracle as T  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

NAME = 'densenet121'
STEP = (2, 64, 96, 4)      # (batch, H, W, image seed)
HEAD = 16


def main():
    model, _, _ = G.import_reference()
    import torchvision.models.densenet as tvd
    if not hasattr(tvd, 'model_urls'):
        tvd.model_urls = {}
    if not hasattr(nn.init, 'kaiming_normal'):
        nn.init.kaiming_normal = nn.init.kaiming_normal_
    import model.densenet
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    sd = D.make_densenet_state_dict(NAME, 0)
    net = getattr(model.densenet, NAME)(model.ConfigChannels(config), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    b, h, w, seed = STEP
    x = O.synth_images(b, h, w, seed=seed)
    net.train()
    f = net(x)
    loss = (f * T.loss_weights(tuple(f.shape))).sum()
    loss.backward()
    o_loss, _, o_grads, o_stats = T.step(sd, x, name=NAME, dtype=torch.float32)
    assert abs(o_loss.item() - loss.item()) <= 1e-5 * abs(loss.item()), (o_loss.item(), loss.item())
    rec = {'image_seed': np.int64(seed), 'shape': np.array([b, h, w]), 'loss': np.float64(loss.item())}
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
    print('loss %.6f, worst gradient-norm difference of the restatement %.2e' % (loss.item(), worst))
    path = os.path.join(HERE, 'densenet_train.npz')
    np.savez_compressed(path, **rec)
    print('densenet_train.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
