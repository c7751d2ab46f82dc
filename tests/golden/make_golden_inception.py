#!/usr/bin/env python
"""Golden fixture for the Inception-v3 plugin, produced by EXECUTING the reference's `model.inception3.Inception3` (model/inception3.py:29-118
over torchvision's BasicConv2d / InceptionA-E) on CPU with the deterministic synthetic weights of tests/inception_oracle.py:

    python tests/golden/make_golden_inception.py        # build container only (needs the reference checkout)

Stores the head at 75x75, 107x139, 416x416 and 320x608, both stem max-pools and every Mixed_* output at 107x139, and the state_dict key names
and shapes.  The reference is imported with make_golden.py's in-memory shims plus one more: its initialiser copies a 1-D tensor of truncated
normal draws into each 4-D conv weight (`m.weight.data.copy_(torch.Tensor(X.rvs(numel)))`, model/inception3.py:58-59), which torch 0.3.1
allowed and current torch refuses, so `Tensor.copy_` reshapes its source when the element counts match while the reference is constructed.
Nothing is copied from the reference.  Asserts that the restatement in inception_oracle.py agrees to 1e-5."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
import inception_oracle as I  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

SIZES = ((75, 75, 1), (107, 139, 2), (416, 416, 0), (320, 608, 3))   # (H, W, seed of the synthetic image)
ACTS_AT = (107, 139)


def construct(model, config, anchors):
    import model.inception3
    orig = torch.Tensor.copy_

    def copy_(self, src, non_blocking=False):
        if isinstance(src, torch.Tensor) and src.shape != self.shape and src.numel() == self.numel():
            src = src.reshape(self.shape)
        return orig(self, src, non_blocking)
    torch.Tensor.copy_ = copy_
    try:
        return model.inception3.Inception3(model.ConfigChannels(config), anchors, 20)
    finally:
        torch.Tensor.copy_ = orig


def main():
    model, utils, detect = G.import_reference()
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    anchors = O.anchors_yolo_voc()
    net = construct(model, config, anchors)
    rec = {}
    sd_ref = net.state_dict()
    rec['keys'] = np.array(list(sd_ref.keys()))
    rec['shapes'] = np.array([','.join(str(d) for d in v.shape) for v in sd_ref.values()])
    sd = I.make_inception_state_dict(seed=0)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    net.eval()
    outs = {}
    names = ('Mixed_5b', 'Mixed_5c', 'Mixed_5d', 'Mixed_6a', 'Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e', 'Mixed_7a', 'Mixed_7b', 'Mixed_7c')
    hooks = [getattr(net, n).register_forward_hook(lambda mod, inp, out, key=n: outs.__setitem__(key, out.detach().clone())) for n in names]
    # the stem pools are functional calls in the reference's forward: the inputs of Conv2d_3b_1x1 and Mixed_5b
    hooks.append(net.Conv2d_3b_1x1.register_forward_hook(lambda mod, inp, out: outs.__setitem__('pool1', inp[0].detach().clone())))
    hooks.append(net.Mixed_5b.register_forward_hook(lambda mod, inp, out: outs.__setitem__('pool2', inp[0].detach().clone())))
    with torch.no_grad():
        for h, w, seed in SIZES:
            outs.clear()
            x = O.synth_images(1, h, w, seed=seed)
            f = net(x)
            rec['feature_%dx%d' % (h, w)] = f.numpy()
            got = {}
            o = I.inception_forward(sd, x, collect=got)
            err = ((o - f).norm() / f.norm()).item()
            assert err < 1e-5, (h, w, err)
            print('%dx%d head %s, restatement %.2e' % (h, w, tuple(f.shape), err))
            if (h, w) == ACTS_AT:
                for k, v in outs.items():
                    rec['act_' + k] = v.numpy()
                    e = ((got[k] - v).norm() / v.norm()).item()
                    assert e < 1e-5, (k, e)
    for hk in hooks:
        hk.remove()
    path = os.path.join(HERE, 'inception.npz')
    np.savez_compressed(path, **rec)
    print('inception.npz %.1f KB, %d state_dict entries' % (os.path.getsize(path) / 1024, len(rec['keys'])))


if __name__ == '__main__':
    main()
