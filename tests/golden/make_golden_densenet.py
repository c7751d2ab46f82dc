#!/usr/bin/env python
"""Golden fixture for the DenseNet plugin, produced by EXECUTING the reference's `model.densenet` (model/densenet.py:29-117 over
torchvision's _DenseBlock / _Transition) on CPU with the deterministic synthetic weights of tests/densenet_oracle.py:

    python tests/golden/make_golden_densenet.py        # build container only (needs the reference checkout)

Stores the densenet121 head at 64x64 and 416x416, the densenet169 / 201 heads at 64x64, every dense block's and transition's output of
densenet121 at 64x64 (denseblock4 is the norm5 input), and the state_dict key names and shapes of all four constructors.  The reference is
imported with make_golden.py's in-memory shims plus two more: `torchvision.models.densenet.model_urls` (which current torchvision removed)
and the `nn.init.kaiming_normal` alias; nothing is copied.  Asserts that the restatement in densenet_oracle.py agrees to 1e-5."""
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
from oracle import yolo2_oracle as O  # noqa: E402


def run(model, config, anchors, name, sizes, acts_at):
    import model.densenet
    sd = D.make_densenet_state_dict(name, seed=0)
    net = getattr(model.densenet, name)(model.ConfigChannels(config), anchors, 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    net.eval()
    outs = {}
    hooks = []
    for mname, m in net.features.named_children():
        if mname.startswith('denseblock') or mname.startswith('transition'):
            hooks.append(m.register_forward_hook(lambda mod, inp, out, key=mname: outs.__setitem__(key, out.detach().clone())))
    rec = {}
    with torch.no_grad():
        for size, seed in sizes:
            x = O.synth_images(1, size, size, seed=seed)
            f = net(x)
            rec['%s_feature%d' % (name, size)] = f.numpy()
            if size == acts_at:
                rec.update({'%s_act_%s' % (name, k): v.numpy() for k, v in outs.items()})
            got = {}
            o = D.densenet_forward(sd, x, name, collect=got)
            err = ((o - f).norm() / f.norm()).item()
            assert err < 1e-5, (name, size, err)
            if size == acts_at:
                for k, v in outs.items():
                    e = ((got[k] - v).norm() / v.norm()).item()
                    assert e < 1e-5, (name, k, e)
    for h in hooks:
        h.remove()
    return rec


def main():
    model, utils, detect = G.import_reference()
    import torchvision.models.densenet as tvd
    if not hasattr(tvd, 'model_urls'):
        tvd.model_urls = {}
    if not hasattr(nn.init, 'kaiming_normal'):
        nn.init.kaiming_normal = nn.init.kaiming_normal_
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    anchors = O.anchors_yolo_voc()
    rec = {}
    rec.update(run(model, config, anchors, 'densenet121', [(64, 10), (416, 0)], 64))
    rec.update(run(model, config, anchors, 'densenet169', [(64, 10)], None))
    rec.update(run(model, config, anchors, 'densenet201', [(64, 10)], None))
    import model.densenet
    for name in ('densenet121', 'densenet169', 'densenet201', 'densenet161'):
        sd = getattr(model.densenet, name)(model.ConfigChannels(config), anchors, 20).state_dict()
        rec['%s_keys' % name] = np.array(list(sd.keys()))
        rec['%s_shapes' % name] = np.array([','.join(str(d) for d in v.shape) for v in sd.values()])
    path = os.path.join(HERE, 'densenet.npz')
    np.savez_compressed(path, **rec)
    print('densenet.npz %.1f KB' % (os.path.getsize(path) / 1024), sorted(rec)[:6])


if __name__ == '__main__':
    main()
