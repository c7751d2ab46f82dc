#!/usr/bin/env python
"""Golden fixture for the Inception-v4 plugin, produced by EXECUTING the reference's `model.inception4.Inception4` on CPU with the deterministic
synthetic weights of tests/inception4_oracle.py:

    python tests/golden/make_golden_inception4.py        # build container only (needs the reference checkout)

Stores the state_dict key names and shapes with BatchNorm on and off; the head at 75x75, 107x139, 416x416 and 320x608; at 107x139 the output
of one block of each kind (features.3 Mixed_3a, 4 Mixed_4a, 5 Mixed_5a, 6 the first Inception_A, 10 Reduction_A, 11 the first Inception_B,
18 Reduction_B, 21 the last Inception_C; the large ones as a seeded sample, oracle/yolo2_oracle.py:store_sampled); and the head at 107x139 with
BatchNorm disabled, with ratio = 0.5 and with a channel-pruned checkpoint built as ConfigChannels(config, state_dict) (widths not multiples of
8, features.0 with 29 filters).  The reference is imported with make_golden.py's in-memory shims plus one more: the reference imports
`pretrainedmodels.models.inceptionv4.pretrained_settings` at module level, so an empty module of that name is registered first (it is only
read when `[model] pretrained` is on).  Nothing is copied from the reference.  Asserts that the restatement in inception4_oracle.py agrees to
1e-5."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
import inception4_oracle as I  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

SIZES = ((75, 75, 1), (107, 139, 2), (416, 416, 0), (320, 608, 3))   # (H, W, seed of the synthetic image)
ACTS_AT = (107, 139)
BLOCKS = (3, 4, 5, 6, 10, 11, 18, 21)
VARIANT_SEED = 7                                                    # the image of the BatchNorm-off / ratio / pruned heads at 107x139


def shim_pretrainedmodels():
    pkg = types.ModuleType('pretrainedmodels')
    models = types.ModuleType('pretrainedmodels.models')
    v4 = types.ModuleType('pretrainedmodels.models.inceptionv4')
    v4.pretrained_settings = {}
    pkg.models, models.inceptionv4 = models, v4
    sys.modules.update({'pretrainedmodels': pkg, 'pretrainedmodels.models': models, 'pretrainedmodels.models.inceptionv4': v4})


def construct(model, bn, ratio=1, state_dict=None):
    import model.inception4
    config = G.make_config(1)
    config.read_dict({'batch_norm': {'enable': str(int(bn))}, 'model': {'pretrained': '0'}})
    net = model.inception4.Inception4(model.ConfigChannels(config, state_dict), O.anchors_yolo_voc(), 20, ratio=ratio)
    return net


def load(net, sd):
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net.eval()


def check(o, f, tag):
    err = ((o - f).norm() / f.norm()).item()
    assert err < 1e-5, (tag, err)
    print('%-24s %s, restatement %.2e' % (tag, tuple(f.shape), err))


def main():
    shim_pretrainedmodels()
    model, _, _ = G.import_reference()
    rec = {}
    for bn, tag in ((True, ''), (False, '_nobn')):
        sd_ref = construct(model, bn).state_dict()
        rec['keys' + tag] = np.array(list(sd_ref.keys()))
        rec['shapes' + tag] = np.array([','.join(str(d) for d in v.shape) for v in sd_ref.values()])
        own = I.make_state_dict(0, bn=bn)
        assert [k for k in sd_ref if not k.endswith('num_batches_tracked')] == list(own.keys()), tag
        assert all(tuple(sd_ref[k].shape) == tuple(v.shape) for k, v in own.items()), tag
    sd = I.make_state_dict(0)
    net = load(construct(model, True), sd)
    outs = {}
    hooks = [net.features[i].register_forward_hook(lambda mod, inp, out, key=i: outs.__setitem__(key, out.detach().clone())) for i in BLOCKS]
    with torch.no_grad():
        for h, w, seed in SIZES:
            outs.clear()
            x = O.synth_images(1, h, w, seed=seed)
            f = net(x)
            rec['feature_%dx%d' % (h, w)] = f.numpy()
            got = {}
            check(I.inception4_forward(sd, x, collect=got), f, 'head %dx%d' % (h, w))
            if (h, w) == ACTS_AT:
                for k in BLOCKS:
                    O.store_sampled(rec, 'act_%d' % k, outs[k].numpy())
                    check(got[k], outs[k], 'features.%d' % k)
    for hk in hooks:
        hk.remove()
    # variants at 107 x 139: BatchNorm disabled, ratio 0.5, a pruned checkpoint
    x = O.synth_images(1, 107, 139, seed=VARIANT_SEED)
    pruned_sd = I.make_state_dict(3, pruned=I.pruned_widths())
    for tag, bn, ratio, sd_v, ref_sd in (('nobn', False, 1, I.make_state_dict(1, bn=False), None),
                                         ('ratio05', True, 0.5, I.make_state_dict(2, ratio=0.5), None),
                                         ('pruned', True, 1, pruned_sd, pruned_sd)):
        net = load(construct(model, bn, ratio, ref_sd), sd_v)
        with torch.no_grad():
            f = net(x)
            check(I.inception4_forward(sd_v, x), f, tag)
        rec['feature_' + tag] = f.numpy()
        rec['shapes_' + tag] = np.array([','.join(str(d) for d in v.shape) for k, v in net.state_dict().items()
                                         if not k.endswith('num_batches_tracked')])
    path = os.path.join(HERE, 'inception4.npz')
    np.savez_compressed(path, **rec)
    print('inception4.npz %.1f KB, %d / %d state_dict entries' % (os.path.getsize(path) / 1024, len(rec['keys']), len(rec['keys_nobn'])))


if __name__ == '__main__':
    main()
