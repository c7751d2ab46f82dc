#!/usr/bin/env python
"""Golden fixture for the deep ResNet constructors, produced by EXECUTING the reference's own `model.resnet.resnet101` ([3, 4, 23, 3]) and
`resnet152` ([3, 8, 36, 3]) on CPU (model/resnet.py:200-224) with the oracle's deterministic synthetic weights
(oracle.yolo2_oracle.make_resnet_state_dict):

    python tests/golden/make_golden_resnet_deep.py        # build container only (needs /root/reference)

Stores, in resnet_deep.npz:
  - the head feature at 64x64 for both depths and at 416x416 for resnet101;
  - every resnet101 block output at 64x64 (eval mode), as its L2 norm (fp64) and its first 64 elements (`resnet101_blocks` names the
    rows of `resnet101_actnorm` / `resnet101_acthead`); the whole tensor is asserted here to agree with the restatement to 1e-5;
  - the state_dict keys and shapes of both constructors;
  - one train() step of resnet101 at 2 x 3 x 64 x 64, the content of make_golden_resnet_train.py with its per-tensor entries stacked
    (each npz entry costs a zip header, which would otherwise outweigh the data): the five loss terms; every parameter's gradient norm and
    first 16 elements (`resnet101_params` names the rows of `resnet101_gnorm` / `resnet101_ghead`); the stem's, layer1's and the head's
    small gradients (<= 2048 elements) in full (`resnet101_gfull_<name>`); the running statistics after the step in full for the stem and
    layer1 (`resnet101_buf_<name>`), and for every BatchNorm the L2 norms and first 16 elements of its running mean and variance
    (`resnet101_bns` names the rows of `resnet101_bufnorm` [., 2] / `resnet101_bufhead` [., 2, 16]).
The fp32 restatements (oracle.yolo2_oracle.resnet_forward and tests/resnet_train_oracle.py, given the deep layer counts by
tests/resnet_deep_oracle.py) are asserted to agree with every stored head to 1e-5.  No weights are stored, and nothing is stored in full
beyond what the CPU test needs: the file stays small.  The reference is imported with make_golden.py's in-memory shims plus the `nn.init.kaiming_normal` alias of
make_golden_resnet.py; nothing is copied."""
import os
import sys
import types
import warnings

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
warnings.filterwarnings('ignore')
import make_golden as G  # noqa: E402
import make_golden_loss as L  # noqa: E402
import make_golden_resnet as GR  # noqa: E402
import make_golden_resnet_train as GT  # noqa: E402
import resnet_deep_oracle  # noqa: E402,F401  (resnet101 / 152 in the oracle's ResNet table)
from oracle import yolo2_oracle as O  # noqa: E402

NETS = ('resnet101', 'resnet152')
TRAIN_CASE = ('resnet101', 2, 64, 42, 43)          # (net, batch, size, image seed, target seed)
FULL = ('bn1.', 'conv.', 'layer1.')                 # parameters / BatchNorms stored in full (the rest as norm and first elements)


def shapes(model, config, anchors, name):
    import model.resnet
    net = getattr(model.resnet, name)(model.ConfigChannels(config), anchors, 20)
    sd = net.state_dict()
    return {'%s_keys' % name: np.array(list(sd)), '%s_shapes' % name: np.array([';'.join(str(d) for d in v.shape) for v in sd.values()])}


def main():
    model, utils, detect = G.import_reference()
    if not hasattr(nn.init, 'kaiming_normal'):
        nn.init.kaiming_normal = nn.init.kaiming_normal_
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    anchors = O.anchors_yolo_voc()
    rec = {}
    rec.update(GR.run(model, config, anchors, 'resnet101', [(64, 10), (416, 0)], 64))
    rec.update(GR.run(model, config, anchors, 'resnet152', [(64, 10)], None))
    # block outputs: checked here against the restatement to 1e-5 in full, stored as norm and first elements
    collect, blocks = {}, []
    with torch.no_grad():
        O.resnet_forward(O.make_resnet_state_dict('resnet101', seed=0), O.synth_images(1, 64, 64, seed=10), 'resnet101', collect=collect)
    for key in [k for k in rec if k.startswith('resnet101_act_')]:
        ref, got = rec.pop(key), collect[key[len('resnet101_act_'):]].numpy()
        err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
        assert err < 1e-5, (key, err)
        blocks.append((key[len('resnet101_act_'):], np.linalg.norm(ref.astype(np.float64)), ref.flatten()[:64]))
    rec['resnet101_blocks'] = np.array([k for k, _, _ in blocks])
    rec['resnet101_actnorm'] = np.array([n for _, n, _ in blocks])
    rec['resnet101_acthead'] = np.stack([h for _, _, h in blocks])
    for name in NETS:
        rec.update(shapes(model, config, anchors, name))
    shim = L.Torch031('torch')
    fns = {}
    for fname in ('iou_match', 'fit_positive', 'fill_norm', 'square', 'loss'):
        f = getattr(model, fname)
        g = dict(f.__globals__)
        g['torch'] = shim
        fns[fname] = types.FunctionType(f.__code__, g, fname, f.__defaults__, f.__closure__)
    for f in fns.values():
        f.__globals__.update(fns)
    torch.set_num_threads(8)
    name = TRAIN_CASE[0]
    step = GT.run(model, fns, config, anchors, *TRAIN_CASE)
    params = [k[len(name + '_gnorm_'):] for k in step if k.startswith(name + '_gnorm_')]
    rec[name + '_params'] = np.array(params)
    rec[name + '_gnorm'] = np.array([step[name + '_gnorm_' + p] for p in params])
    rec[name + '_ghead'] = np.stack([step[name + '_ghead_' + p] for p in params])
    bns = [k[len(name + '_buf_'):-len('.running_mean')] for k in step if k.startswith(name + '_buf_') and k.endswith('.running_mean')]
    buf = [(step['%s_buf_%s.running_mean' % (name, b)], step['%s_buf_%s.running_var' % (name, b)]) for b in bns]
    rec[name + '_bns'] = np.array(bns)
    rec[name + '_bufnorm'] = np.array([[np.linalg.norm(m.astype(np.float64)), np.linalg.norm(v.astype(np.float64))] for m, v in buf])
    rec[name + '_bufhead'] = np.stack([np.stack([m[:16], v[:16]]) for m, v in buf])
    for key, v in step.items():
        if '_loss_' in key or (('_gfull_' in key or '_buf_' in key) and key.split('_', 2)[2].startswith(FULL)):
            rec[key] = v
    path = os.path.join(HERE, 'resnet_deep.npz')
    np.savez_compressed(path, **rec)
    print('resnet_deep.npz %.1f KB' % (os.path.getsize(path) / 1024), {k: float(v) for k, v in rec.items() if '_loss_' in k})


if __name__ == '__main__':
    main()
