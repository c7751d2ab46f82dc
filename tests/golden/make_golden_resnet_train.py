#!/usr/bin/env python
"""Golden fixture for ONE TRAINING STEP of the ResNet plugin, produced by EXECUTING the reference: its own `model.resnet.resnet18`
(BasicBlock) and `resnet50` (Bottleneck) in train() mode (batch-statistics BatchNorm, momentum 0.1; model/resnet.py:28-142), `model.Inference`
decode, `model.loss` (under the torch-0.3.1 shims of make_golden_loss.py), the hparam-weighted sum (train.py:348-349) and torch autograd.

Stored per net (resnet18: 4 x 3 x 128 x 128, resnet50: 2 x 3 x 64 x 64): the five loss terms, for every parameter the gradient's L2 norm and its
first 16 elements, the full gradient of tensors with <= 2048 elements, and the BatchNorm running statistics after the step.  Weights are
regenerated from the oracle's seed (oracle.yolo2_oracle.make_resnet_state_dict); only the reference's outputs are stored.

    python tests/golden/make_golden_resnet_train.py     # build container only (needs /root/reference)
"""
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
import resnet_train_oracle as RT  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

# (net, batch, size, image seed, target seed)
CASES = (('resnet18', 4, 128, 40, 41), ('resnet50', 2, 64, 42, 43))


def run(model, fns, config, anchors, name, b, size, seed_x, seed_t):
    import model.resnet
    sd = O.make_resnet_state_dict(name, seed=0)
    dnn = getattr(model.resnet, name)(model.ConfigChannels(config), anchors, 20)
    res = dnn.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    dnn.train()
    s = size // 32
    x = O.synth_images(b, size, size, seed=seed_x)
    data = O.norm_data(O.synth_targets(b, size, size, slots=6, seed=seed_t), size, size, s, s)
    inference = model.Inference(config, dnn, anchors)
    inference.train()
    pred = model._inference(inference, x)
    losses, _ = fns['loss'](anchors, data, pred, 0.6)
    total = sum(losses[k] * O.HPARAM_DEFAULT[k] for k in losses)
    dnn.zero_grad()
    total.backward()
    # the restatement must agree with the executed reference to fp32 rounding
    f = RT.resnet_train_forward(sd, x, name)
    err = ((f - pred['feature'].detach()).norm() / pred['feature'].detach().norm()).item()
    assert err < 1e-5, (name, err)
    out = {}
    for k, v in losses.items():
        out['%s_loss_%s' % (name, k)] = np.float64(v.item())
    for pname, p in dnn.named_parameters():
        gr = p.grad.detach()
        out['%s_gnorm_%s' % (name, pname)] = np.float64(gr.double().norm().item())
        out['%s_ghead_%s' % (name, pname)] = gr.flatten()[:16].numpy()
        if gr.numel() <= 2048:
            out['%s_gfull_%s' % (name, pname)] = gr.numpy()
    for bname, buf in dnn.named_buffers():
        if 'running' in bname:
            out['%s_buf_%s' % (name, bname)] = buf.detach().numpy()
    return out


def main():
    model, utils, detect = G.import_reference()
    if not hasattr(nn.init, 'kaiming_normal'):
        nn.init.kaiming_normal = nn.init.kaiming_normal_
    shim = L.Torch031('torch')
    fns = {}
    for fname in ('iou_match', 'fit_positive', 'fill_norm', 'square', 'loss'):
        f = getattr(model, fname)
        g = dict(f.__globals__)
        g['torch'] = shim
        fns[fname] = types.FunctionType(f.__code__, g, fname, f.__defaults__, f.__closure__)
    for f in fns.values():
        f.__globals__.update(fns)
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    anchors = O.anchors_yolo_voc()
    out = {}
    for case in CASES:
        out.update(run(model, fns, config, anchors, *case))
    path = os.path.join(HERE, 'resnet_train.npz')
    np.savez_compressed(path, **out)
    print('resnet_train.npz %.1f KB' % (os.path.getsize(path) / 1024), {k: float(v) for k, v in out.items() if '_loss_' in k})


if __name__ == '__main__':
    main()
