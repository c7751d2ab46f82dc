#!/usr/bin/env python
"""Golden fixture for the VGG plugin, produced by EXECUTING the reference's `model/vgg.py` on CPU with the deterministic synthetic weights
of tests/vgg_oracle.py:

    python tests/golden/make_golden_vgg.py        # build container only (needs the reference checkout)

Stores the state_dict key names and shapes of all eight constructors; the heads of vgg11, vgg11_bn, vgg16 and vgg19_bn at 64x64, 96x160
and 416x416; every MaxPool2d output of vgg16_bn at 96x160 (the large ones as a seeded sample, oracle/yolo2_oracle.py:store_sampled); and the
head of a channel-pruned vgg11_bn (ConfigChannels(config, state_dict), widths not multiples of 32, features.0 with 48 filters) at 96x160;
and one train-mode step of vgg11 and vgg11_bn at batch 2, 64x96, on the loss sum(feature * R) (vgg_oracle.loss_weights): the loss, every
parameter gradient's norm and first 16 elements, and the running statistics after the step.
The reference is written against torchvision 0.2; three in-memory shims on `torchvision.models.vgg` let it import and construct under the
installed torchvision (nothing is copied from the reference):
  * `cfg = cfgs`: the configuration table was renamed;
  * `model_urls = {}`: imported at module level, read only with `[model] pretrained = 1`;
  * `VGG._initialize_weights`: torchvision 0.2's body (conv weights N(0, 2 / (kh * kw * out_channels)), conv biases 0, BatchNorm weight 1
    and bias 0), which the reference's VGG.__init__ calls and current torchvision no longer has.
Asserts that the restatement in vgg_oracle.py agrees to 1e-5."""
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
import vgg_oracle as V  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402

HEADS = ('vgg11', 'vgg11_bn', 'vgg16', 'vgg19_bn')
SIZES = ((64, 64, 1), (96, 160, 2), (416, 416, 0))   # (H, W, seed of the synthetic image)
POOLS = ('vgg16_bn', 96, 160, 2)
PRUNED = ('vgg11_bn', 96, 160, 5)                     # (constructor, H, W, image seed); state dict seed 3
TRAIN = (2, 64, 96, 9)                                # (batch, H, W, image seed) of the train-mode step of vgg11 and vgg11_bn


def _initialize_weights(self):
    for m in self.modules():
        if isinstance(m, nn.Conv2d):
            n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
            m.weight.data.normal_(0, math.sqrt(2. / n))
            if m.bias is not None:
                m.bias.data.zero_()
        elif isinstance(m, nn.BatchNorm2d):
            m.weight.data.fill_(1)
            m.bias.data.zero_()
        elif isinstance(m, nn.Linear):
            m.weight.data.normal_(0, 0.01)
            m.bias.data.zero_()


def shim_torchvision():
    import torchvision.models.vgg as tv
    tv.cfg = tv.cfgs
    tv.model_urls = {}
    tv.VGG._initialize_weights = _initialize_weights


def construct(name, state_dict=None):
    import model.vgg
    config = G.make_config(1)
    config.read_dict({'model': {'pretrained': '0'}})
    return getattr(model.vgg, name)(model.ConfigChannels(config, state_dict), O.anchors_yolo_voc(), 20)


def load(net, sd):
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net.eval()


def check(o, f, tag):
    err = ((o - f).norm() / f.norm()).item()
    assert err < 1e-5, (tag, err)
    print('%-28s %s, restatement %.2e' % (tag, tuple(f.shape), err))


def main():
    shim_torchvision()
    G.import_reference()
    rec = {}
    for name in V.NAMES:
        sd_ref = construct(name).state_dict()
        rec['keys_' + name] = np.array(list(sd_ref.keys()))
        rec['shapes_' + name] = np.array([','.join(str(d) for d in v.shape) for v in sd_ref.values()])
        own = V.make_state_dict(name)
        assert [k for k in sd_ref if not k.endswith('num_batches_tracked')] == list(own.keys()), name
        assert all(tuple(sd_ref[k].shape) == tuple(v.shape) for k, v in own.items()), name
    with torch.no_grad():
        for name in HEADS:
            sd = V.make_state_dict(name)
            net = load(construct(name), sd)
            for h, w, seed in SIZES:
                x = O.synth_images(1, h, w, seed=seed)
                f = net(x)
                rec['feature_%s_%dx%d' % (name, h, w)] = f.numpy()
                check(V.vgg_forward(sd, x, name), f, '%s %dx%d' % (name, h, w))
        name, h, w, seed = POOLS
        sd = V.make_state_dict(name)
        net = load(construct(name), sd)
        outs = {}
        idx = [i for kind, i, _ in V.layers(name) if kind == 'pool']
        hooks = [net.features[i].register_forward_hook(lambda mod, inp, out, key=i: outs.__setitem__(key, out.detach().clone())) for i in idx]
        x = O.synth_images(1, h, w, seed=seed)
        net(x)
        got = {}
        V.vgg_forward(sd, x, name, collect=got)
        for i in idx:
            O.store_sampled(rec, 'pool_%d' % i, outs[i].numpy())
            check(got[i], outs[i], 'features.%d' % i)
        for hk in hooks:
            hk.remove()
        name, h, w, seed = PRUNED
        pruned = V.pruned_widths()
        sd = V.make_state_dict(name, seed=3, pruned=pruned)
        net = load(construct(name, sd), sd)
        x = O.synth_images(1, h, w, seed=seed)
        f = net(x)
        check(V.vgg_forward(sd, x, name, pruned=pruned), f, 'pruned ' + name)
        rec['feature_pruned'] = f.numpy()
        rec['shapes_pruned'] = np.array([','.join(str(d) for d in v.shape) for k, v in net.state_dict().items()
                                         if not k.endswith('num_batches_tracked')])
    b, h, w, seed = TRAIN
    x = O.synth_images(b, h, w, seed=seed)
    for name in ('vgg11', 'vgg11_bn'):
        sd = V.make_state_dict(name, seed=4)
        net = construct(name)
        net.load_state_dict(sd, strict=False)
        net.train()
        f = net(x)
        loss = (f * V.loss_weights(tuple(f.shape))).sum()
        loss.backward()
        o_loss, o_grads, o_stats = V.train_step(sd, x, name, dtype=torch.float32)
        assert abs(o_loss.item() - loss.item()) <= 1e-5 * abs(loss.item()), (name, o_loss.item(), loss.item())
        rec['train_%s_loss' % name] = np.float64(loss.item())
        for k, p in net.named_parameters():
            rec['train_%s_gnorm_%s' % (name, k)] = np.float64(p.grad.norm().item())
            rec['train_%s_ghead_%s' % (name, k)] = p.grad.flatten()[:16].numpy()
            check_grad = (o_grads[k] - p.grad).norm().item() / max(p.grad.norm().item(), 1e-30)
            assert check_grad < 1e-4 or p.grad.norm().item() < 1e-6, (name, k, check_grad)
        for k, v in net.state_dict().items():
            if 'running' in k:
                rec['train_%s_%s' % (name, k)] = v.numpy()
                assert (o_stats[k] - v).abs().max().item() <= 1e-5 * max(v.abs().max().item(), 1.0), (name, k)
        print('train step %-10s loss %.6f' % (name, loss.item()))
    path = os.path.join(HERE, 'vgg.npz')
    np.savez_compressed(path, **rec)
    print('vgg.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
