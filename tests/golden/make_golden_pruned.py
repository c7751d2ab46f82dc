#!/usr/bin/env python
"""Golden fixture for channel-pruned Darknet-19 and Tiny YOLOv2, produced by EXECUTING the reference's `model.yolo2.Darknet` and `Tiny`
(model/yolo2.py:68-173) on CPU, rebuilt from the pruned checkpoint by the reference's own `model.ConfigChannels(config, state_dict)`:

    python tests/golden/make_golden_pruned.py          # build container only (needs /root/reference)

The pruned checkpoints are tests/pruned_oracle.py's: seeded, non-prefix kept subsets of the oracle's seed-0 weights, cascaded to each
consumer's input channels and through the reference's `Darknet.get_mapper(94)` for layers3.0, as the reference's pruner.py does.
`Darknet(ratio=0.75)` runs on the oracle's ratio-0.75 weights.  Stored: the kept index lists (not the weights) and the head features at
64x64 (seed 10) and 416x416 (seed 0).  The reference is imported with make_golden.py's in-memory shims; nothing is copied."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as G  # noqa: E402
from oracle import yolo2_oracle as O  # noqa: E402
import pruned_oracle as PO  # noqa: E402


def run(net, sd):
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    for k, v in sd.items():
        assert tuple(net.state_dict()[k].shape) == tuple(v.shape), k
    net.eval()
    with torch.no_grad():
        return net(O.synth_images(1, 64, 64, seed=10)), net(O.synth_images(1, 416, 416, seed=0))


def check_oracle(forward, sd, f64, f416):
    """The oracle's restatement (used by the GPU tests at other shapes) agrees with the executed reference."""
    with torch.no_grad():
        o64, o416 = forward(sd, O.synth_images(1, 64, 64, seed=10)), forward(sd, O.synth_images(1, 416, 416, seed=0))
    np.testing.assert_allclose(o64.numpy(), f64.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(o416.numpy(), f416.numpy(), rtol=1e-4, atol=1e-5)


def main():
    model, utils, detect = G.import_reference()
    config = G.make_config(1)
    anchors = O.anchors_yolo_voc()
    out = {}

    keep = PO.darknet_keep()
    full = model.yolo2.Darknet(model.ConfigChannels(config), anchors, 20)
    # layers3.0's input cascade through the reference's own reorg mapper
    c_pt = PO.darknet_widths()['passthrough']
    assert torch.equal(full.get_mapper(94)(keep['passthrough'], c_pt), PO.reorg_mapper(keep['passthrough'], c_pt))
    sd = PO.prune_darknet(O.make_state_dict(0), keep)
    net = model.yolo2.Darknet(model.ConfigChannels(config, sd), anchors, 20)
    f64, f416 = run(net, sd)
    check_oracle(O.darknet_forward, sd, f64, f416)
    out.update({'darknet_keep_' + k: v.numpy().astype(np.int32) for k, v in keep.items()})
    out.update(darknet_feature64=f64.numpy(), darknet_feature416=f416.numpy())

    sd = O.make_state_dict(0, ratio=0.75)
    net = model.yolo2.Darknet(model.ConfigChannels(config), anchors, 20, ratio=0.75)
    f64, f416 = run(net, sd)
    check_oracle(O.darknet_forward, sd, f64, f416)
    out.update(ratio075_feature64=f64.numpy(), ratio075_feature416=f416.numpy())

    keep = PO.tiny_keep()
    sd = PO.prune_tiny(O.make_tiny_state_dict(0), keep)
    net = model.yolo2.Tiny(model.ConfigChannels(config, sd), anchors, 20)
    f64, f416 = run(net, sd)
    check_oracle(O.tiny_forward, sd, f64, f416)
    out.update({'tiny_keep_' + k: v.numpy().astype(np.int32) for k, v in keep.items()})
    out.update(tiny_feature64=f64.numpy(), tiny_feature416=f416.numpy())

    path = os.path.join(HERE, 'pruned.npz')
    np.savez_compressed(path, **out)
    print('pruned.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
