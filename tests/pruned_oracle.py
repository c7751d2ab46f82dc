"""Channel-pruned Darknet-19 and Tiny YOLOv2 state_dicts for the pruned-width tests (tests/test_pruned_darknet*.py) and their golden
generator (tests/golden/make_golden_pruned.py).

A pruned checkpoint is the oracle's full-width synthetic state_dict (oracle/yolo2_oracle.py, seed 0) with a kept subset of every unit's
filters, cascaded to the consumer's input channels the way the reference's pruner.py does (`var[keep]` on the producer,
`var[mapper(keep, channels)]` on the consumer).  The subsets are seeded and are not prefixes.  Only the kept index lists go into the
fixture; the weights are rebuilt from the seed here.
"""
import numpy as np
import torch

from oracle import yolo2_oracle as O

# filters kept per unit.  The pattern covers: layers1.0 under 32 filters; widths with Cout % 8 != 0 (so the next unit reads a
# zero-padded tail); an odd passthrough width; a pruned layers3.0; and widths that are multiples of 32 (layers1.6, layers2.4).
DARKNET_KEEP = {
    'layers1.0': 27, 'layers1.2': 58, 'layers1.4': 115, 'layers1.5': 57, 'layers1.6': 96, 'layers1.8': 230, 'layers1.9': 121,
    'layers1.10': 250, 'layers1.12': 461, 'layers1.13': 199, 'layers1.15': 230, 'layers1.16': 470,
    'layers2.1': 1000, 'layers2.2': 450, 'layers2.3': 922, 'layers2.4': 480, 'layers2.5': 1010, 'layers2.6': 1001, 'layers2.7': 999,
    'passthrough': 57, 'layers3.0': 921,
}
TINY_KEEP = {'layers.0': 13, 'layers.2': 27, 'layers.4': 61, 'layers.6': 100, 'layers.8': 224, 'layers.10': 469, 'layers.13': 1000,
             'layers.14': 923}


def keep_lists(counts, widths, seed):
    """{unit: sorted LongTensor of kept filters}: a seeded random subset of `counts[unit]` of the unit's `widths[unit]` filters."""
    rng = np.random.default_rng(seed)
    out = {}
    for key in sorted(counts):
        idx = np.sort(rng.choice(widths[key], counts[key], replace=False))
        out[key] = torch.from_numpy(idx).long()
    return out


def reorg_mapper(indices, channels, stride=2):
    """The reference's get_mapper(94) (model/yolo2.py:135-137): channel c of the passthrough is channel s*channels + c of the reorg."""
    return torch.cat([indices + s * channels for s in range(stride * stride)])


def _prune(sd, units, keep, inputs):
    """units: [(key, full Cout)] in network order; inputs(key, prev) -> LongTensor of the unit's kept input channels."""
    out = dict(sd)
    prev = None
    for key, cout in units:
        kout = keep.get(key, torch.arange(cout))
        kin = inputs(key, prev)
        out[key + '.conv.weight'] = sd[key + '.conv.weight'][kout][:, kin].contiguous()
        for name in ('.conv.bias', '.bn.weight', '.bn.bias', '.bn.running_mean', '.bn.running_var'):
            if key + name in sd:
                out[key + name] = sd[key + name][kout].contiguous()
        prev = kout
    return out


def darknet_widths():
    return {l['key']: l['cout'] for l in O.darknet19_layers()}


def darknet_keep(seed=1):
    return keep_lists(DARKNET_KEEP, darknet_widths(), seed)


def prune_darknet(sd, keep):
    """The full-width Darknet-19 state_dict `sd` cut to the kept filters `keep` ({unit: LongTensor}), inputs cascaded; layers3.0 reads the
    kept passthrough channels through the reorg map and the kept layers2.7 channels after the 4 * Cpt reorg channels."""
    widths = darknet_widths()

    def inputs(key, prev):
        if key == 'layers1.0':
            return torch.arange(3)
        if key in ('passthrough', 'layers2.1'):
            return keep.get('layers1.16', torch.arange(widths['layers1.16']))
        if key == 'layers3.0':
            c_pt = widths['passthrough']
            k_pt = keep.get('passthrough', torch.arange(c_pt))
            k_27 = keep.get('layers2.7', torch.arange(widths['layers2.7']))
            return torch.cat([reorg_mapper(k_pt, c_pt), k_27 + 4 * c_pt])
        return prev

    return _prune(sd, [(l['key'], l['cout']) for l in O.darknet19_layers()], keep, inputs)


def tiny_widths():
    return {l['key']: l['cout'] for l in O.tiny_layers()}


def tiny_keep(seed=2):
    return keep_lists(TINY_KEEP, tiny_widths(), seed)


def prune_tiny(sd, keep):
    def inputs(key, prev):
        return torch.arange(3) if prev is None else prev

    return _prune(sd, [(l['key'], l['cout']) for l in O.tiny_layers()], keep, inputs)


def darknet_pruned_state_dict(keep=None):
    return prune_darknet(O.make_state_dict(0), darknet_keep() if keep is None else keep)


def tiny_pruned_state_dict(keep=None):
    return prune_tiny(O.make_tiny_state_dict(0), tiny_keep() if keep is None else keep)


def keep_from_npz(g, prefix):
    """{unit: LongTensor} stored by make_golden_pruned.py as `<prefix>keep_<unit>` arrays."""
    return {k[len(prefix) + 5:]: torch.from_numpy(g[k]).long() for k in g.files if k.startswith(prefix + 'keep_')}
