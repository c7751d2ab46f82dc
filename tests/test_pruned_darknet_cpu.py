"""Channel-pruned Darknet-19 and Tiny YOLOv2 without a GPU: the channel layout of the pruned engine, its concat map against the reorg
mapper, the pruned checkpoints of tests/golden/pruned.npz, and the ValueErrors of strict precision and training at pruned widths."""
import configparser
import os

import numpy as np
import pytest
import torch

import pruned_oracle as PO
from oracle import yolo2_oracle as O


def make_config(precision=None):
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    if precision:
        config.read_dict({'b200': {'precision': precision}})
    return config


def darknet(sd=None, ratio=1, precision=None):
    import model
    import model.yolo2
    return model.yolo2.Darknet(model.ConfigChannels(make_config(precision), sd), O.anchors_yolo_voc(), 20, ratio=ratio)


def tiny(sd=None):
    import model
    import model.yolo2
    return model.yolo2.Tiny(model.ConfigChannels(make_config(), sd), O.anchors_yolo_voc(), 20)


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'pruned.npz'))


def test_fixture_keep_lists_are_the_seeded_subsets(golden):
    """The stored kept filters are what pruned_oracle draws from its seed: pattern, sizes, sortedness and non-prefix subsets."""
    for prefix, keep, counts, widths in (('darknet_', PO.darknet_keep(), PO.DARKNET_KEEP, PO.darknet_widths()),
                                         ('tiny_', PO.tiny_keep(), PO.TINY_KEEP, PO.tiny_widths())):
        stored = PO.keep_from_npz(golden, prefix)
        assert sorted(stored) == sorted(counts)
        for key, idx in stored.items():
            assert torch.equal(idx, keep[key]), key
            assert idx.numel() == counts[key] and bool((idx[1:] > idx[:-1]).all()) and int(idx[-1]) < widths[key]
            assert not torch.equal(idx, torch.arange(idx.numel())), key
    c = PO.DARKNET_KEEP
    assert c['layers1.0'] < 32 and c['passthrough'] % 8 and c['layers3.0'] < 1024
    assert any(v % 8 for v in c.values()) and any(v % 32 == 0 for v in c.values())


def test_concat_map_against_the_reorg_mapper():
    """layers3.0's input layout: the reference's concat channel s*Cpt + c sits at s*P + c -- get_mapper(94) with P channels -- and
    4*Cpt + j at 4P + j, for P = round_up(Cpt, 8)."""
    from b200.engine import DarknetEngine
    dnn = darknet()
    for c_pt, c_27 in ((57, 999), (64, 1024), (1, 8), (48, 768)):
        p = (c_pt + 7) // 8 * 8
        idx = DarknetEngine.concat_index(c_pt, p, c_27)
        assert torch.equal(idx[:4 * c_pt], dnn.get_mapper(94)(torch.arange(c_pt), p))
        assert torch.equal(idx[4 * c_pt:], torch.arange(c_27) + 4 * p)
        assert idx.numel() == len(set(idx.tolist()))
    # the pruned checkpoint's layers3.0 reads the kept channels of the reference's concat through the same mapper
    keep = PO.darknet_keep()
    assert torch.equal(PO.reorg_mapper(keep['passthrough'], 64), dnn.get_mapper(94)(keep['passthrough'], 64))


def test_pruned_layout(golden):
    """Stored widths round_up(Cout, 8), layers1.0 at the first-layer kernel's 32, the passthrough's 4 groups of P, layers2.7 at 4P, and
    each unit reading its producer's stored width."""
    sd = PO.darknet_pruned_state_dict(PO.keep_from_npz(golden, 'darknet_'))
    dnn = darknet(sd)
    dnn.load_state_dict(sd, strict=False)
    eng = dnn.engine
    units = dict(zip(eng.unit_keys(), eng.all_units()))
    assert units['layers1.0'].out_ch == 32 and units['layers1.2'].in_ch == 32
    for key, u in units.items():
        if key != 'layers3.1':
            assert u.out_ch == (u.cout + 7) // 8 * 8, key
    assert units['passthrough'].out_ch == 64 and units['layers3.0'].in_ch == 4 * 64 + 1000
    assert units['passthrough'].in_ch == units['layers2.1'].in_ch == units['layers1.16'].out_ch
    assert torch.equal(units['layers3.0'].cin_index, eng.concat_index(57, 64, 999))
    tails = [k for k, u in units.items() if u.in_ch % 32 and k != 'layers1.0']
    assert 'layers1.5' in tails and 'layers3.0' in tails and 'layers1.2' not in tails
    assert eng.padded_unit() == 'layers1.0'
    # ratio 0.75: the tail only where a 48-channel buffer is read (layers1.0 reads the image on the first-layer kernel)
    eng75 = darknet(ratio=0.75).engine
    tails75 = [(k, u.cin, u.in_ch, u.k_ch) for k, u in zip(eng75.unit_keys()[1:], eng75.all_units()[1:]) if u.in_ch % 32]
    assert tails75 == [('layers1.4', 48, 48, 64), ('layers1.6', 48, 48, 64)]
    assert eng75.padded_unit() == 'layers1.0'
    assert [k for k, u in zip(eng75.unit_keys(), eng75.all_units()) if u.padded] == ['layers1.0', 'layers1.2', 'layers1.4', 'layers1.6']


def test_full_width_layout_is_the_units_own():
    eng = darknet().engine
    assert eng.padded_unit() is None
    for u in eng.all_units():
        assert (u.in_ch, u.k_ch, u.out_ch, u.cin_index) == (u.cin, u.cin, u.cout, None) and not u.padded
    assert tiny().padded_unit() is None
    with pytest.raises(ValueError, match='layers1.0'):
        darknet(ratio=2).engine             # 64 first-layer filters: more than the first-layer kernel's 32


def test_strict_precision_at_pruned_widths_names_the_unit(golden):
    sd = PO.darknet_pruned_state_dict(PO.keep_from_npz(golden, 'darknet_'))
    with pytest.raises(ValueError, match='layers1.0'):
        darknet(sd, precision='strict').engine
    eng = darknet(sd).engine
    with pytest.raises(ValueError, match="strict.*layers1.0"):
        eng.set_precision('strict')
    assert eng.precision == 'fast'
    with pytest.raises(ValueError, match='layers1.0'):
        darknet(ratio=0.5).engine.set_precision('strict')


def test_training_at_pruned_widths_names_the_unit(golden):
    sd = PO.darknet_pruned_state_dict(PO.keep_from_npz(golden, 'darknet_'))
    dnn = darknet(sd)
    dnn.load_state_dict(sd, strict=False)
    dnn.train()
    with pytest.raises(ValueError, match='training.*layers1.0'):
        dnn(torch.zeros(1, 3, 64, 64))
    sd = PO.tiny_pruned_state_dict(PO.keep_from_npz(golden, 'tiny_'))
    net = tiny(sd)
    net.load_state_dict(sd, strict=False)
    net.train()
    with pytest.raises(ValueError, match='training.*layers.2'):
        net(torch.zeros(1, 3, 64, 64))
    with pytest.raises(ValueError, match='layers.2'):
        net.trainer
