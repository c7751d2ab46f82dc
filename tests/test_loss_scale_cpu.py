"""Dynamic loss scaling without a GPU: the `[train] loss_scale` and `loss_scale_growth_interval` keys, the trainer's setting, and the new
C-ABI entry's declaration against its ctypes binding."""
import configparser
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def config(**train):
    cfg = configparser.ConfigParser()
    cfg.read_dict({'train': dict(cross_entropy='1', **train)})
    return cfg


def test_absent_key_is_static():
    import train
    assert train.loss_scale_config(config()) == ('static', 2000)
    cfg = configparser.ConfigParser()
    cfg.read_dict({'model': {'threshold': '0.6'}})              # no [train] section at all
    assert train.loss_scale_config(cfg) == ('static', 2000)


def test_dynamic_with_interval_accepted():
    import train
    assert train.loss_scale_config(config(loss_scale='dynamic')) == ('dynamic', 2000)
    assert train.loss_scale_config(config(loss_scale=' dynamic ', loss_scale_growth_interval='2')) == ('dynamic', 2)
    assert train.loss_scale_config(config(loss_scale='static', loss_scale_growth_interval='50')) == ('static', 50)


@pytest.mark.parametrize('train_keys, key', [(dict(loss_scale='foo'), 'loss_scale'),
                                             (dict(loss_scale='Dynamic'), 'loss_scale'),
                                             (dict(loss_scale='dynamic', loss_scale_growth_interval='0'), 'loss_scale_growth_interval'),
                                             (dict(loss_scale='dynamic', loss_scale_growth_interval='-3'), 'loss_scale_growth_interval'),
                                             (dict(loss_scale='dynamic', loss_scale_growth_interval='2.5'), 'loss_scale_growth_interval'),
                                             (dict(loss_scale_growth_interval='many'), 'loss_scale_growth_interval')])
def test_bad_values_raise_naming_the_key(train_keys, key):
    import train
    with pytest.raises(ValueError, match=r'\[train\] %s ' % key):
        train.loss_scale_config(config(**train_keys))


def test_trainer_setting():
    from b200 import train_engine
    t = train_engine.TrainerBase(dnn=None)
    assert (t.loss_scale, t.growth_interval, t.loss_factor) == ('static', 2000, None)
    assert t.loss_scale_state('cpu') == []                       # static mode creates no state
    t.set_loss_scale('dynamic', 7)
    assert (t.loss_scale, t.growth_interval) == ('dynamic', 7)
    with pytest.raises(ValueError):
        t.set_loss_scale('auto')
    with pytest.raises(ValueError):
        t.set_loss_scale('dynamic', 0)


def test_new_entry_declared_and_bound():
    from b200 import lib
    with open(os.path.join(ROOT, 'include', 'yolo2_b200.h')) as fh:
        header = fh.read()
    m = re.search(r'int yb_grad_unscale_guard\(([^;]*)\);', header)
    assert m is not None
    args = [a for a in m.group(1).split(',') if a.strip()]
    assert len(args) == len(lib.SIGNATURES['yb_grad_unscale_guard']) == 7
    with open(os.path.join(ROOT, 'yolo2-pytorch_b200', 'csrc', 'capi.cu')) as fh:
        assert re.search(r'int yb_grad_unscale_guard\(', fh.read())
