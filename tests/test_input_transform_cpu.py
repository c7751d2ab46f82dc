"""The tensor transform without a GPU: `transform.TensorTransform`'s table against torchvision's own chain on every byte value, the port's
`transform.image.Normalize` against the executed reference (tests/golden/normalize.npz), the chain refusals, and the `_lut` entries'
declarations against their ctypes bindings."""
import configparser
import hashlib
import os
import re

import numpy as np
import pytest
import torch
import torchvision.transforms as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')

IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
CHAINS = {
    'to_tensor': [],
    'reference_default': [((0.5, 0.5, 0.5), (1.0, 1.0, 1.0))],
    'imagenet': [IMAGENET],
    'std_not_pow2': [((0.25, 0.5, 0.75), (0.3, 0.7, 0.11))],
    'two_normalizes': [IMAGENET, ((0.5, -0.25, 0.125), (3.0, 0.6, 1.7))],
}
NEW_ENTRIES = {
    'yb_totensor_lut_u8': 7,
    'yb_conv0_bn_leaky_pool_lut_fwd': 12,
    'yb_conv0_c64_bn_act_lut_fwd': 12,
    'yb_mb_conv0_bn_relu_lut_fwd': 10,
    'yb_mb_conv0_split_lut_fwd': 10,
    'yb_stem3x3_s2_bn_relu_lut_fwd': 11,
    'yb_stem7x7_bn_relu_lut_fwd': 10,
}


def chain(name):
    return [T.ToTensor()] + [T.Normalize(m, s) for m, s in CHAINS[name]]


def bits(t):
    return np.ascontiguousarray(np.asarray(t, np.float32)).view(np.int32)


def lookup(table, image):
    """table [3, 256] applied to a uint8 HWC image -> [3, H, W]."""
    return torch.stack([table[c][torch.from_numpy(image[:, :, c].astype(np.int64))] for c in range(3)])


@pytest.mark.parametrize('name', sorted(CHAINS))
def test_table_equals_torchvision_on_every_byte(name):
    import transform
    t = transform.TensorTransform(chain(name))
    assert t.table.shape == (3, 256) and t.table.dtype == torch.float32
    every = np.repeat(np.arange(256, dtype=np.uint8).reshape(256, 1, 1), 3, axis=2)
    ref = T.Compose(chain(name))(every)[:, :, 0]
    assert np.array_equal(bits(t.table), bits(ref))
    # and on an image whose channels hold different values at every pixel
    rng = np.random.default_rng(7)
    image = rng.integers(0, 256, (19, 23, 3), dtype=np.uint8)
    assert np.array_equal(bits(lookup(t.table, image)), bits(T.Compose(chain(name))(image)))


def test_to_tensor_table_is_division_by_255():
    import transform
    t = transform.to_tensor_transform()
    v = torch.arange(256, dtype=torch.float32)
    assert torch.equal(t.table, torch.stack([v.div(255)] * 3))


def config(normalize):
    cfg = configparser.ConfigParser()
    cfg.read_dict({'transform': {'tensor': 'torchvision.transforms.ToTensor transform.image.Normalize', 'normalize': normalize}})
    return cfg


def test_normalize_matches_executed_reference():
    import transform
    import transform.image
    z = np.load(os.path.join(GOLDEN, 'normalize.npz'))
    rgb = np.load(os.path.join(GOLDEN, 'c1_image.npz'))['rgb']
    assert hashlib.sha256(rgb.tobytes()).digest() == z['rgb_sha'].tobytes()
    for k, setting in enumerate(z['settings']):
        cfg = config(str(setting))
        t = transform.get_transform(cfg, cfg.get('transform', 'tensor').split(), compose=transform.TensorTransform)
        n = t.transforms[1]
        assert isinstance(n, transform.image.Normalize) and isinstance(n, T.Normalize)
        mean, std = map(float, str(setting).split())
        assert tuple(n.mean) == (mean,) * 3 and tuple(n.std) == (std,) * 3
        assert np.array_equal(bits(t.table), bits(z['table_%d' % k]))
        x = lookup(t.table, rgb).numpy()
        assert hashlib.sha256(np.ascontiguousarray(x).tobytes()).digest() == z['c1_sha_%d' % k].tobytes()
        assert np.array_equal(bits(x[:, 200:216, 300:316]), bits(z['c1_crop_%d' % k]))


@pytest.mark.parametrize('items, named', [
    ([T.Normalize((0.5,) * 3, (1.0,) * 3), T.ToTensor()], r'Normalize\(mean=\(0\.5'),
    ([T.ToTensor(), T.Normalize((0.5,), (1.0,))], r'Normalize\(mean=\(0\.5,\)'),
    ([T.ToTensor(), T.Normalize((0.1, 0.2, 0.3, 0.4), (1.0,) * 4)], r'Normalize\(mean=\(0\.1, 0\.2, 0\.3, 0\.4\)'),
    ([T.ToTensor(), T.Normalize((0.5,) * 3, (1.0,)), ], r'Normalize\(mean=\(0\.5, 0\.5, 0\.5\), std=\(1\.0,\)\)'),
    ([T.ToTensor(), T.ToTensor()], r'ToTensor\(\)'),
    ([T.ToTensor(), T.Normalize((0.5,) * 3, (1.0,) * 3), T.RandomHorizontalFlip()], r'RandomHorizontalFlip'),
    ([T.Resize(32), T.ToTensor()], r'Resize'),
    ([], r'empty'),
])
def test_chain_refusals_name_the_item(items, named):
    import transform
    with pytest.raises(ValueError, match=named):
        transform.TensorTransform(items)


def test_refusal_through_config():
    import transform
    cfg = configparser.ConfigParser()
    cfg.read_dict({'transform': {'tensor': 'transform.image.Normalize torchvision.transforms.ToTensor', 'normalize': '0.5 1'}})
    with pytest.raises(ValueError, match='Normalize'):
        transform.get_transform(cfg, cfg.get('transform', 'tensor').split(), compose=transform.TensorTransform)


def test_set_input_transform_takes_a_tensor_transform():
    import model.resnet
    import transform
    cc = __import__('model').ConfigChannels(configparser.ConfigParser())
    net = model.resnet.resnet18(cc, torch.zeros(5, 2), 20)
    assert net.input_transform is None
    t = transform.TensorTransform(chain('imagenet'))
    assert net.set_input_transform(t) is net and net.input_transform is t
    assert net.set_input_transform(None).input_transform is None
    with pytest.raises(TypeError):
        net.set_input_transform(T.Compose(chain('imagenet')))


def test_new_entries_declared_and_bound():
    from b200 import lib
    with open(os.path.join(ROOT, 'include', 'yolo2_b200.h')) as fh:
        header = fh.read()
    with open(os.path.join(ROOT, 'yolo2-pytorch_b200', 'csrc', 'capi.cu')) as fh:
        capi = fh.read()
    for name, arity in NEW_ENTRIES.items():
        m = re.search(r'int %s\(([^;]*)\);' % name, header)
        assert m is not None, name
        args = [a for a in m.group(1).split(',') if a.strip()]
        assert len(args) == len(lib.SIGNATURES[name]) == arity, name
        assert re.search(r'int %s\(' % name, capi), name
        if name != 'yb_totensor_lut_u8':
            assert args[0].split() == ['const', 'unsigned', 'char*', 'x_nhwc_u8'] and args[1].split() == ['const', 'float*', 'lut'], name
            # the fp32 entry it mirrors: the same arguments after x, one fewer in all
            fp32 = name.replace('_lut_fwd', '_fwd')
            assert len(lib.SIGNATURES[fp32]) == arity - 1, fp32
