#!/usr/bin/env python
"""Golden fixture for the tensor transform (`[transform] tensor = torchvision.transforms.ToTensor transform.image.Normalize`, the reference's
default config.ini), produced by EXECUTING the reference's own `transform.image.Normalize` through the reference's own
`transform.get_transform` (default compose: torchvision.transforms.Compose).  The reference's modules import `inflection` (absent) and its
`utils` (pandas, PIL), so the class and the two functions are extracted with `ast` and given shims:
  - inflection.underscore: CamelCase -> snake_case;
  - utils.parse_attr: the dotted name resolved with importlib, `transform.image.Normalize` to the extracted class.

Stored per `[transform] normalize` setting k (SETTINGS):
  - table_k  fp32 [3, 256]: the chain's output over a uint8 HWC image [256, 1, 3] holding every byte value in every channel;
  - c1_sha_k SHA-256 of the chain's fp32 output [3, 416, 416] on the C1 input (image.jpg -> cv2.resize 416 -> BGR2RGB, the `rgb` of
    c1_image.npz, whose SHA-256 is `rgb_sha`), and c1_crop_k = that output's [:, 200:216, 300:316].

    python tests/golden/make_golden_normalize.py          # build container only (needs /root/reference + cv2)
"""
import ast
import configparser
import hashlib
import importlib
import inspect
import os
import re
import types

import cv2
import numpy as np
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
SETTINGS = ('0.5 1', '0.485 0.229')       # the reference's default; a mean and a std that are not powers of two
CROP = (slice(None), slice(200, 216), slice(300, 316))


def extract(path, names, ns):
    tree = ast.parse(open(path).read())
    nodes = [n for n in tree.body if isinstance(n, (ast.ClassDef, ast.FunctionDef)) and n.name in names]
    exec(compile(ast.Module(body=nodes, type_ignores=[]), path, 'exec'), ns)
    return ns


def load_reference():
    inflection = types.SimpleNamespace(underscore=lambda s: re.sub(r'([a-z\d])([A-Z])', r'\1_\2', re.sub(r'([A-Z]+)([A-Z][a-z])', r'\1_\2', s)).lower())
    image = extract(os.path.join(REF, 'transform', 'image.py'), ('Normalize',), dict(torchvision=torchvision, inflection=inflection))

    def parse_attr(s):
        if s == 'transform.image.Normalize':
            return image['Normalize']
        m, n = s.rsplit('.', 1)
        return getattr(importlib.import_module(m), n)

    utils = types.SimpleNamespace(parse_attr=parse_attr)
    tr = extract(os.path.join(REF, 'transform', '__init__.py'), ('parse_transform', 'get_transform'),
                 dict(inspect=inspect, torchvision=torchvision, utils=utils))
    return tr['get_transform']


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    get_transform = load_reference()
    ref_config = configparser.ConfigParser()
    ref_config.read(os.path.join(REF, 'config.ini'))
    sequence = ref_config.get('transform', 'tensor').split()
    assert sequence == ['torchvision.transforms.ToTensor', 'transform.image.Normalize'], sequence
    assert ref_config.get('transform', 'normalize') == SETTINGS[0]
    every = np.repeat(np.arange(256, dtype=np.uint8).reshape(256, 1, 1), 3, axis=2)
    image_bgr = cv2.imread(os.path.join(REF, 'image.jpg'))
    rgb = cv2.cvtColor(cv2.resize(image_bgr, (416, 416)), cv2.COLOR_BGR2RGB)
    c1 = np.load(os.path.join(HERE, 'c1_image.npz'))
    assert np.array_equal(rgb, c1['rgb'])
    out = dict(rgb_sha=sha(rgb), settings=np.array(SETTINGS))
    for k, setting in enumerate(SETTINGS):
        config = configparser.ConfigParser()
        config.read_dict({'transform': {'tensor': ' '.join(sequence), 'normalize': setting}})
        chain = get_transform(config, config.get('transform', 'tensor').split())
        table = chain(every.copy()).numpy()
        assert table.shape == (3, 256, 1) and table.dtype == np.float32
        out['table_%d' % k] = table[:, :, 0].copy()
        x = chain(rgb.copy()).numpy()
        assert x.shape == (3, 416, 416) and x.dtype == np.float32
        out['c1_sha_%d' % k] = sha(x)
        out['c1_crop_%d' % k] = x[CROP].copy()
    path = os.path.join(HERE, 'normalize.npz')
    np.savez_compressed(path, **out)
    print('normalize.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
