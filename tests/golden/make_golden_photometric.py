#!/usr/bin/env python
"""Golden fixture for the photometric augmentations, produced by EXECUTING the reference's own classes of transform/image.py
(RandomBlur, BGR2HSV, RandomHue, RandomSaturation, RandomBrightness, HSV2RGB, RandomGamma, BGR2RGB) with cv2, the way the reference's
`Collate` runs them (utils/data.py:114-133): `random` is seeded once per batch, then every image draws op after op in the configured
order.  The module imports `inflection` and `skimage` (absent) and uses `np.int` (gone from numpy 2), so the classes are extracted with
`ast` and given shims:
  - inflection.underscore: CamelCase -> snake_case;
  - np.int: the builtin int;
  - skimage.exposure.adjust_gamma: RESTATED, not executed -- the uint8 rule of the scikit-image releases of the reference's dependency
    era (<= 0.18): uint8(((image / 255) ** gamma) * 255 * gain) in float64, truncated.  scikit-image >= 0.19 rounds through a table.
Every recorded draw is stored, so a test can replay the same chain, and every output is stored as a SHA-256.

Also stored: SHA-256 of cv2's BGR2HSV and HSV2RGB over all 2^24 inputs, and of cv2.blur for every kernel 1..5 x 1..5 on frames that
include 1 x N, N x 1, odd and 608-wide sizes.  Each stored value is also checked against the numpy restatement in
tests/photometric_oracle.py before the file is written.

    python tests/golden/make_golden_photometric.py          # build container only (needs /root/reference + cv2)
"""
import ast
import configparser
import hashlib
import os
import random
import re
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import yolo2_oracle as O  # noqa: E402
import photometric_oracle as P  # noqa: E402

REF = '/root/reference'
CLASSES = ('BGR2RGB', 'BGR2HSV', 'HSV2RGB', 'RandomBlur', 'RandomHue', 'RandomSaturation', 'RandomBrightness', 'RandomGamma')
CANONICAL = ('RandomBlur', 'BGR2HSV', 'RandomHue', 'RandomSaturation', 'RandomBrightness', 'HSV2RGB', 'RandomGamma')
# a blur in the middle (two launches), the colour stages in another order, a channel swap at the end
OTHER = ('RandomGamma', 'BGR2HSV', 'RandomSaturation', 'RandomHue', 'HSV2RGB', 'RandomBlur', 'RandomBrightness', 'BGR2RGB')
AUGMENTATION = {'random_blur': '5 5', 'random_hue': '0 25', 'random_saturation': '0.5 1.5', 'random_brightness': '0.5 1.5',
                'random_gamma': '0.9 1.5'}
BLUR_FRAMES = [(1, 37), (29, 1), (1, 1), (2, 3), (33, 45), (17, 608)]
# (name, sequence, batch, height, width, seed)
CASES = [('canon416', CANONICAL, 8, 416, 416, 1), ('canon608', CANONICAL, 8, 608, 608, 2), ('canon97', CANONICAL, 8, 97, 131, 3),
         ('canon1xn', CANONICAL, 8, 1, 53, 4), ('other416', OTHER, 8, 416, 416, 5), ('other97', OTHER, 8, 97, 131, 6),
         ('other1xn', OTHER, 8, 61, 1, 7)]
ALONE = [(c, 10 + k) for k, c in enumerate(CLASSES)]


class Recorder(object):
    """`random` as the reference's classes see it, recording every value they draw."""

    def __init__(self):
        self.log = []

    def randint(self, a, b):
        v = random.randint(a, b)
        self.log.append(v)
        return v

    def uniform(self, a, b):
        v = random.uniform(a, b)
        self.log.append(v)
        return v


def adjust_gamma(image, gamma=1, gain=1):
    scale = 255.0
    return np.uint8(((image / scale) ** gamma) * scale * gain)


def load_classes(rec):
    path = os.path.join(REF, 'transform', 'image.py')
    tree = ast.parse(open(path).read())
    nodes = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name in CLASSES]
    npx = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith('__')})
    npx.int = int
    inflection = types.SimpleNamespace(underscore=lambda s: re.sub(r'([a-z\d])([A-Z])', r'\1_\2', re.sub(r'([A-Z]+)([A-Z][a-z])', r'\1_\2', s)).lower())
    skimage = types.SimpleNamespace(exposure=types.SimpleNamespace(adjust_gamma=adjust_gamma))
    ns = dict(np=npx, cv2=cv2, random=rec, inflection=inflection, skimage=skimage)
    exec(compile(ast.Module(body=nodes, type_ignores=[]), path, 'exec'), ns)
    return ns


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


ORACLE_OP = dict(RandomBlur='blur', BGR2HSV='bgr2hsv', HSV2RGB='hsv2rgb', BGR2RGB='bgr2rgb', RandomHue='hue', RandomSaturation='saturation',
                 RandomBrightness='brightness', RandomGamma='gamma')


def oracle_chain(seq, image, draws):
    k = 0
    for name in seq:
        n = {'RandomBlur': 2, 'RandomHue': 1, 'RandomSaturation': 1, 'RandomBrightness': 1, 'RandomGamma': 1}.get(name, 0)
        d = tuple(draws[k:k + n]) if n == 2 else (draws[k] if n else None)
        image = P.apply(ORACLE_OP[name], image, d)
        k += n
    return image


def main():
    rec = Recorder()
    ns = load_classes(rec)
    config = configparser.ConfigParser()
    config.read_dict({'augmentation': AUGMENTATION})

    def make(name):
        return ns[name](config) if name.startswith('Random') else ns[name]()

    out = {}
    cube = P.hsv_cube()
    # 4096 wide: every pixel in a row's vector body; 16 wide: every pixel in a row's scalar tail
    for key, frame, code, fn in (('cube_bgr2hsv', cube, cv2.COLOR_BGR2HSV, P.bgr2hsv), ('cube_hsv2rgb', cube, cv2.COLOR_HSV2RGB, P.hsv2rgb),
                                 ('cube16_bgr2hsv', cube.reshape(-1, 16, 3), cv2.COLOR_BGR2HSV, P.bgr2hsv),
                                 ('cube16_hsv2rgb', cube.reshape(-1, 16, 3), cv2.COLOR_HSV2RGB, P.hsv2rgb)):
        ref = cv2.cvtColor(frame, code)
        assert (fn(frame) == ref).all(), key
        out[key + '_sha'] = sha(ref)
    blur_sha = np.zeros((len(BLUR_FRAMES), P.BLUR_MAX, P.BLUR_MAX, 32), np.uint8)
    for f, (h, w) in enumerate(BLUR_FRAMES):
        src = O.synth_frame(50 + f, h, w)
        for kw in range(1, P.BLUR_MAX + 1):
            for kh in range(1, P.BLUR_MAX + 1):
                ref = cv2.blur(src, (kw, kh))
                assert (P.blur(src, kw, kh) == ref).all(), (h, w, kw, kh)
                blur_sha[f, kw - 1, kh - 1] = sha(ref)
    out['blur_frames'], out['blur_seeds'], out['blur_sha'] = np.array(BLUR_FRAMES), 50 + np.arange(len(BLUR_FRAMES)), blur_sha
    out['augmentation'] = np.array(['%s=%s' % kv for kv in sorted(AUGMENTATION.items())])
    # each op alone on one frame, 4 draws each (random seeded once)
    for name, seed in ALONE:
        op = make(name)
        src = O.synth_frame(seed, 61, 83)
        random.seed(seed)
        shas, draws = [], []
        for _ in range(4):
            rec.log = []
            r = op(src)
            assert (oracle_chain((name,), src, rec.log) == r).all(), name
            shas.append(sha(r))
            draws.append(list(rec.log) or [0])
        out['alone_%s_seed' % name], out['alone_%s_sha' % name] = np.array(seed), np.stack(shas)
        out['alone_%s_draws' % name] = np.array(draws, np.float64)
    # chains over batches: draws image by image, op by op, as Collate makes them
    for name, seq, b, h, w, seed in CASES:
        ops = [make(n) for n in seq]
        random.seed(seed)
        shas, draws = [], []
        for i in range(b):
            img = O.synth_frame(1000 * seed + i, h, w)
            rec.log = []
            for op in ops:
                img = op(img)
            assert (oracle_chain(seq, O.synth_frame(1000 * seed + i, h, w), rec.log) == img).all(), (name, i)
            shas.append(sha(img))
            draws.append(list(rec.log))
        out['case_%s_seq' % name] = np.array(seq)
        out['case_%s_dims' % name] = np.array([b, h, w, seed])
        out['case_%s_sha' % name], out['case_%s_draws' % name] = np.stack(shas), np.array(draws, np.float64)
    out['cases'] = np.array([c[0] for c in CASES])
    out['alone'] = np.array([c[0] for c in ALONE])
    path = os.path.join(HERE, 'photometric.npz')
    np.savez_compressed(path, **out)
    print('photometric.npz %.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
