"""transform.image -- the image transforms of the reference (transform/image.py) for uint8 HWC frames, on the GPU.

`BGR2RGB` is a strided view stand-alone; inside `transform.resize_batch` the swap is fused into the resize kernel.
The photometric chain -- `RandomBlur`, `BGR2HSV`, `RandomHue`, `RandomSaturation`, `RandomBrightness`, `HSV2RGB`, `RandomGamma`, the
`transform/image_train` sequence the reference's config.ini offers -- runs bit-exactly with cv2 4.13 in yb_photometric_batch_u8.  Each
class takes the reference's constructor arguments and draws Python's `random` exactly as the reference does (`draw`); hue, saturation,
brightness and gamma become per-image, per-channel 256-entry tables built on the host (gamma in float64, the scikit-image <= 0.18
`adjust_gamma` rule of the reference's dependency era), and consecutive tables compose exactly.

`Compose` compiles a sequence into launches of one kernel: each segment is at most one blur followed by per-pixel stages in registers
(BGR<->RGB swap, BGR2HSV, lookup table, HSV2RGB), so the reference's order is a single launch and any other order stays exact.  Calling a
single op, or a `Compose`, on one frame runs the same kernel on a batch of one; `Compose.batch` runs a whole resized batch with the draws
made image by image, op by op, as the reference's `Collate` makes them."""
import random
import re

import numpy as np
import torch
import torchvision

from b200 import ops as _ops

BLUR_MAX = 5                  # largest blur kernel width / height whose cv2 rounding is pinned (tests/golden/photometric.npz)
MAX_STAGES, MAX_LUTS = 7, 4   # per launch (include/yolo2_b200.h)
BLUR, SWAP, HSV, RGB, LUT = 1, 2, 3, 4, 5   # YB_PH_* stage codes


def underscore(name):
    """inflection.underscore: 'RandomBlur' -> 'random_blur' (the reference's option names)."""
    return re.sub(r'([a-z\d])([A-Z])', r'\1_\2', re.sub(r'([A-Z]+)([A-Z][a-z])', r'\1_\2', name)).lower()


def _adjust(obj, config, cast):
    return tuple(map(cast, config.get('augmentation', underscore(type(obj).__name__)).split()))


class Normalize(torchvision.transforms.Normalize):
    """The reference's tensor transform (transform/image.py): `[transform] normalize = mean std`, each repeated over the 3 channels.  It
    runs in a `transform.TensorTransform` chain after torchvision's ToTensor."""

    def __init__(self, config):
        name = underscore(type(self).__name__)
        mean, std = tuple(map(float, config.get('transform', name).split()))
        torchvision.transforms.Normalize.__init__(self, (mean, mean, mean), (std, std, std))


class _Op(object):
    kind = None

    def draw(self):
        return None

    def __call__(self, image):
        return Compose([self])(image)


class BGR2RGB(_Op):
    kind = SWAP

    def __call__(self, image):
        return image.flip(-1)


class BGR2HSV(_Op):
    kind = HSV


class HSV2RGB(_Op):
    kind = RGB


class RandomBlur(_Op):
    """cv2.blur with a (randint(1, kw_max), randint(1, kh_max)) kernel.  Maxima beyond BLUR_MAX raise: cv2 changes its rounding for
    larger kernels and that rule is not pinned, so those draws could not be reproduced bit-exactly."""
    kind = BLUR

    def __init__(self, config):
        self.adjust = _adjust(self, config, int)
        if len(self.adjust) != 2 or not all(1 <= a <= BLUR_MAX for a in self.adjust):
            raise ValueError('random_blur = %s: kernel maxima must be two integers in 1..%d (the cv2 rounding pinned for the device blur)'
                             % (' '.join(map(str, self.adjust)), BLUR_MAX))

    def draw(self):
        return tuple(random.randint(1, adjust) for adjust in self.adjust)


class _Table(_Op):
    kind = LUT
    channel = None

    def table(self, draw):
        """[3, 256] uint8 per-channel lookup table for one draw (identity on the channels the op leaves alone)."""
        t = np.tile(np.arange(256, dtype=np.uint8), (3, 1))
        lut = self.lut(draw)
        if self.channel is None:
            t[:] = lut
        else:
            t[self.channel] = lut
        return t


class RandomHue(_Table):
    channel = 0

    def __init__(self, config):
        self.adjust = _adjust(self, config, int)

    def draw(self):
        return random.randint(*self.adjust)

    def lut(self, adjust):
        return np.clip(np.arange(256) + int(adjust), 0, 179).astype(np.uint8)


class RandomSaturation(_Table):
    channel = 1

    def __init__(self, config):
        self.adjust = _adjust(self, config, float)

    def draw(self):
        return random.uniform(*self.adjust)

    def lut(self, adjust):
        return np.clip(np.arange(256, dtype=np.uint8) * float(adjust), 0, 255).astype(np.uint8)


class RandomBrightness(RandomSaturation):
    channel = 2


class RandomGamma(_Table):
    def __init__(self, config):
        self.adjust = _adjust(self, config, float)

    def draw(self):
        return random.uniform(*self.adjust)

    def lut(self, gamma):
        return np.uint8(((np.arange(256, dtype=np.uint8) / 255.0) ** float(gamma)) * 255.0)


def compile_chain(transforms):
    """Sequence of ops -> segments, one launch each: [(stage code, [indices of the ops it runs]), ...].  A blur opens a segment;
    consecutive table ops merge into one table; a segment also closes at MAX_STAGES stages or MAX_LUTS tables."""
    segments, cur = [], []
    for i, t in enumerate(transforms):
        if t.kind == BLUR:
            if cur:
                segments.append(cur)
            cur = [(BLUR, [i])]
            continue
        if t.kind == LUT and cur and cur[-1][0] == LUT:
            cur[-1][1].append(i)
            continue
        if len(cur) == MAX_STAGES or (t.kind == LUT and sum(code == LUT for code, _ in cur) == MAX_LUTS):
            segments.append(cur)
            cur = []
        cur.append((t.kind, [i]))
    if cur:
        segments.append(cur)
    return segments


def stage_word(segment):
    return sum(code << (4 * k) for k, (code, _) in enumerate(segment))


def launch(src, dst, segment, params):
    """One yb_photometric_batch_u8 launch: src / dst uint8 CUDA [B, H, W, 3] (distinct), params a uint8 CUDA tensor [B, stride]."""
    b, h, w, _ = src.shape
    _ops.call('yb_photometric_batch_u8', src, dst, int(b), int(h), int(w), params, int(params.shape[1]), stage_word(segment))
    return dst


class Compose(object):
    """The reference's `transform.get_transform(config, sequence)` for image ops, compiled into segments (`compile_chain`)."""

    def __init__(self, transforms):
        self.transforms = list(transforms)
        for t in self.transforms:
            if not isinstance(t, _Op):
                raise TypeError('transform.image.Compose composes the ops of transform.image, not %r' % (t,))
        self.segments = compile_chain(self.transforms)

    @property
    def swap_only(self):
        """True for the default `image_train = transform.image.BGR2RGB`: the swap stays fused inside the resize kernel."""
        return len(self.transforms) == 1 and isinstance(self.transforms[0], BGR2RGB)

    def draw(self, batch):
        """Draws for `batch` images, image by image and op by op, as the reference's Collate makes them."""
        return [[t.draw() for t in self.transforms] for _ in range(batch)]

    def params(self, draws):
        """Host parameter block per segment: uint8 [B, 16 + 768 * tables] (kw, kh as int32, then the composed tables)."""
        out = []
        for seg in self.segments:
            nlut = sum(code == LUT for code, _ in seg)
            p = np.zeros((len(draws), 16 + 768 * nlut), np.uint8)
            for i, d in enumerate(draws):
                k = 0
                for code, idx in seg:
                    if code == BLUR:
                        p[i, :8] = np.frombuffer(np.array(d[idx[0]], np.int32).tobytes(), np.uint8)
                    elif code == LUT:
                        tab = self.transforms[idx[0]].table(d[idx[0]])
                        for j in idx[1:]:
                            tab = np.take_along_axis(self.transforms[j].table(d[j]), tab.astype(np.int64), 1)
                        p[i, 16 + 768 * k:16 + 768 * (k + 1)] = tab.reshape(-1)
                        k += 1
            out.append(p)
        return out

    def batch(self, frames, draws=None):
        """uint8 CUDA [B, H, W, 3] -> a new uint8 CUDA tensor, one launch per segment; `draws` from `draw` (drawn here if None)."""
        if not (torch.is_tensor(frames) and frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3):
            raise ValueError('Compose.batch expects a uint8 CUDA tensor [B, H, W, 3]')
        if draws is None:
            draws = self.draw(frames.shape[0])
        x = frames.contiguous()
        if not self.segments:
            return x.clone()
        for seg, p in zip(self.segments, self.params(draws)):
            params = torch.from_numpy(p).pin_memory().to(x.device, non_blocking=True)
            x = launch(x, torch.empty_like(x), seg, params)
        return x

    def __call__(self, image):
        """One uint8 [h, w, 3] frame (numpy or tensor) -> uint8 CUDA tensor [h, w, 3]."""
        image = image if torch.is_tensor(image) else torch.from_numpy(np.ascontiguousarray(image))
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3:
            raise ValueError('expected a uint8 [h, w, 3] frame')
        dev = torch.device('cuda', torch.cuda.current_device())
        return self.batch(image.to(dev)[None])[0]
