"""numpy restatement of the photometric augmentations of the reference's `transform/image.py` (RandomBlur, BGR2HSV, RandomHue,
RandomSaturation, RandomBrightness, HSV2RGB, RandomGamma) for uint8 HWC frames.  The arithmetic of the colour conversions and the box blur
lives in cv2 (OpenCV 4.13, 8-bit paths); it is restated here and pinned by `tests/golden/photometric.npz`, made with cv2 itself.  Kept
beside the tests, like `resnet_train_oracle.py`, so `oracle/yolo2_oracle.py` stays as it is.

Rules (each reproduces cv2 on every input the fixture covers):
  BGR2HSV  OpenCV's integer rule, hsv_shift = 12: sdiv[i] = round((255 << 12) / i), hdiv[i] = round((180 << 12) / (6 i));
           s = (diff * sdiv[v] + 2^11) >> 12; h = (h' * hdiv[diff] + 2^11) >> 12, + 180 when negative, where h' = g - b if v == r,
           b - r + 2 diff if v == g, else r - g + 4 diff.
  HSV2RGB  float32: hh = h * float(6/180), s' = s * float(1/255), v' = v * float(1/255); sector = floor(hh) mod 6, f = hh - floor(hh);
           tab = (v', v' (1 - s'), v' * fma(-s', f, 1), v' * fma(-s', 1 - f, 1)); out = tab[..] * 255, truncated in the vector
           body of a row and rounded half to even in its scalar tail, the last w mod 32 pixels.  The fused multiply-adds matter:
           with separate multiply and subtract about 1e-4 of the cube differs by one; with the wrong one of the two roundings about 74 %.
  blur     box sum s over a BORDER_REFLECT_101 frame, d = kw kh.  d = 1 copies.  For 2 <= d <= 24: m = floor(65536 / d),
           delta = floor(d / 2) + 1 when the fraction of 65536 / d is below 1/2, else m + 1 and floor(d / 2); out = ((s + delta) m) >> 16,
           which exceeds 255 only for d = 2 and s = 510: 255 in the 16-byte vector body of a row, 0 (uint8 wrap) in the row's scalar tail,
           the last (3 w) mod 16 bytes.  For d = 25 the quotient is exact, rounded half up: floor((2 s + d) / (2 d)).  Pinned for kw, kh
           in 1..5.
  LUTs     hue: clip(h + a, 0, 179); saturation / brightness: trunc(clip(x * a, 0, 255)) in float64; gamma: the scikit-image <= 0.18
           `adjust_gamma` of the reference's dependency era, uint8(((x / 255) ** g) * 255) in float64 with truncation (scikit-image >=
           0.19 rounds through a table instead, so this is a restatement of the older release, not of what a new install computes)."""
import numpy as np

BLUR_MAX = 5            # largest kernel width / height the box-blur rule is pinned for
SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])   # (b, g, r) taken from tab[] per sector


def hsv_tables():
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide='ignore'):
        sdiv = np.where(i > 0, np.floor((255 << 12) / np.maximum(i, 1) + 0.5), 0).astype(np.int64)
        hdiv = np.where(i > 0, np.floor((180 << 12) / (6 * np.maximum(i, 1)) + 0.5), 0).astype(np.int64)
    return sdiv, hdiv


def bgr2hsv(image):
    sdiv, hdiv = hsv_tables()
    b, g, r = [image[..., k].astype(np.int64) for k in range(3)]
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    s = (diff * sdiv[v] + (1 << 11)) >> 12
    hp = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (hp * hdiv[diff] + (1 << 11)) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


def _fma32(a, b, c):
    """float32 fused multiply-add: the float32 product is exact in float64, one rounding of the sum to float32."""
    return (a.astype(np.float64) * b.astype(np.float64) + np.float64(c)).astype(np.float32)


def hsv2rgb(image):
    f32 = np.float32
    one = f32(1)
    h = image[..., 0].astype(np.float32) * f32(6.0 / 180)
    s = image[..., 1].astype(np.float32) * f32(1.0 / 255)
    v = image[..., 2].astype(np.float32) * f32(1.0 / 255)
    pre = np.floor(h)
    f = h - pre
    tab = np.stack([v, v * (one - s), v * _fma32(-s, f, 1.0), v * _fma32(-s, one - f, 1.0)], -1)
    sector = pre.astype(np.int64) % 6
    bgr = np.take_along_axis(tab, SECTORS[sector], -1) * f32(255)
    w = image.shape[-2]
    tail = (np.arange(w) >= w - w % 32)[:, None]
    out = np.clip(np.where(tail, np.rint(bgr), np.trunc(bgr)), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(out[..., ::-1])


def reflect101(i, n):
    if n == 1:
        return np.zeros_like(i)
    i = np.abs(i)
    i = np.where(i >= n, 2 * n - 2 - i, i)
    return np.abs(i)


def blur_coef(kw, kh):
    d = kw * kh
    m = 65536 // d
    if 2 * (65536 % d) < d:
        return m, d // 2 + 1
    return m + 1, d // 2


def blur_divide(s, d, m, delta, tail):
    """window sum -> pixel.  d == 1 copies; 2 <= d <= 24 is the 16-bit fixed-point rule, whose one overflow (d == 2, s == 510 -> 256)
    saturates to 255 in the 16-byte vector body of a row and wraps to 0 in its scalar tail (`tail`: the last (3 w) mod 16 bytes);
    d == 25 rounds the exact quotient half up."""
    if d == 1:
        return s
    if d == 25:
        return (2 * s + d) // (2 * d)
    v = ((s + delta) * m) >> 16
    return np.where(v > 255, np.where(tail, v & 255, 255), v)


def blur(image, kw, kh):
    """cv2.blur(image, (kw, kh)): centred anchor, BORDER_REFLECT_101."""
    if not (1 <= kw <= BLUR_MAX and 1 <= kh <= BLUR_MAX):
        raise ValueError('the box-blur rule is pinned for kernels up to %d x %d, not %d x %d' % (BLUR_MAX, BLUR_MAX, kw, kh))
    h, w = image.shape[:2]
    ys = reflect101(np.arange(h)[:, None] + np.arange(kh)[None, :] - kh // 2, h)       # [h, kh]
    xs = reflect101(np.arange(w)[:, None] + np.arange(kw)[None, :] - kw // 2, w)       # [w, kw]
    x = image.astype(np.int64)
    rows = x[:, xs, :].sum(2)                                                         # [h, w, 3]
    s = rows[ys, :, :].sum(1)
    m, delta = blur_coef(kw, kh)
    tail = (np.arange(3 * w) >= 3 * w - (3 * w) % 16).reshape(w, 3)
    return blur_divide(s, kw * kh, m, delta, tail[None]).astype(np.uint8)


def hue_lut(a):
    return np.clip(np.arange(256) + int(a), 0, 179).astype(np.uint8)


def scale_lut(a):
    return np.clip(np.arange(256, dtype=np.uint8) * float(a), 0, 255).astype(np.uint8)


def gamma_lut(g):
    return np.uint8(((np.arange(256, dtype=np.uint8) / 255.0) ** float(g)) * 255.0)


def apply_lut(image, lut, channel=None):
    out = image.copy()
    if channel is None:
        return lut[image]
    out[..., channel] = lut[image[..., channel]]
    return out


def apply(op, image, draw):
    """One reference op on one frame with its recorded draw: op in ('blur', 'bgr2hsv', 'hsv2rgb', 'bgr2rgb', 'hue', 'saturation',
    'brightness', 'gamma')."""
    if op == 'blur':
        return blur(image, *draw)
    if op == 'bgr2hsv':
        return bgr2hsv(image)
    if op == 'hsv2rgb':
        return hsv2rgb(image)
    if op == 'bgr2rgb':
        return np.ascontiguousarray(image[..., ::-1])
    if op == 'hue':
        return apply_lut(image, hue_lut(draw), 0)
    if op == 'saturation':
        return apply_lut(image, scale_lut(draw), 1)
    if op == 'brightness':
        return apply_lut(image, scale_lut(draw), 2)
    if op == 'gamma':
        return apply_lut(image, gamma_lut(draw))
    raise ValueError(op)


def hsv_cube():
    """All 2^24 uint8 triples as a 4096 x 4096 frame, first channel slowest."""
    i = np.arange(1 << 24, dtype=np.int64)
    return np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
