"""Contract of the ResNet and MobileNet plugin kernels (resnet_ops.cu, mobilenet_ops.cu, the 3x3 max-pool window of yb_pool.cuh), element by
element against float64 on the exact operands each kernel reads, on non-square, odd and ragged shapes.  Same method and helpers as
test_conv_contract.py and test_train_ops_contract.py: fp16 outputs go through `check_f16` (the bound plus half an fp16 ulp, then RN16(ref)
bit for bit wherever no fp16 rounding boundary lies within the bound), fp32 outputs through `check_f32`.  max|d| / max|ref| is never used.
u = 2^-24 (fp32 unit roundoff), v = 2^-53; sum_err(A, L, G) = 1.01 (L u + (G + 64) v) A is recursive summation with L fp32 and G float64
additions over terms of absolute sum A (test_train_ops_contract).  Every output buffer is filled with SENTINEL and followed by a guard region
that must keep it; a refused launch must leave the whole buffer untouched.

Operands.  The stems (stem7x7, mb_conv0 / stem3x3_s2) read the fp32 NCHW image and fp32 weights; an fp32 x fp32 product is exact in fmaf and
in float64.  The depthwise kernels read fp16 activations and fp32 weights, the split form RN32(hi + lo) per tap.  The weight gradients read
the fp32 image or the fp16 activation and the fp16 dz.

Forward bounds (one thread owns an output pixel's whole sum, an fmaf chain in tap order):
  * stem7x7: 147 taps in (ci, r, s) order, E_acc = sum_err(S, 147, 0) with S = sum |x w| (a float64 conv of |x| and |w|);
  * mb_conv0 / stem3x3_s2: 27 taps, E_acc = sum_err(S, 27, 0);
  * dwconv3x3: 9 taps per channel, E_acc = sum_err(S, 9, 0); the split form adds one fp32 rounding of hi + lo per tap:
    E_acc = sum_err(S, 10, 0) with S over the exact hi + lo;
  * dwconv3x3_dgrad: at most 9 terms, E_acc = sum_err(S, 9, 0).
  The raw forms store RN16(acc).  The BatchNorm forms store RN16(max(acc sc + sh, 0)): the product and the add cost at most two roundings,
  E = |sc| E_acc + 2 u (|sc| (|acc| + E_acc) + |sh|), and the ReLU is 1-Lipschitz.
  The split forms store hi = RN16(v) and lo = RN16(v - hi), v the fp32 result; v - hi is exact in fp32.  So hi is checked against ref with
  E, lo against ref - hi with E: that asserts |hi + lo - ref| <= E + 1/2 ulp16(|ref - hi| + E) (1 + 2^-10), whose half ulp never drops below
  2^-25, the fp16 subnormal floor of lo, and lo == RN16(ref - hi) wherever that is unambiguous.  hi also equals the BatchNorm form bit for bit.

Weight-gradient bounds (an fp32 chain per thread, then unordered fp32 atomics), geometry restated from the host code with sms() SMs:
  * stem7x7_wgrad: 16-pixel slabs, grid = min(ceil(pixels / 256), 4 SMs); a thread walks every grid-th slab, L = 16 ceil(slabs / grid) fmaf;
    then one global atomic per CTA: E = sum_err(S, L + grid + 2, pixels);
  * dwconv3x3_wgrad: lanes = 256 / (C / 8) pixel lanes per CTA, grid = min(ceil(pixels / (16 lanes)), 4 SMs), L = ceil(pixels / (grid
    lanes)); then lanes shared atomics and grid global atomics: E = sum_err(S, L + lanes + grid, pixels);
  * mb_conv0_wgrad / stem3x3_s2_wgrad: lanes = 8, grid = min(ceil(pixels / 256), 6 SMs), same form.
  S = sum |x dz| per weight; the G = pixels float64 additions cover the reference's own sum.  At the training sizes (64 x 416^2 for the
  stem, 32 x 416^2 for MobileNet) the worst err / bound and the worst |err| / |dw| are recorded.

Bit-exact kernels: the 3x3 stride-2 max-pool forward against torch's rule (first maximum in scan order; a NaN in the window gives NaN),
compared on bits, except two points where the device's fp16 max decides: a NaN window is checked for NaN (any payload), and a zero
maximum is +0 when the window holds a +0 (the max orders -0 below +0; torch keeps the first zero's sign).  How often that sign agrees with
torch's first zero is recorded.  Its backward
against an fp32 restatement of the kernel: the winner of each window (first maximum, a later NaN replaces it), then the gradients of the
at most 2 x 2 windows that contain the pixel summed in fp32 in (oy, ox) order from +0, rounded once.  subsample2, upsample2_zero,
residual_bwd (fp32 g_a + g_b, zeroed where !(y > 0), one rounding) and add_relu are restated directly.

Refusals.  Odd H or W for stem7x7 (both forms and the weight gradient) and for mb_conv0 (every form and the weight gradient); C % 8 and H or
W not divisible by the stride for the depthwise kernels; dw_wgrad's C <= 1024 && 256 % (C / 8) == 0.  mb_conv0's raw-with-split combination
is refused inside the library too, but no C entry can ask for it.

The CPU tests check the bounds themselves: float32 stand-ins with the kernels' summation orders pass, and plausible wrong variants fail.
Figures go to $YB_PARITY_OUT/plugin_ops_measured.json.
"""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_conv_contract import MEASURED, SENTINEL, bits, check_f16, check_f32, nchw, np64, record, rel_err, rn16, sentinel
from test_train_ops_contract import H100_SMS, R32, sum_err

DEV = 'cuda'
gpu = pytest.mark.gpu
GUARD = 64                  # elements of sentinel past the end of every output
PLUGIN_MEASURED = {}


def _own(group, fn):
    """Run a recording helper of test_conv_contract for `group`, keeping the figures in PLUGIN_MEASURED (written to
    $YB_PARITY_OUT/plugin_ops_measured.json) and out of conv_measured.json."""
    if not group:
        return fn(None)
    key = 'plugin_ops.' + group
    if group in PLUGIN_MEASURED:
        MEASURED[key] = PLUGIN_MEASURED[group]
    try:
        return fn(key)
    finally:
        if key in MEASURED:
            PLUGIN_MEASURED[group] = MEASURED.pop(key)
        out = os.environ.get('YB_PARITY_OUT')
        if out:
            os.makedirs(out, exist_ok=True)
            for name, d in (('conv_measured.json', MEASURED), ('plugin_ops_measured.json', PLUGIN_MEASURED)):
                with open(os.path.join(out, name), 'w') as f:
                    json.dump(d, f, indent=1, sort_keys=True)


def rec(group, **figs):
    _own(group, lambda key: record(key, **figs))


def check16(name, got, ref, E, group=None):
    return _own(group, lambda key: check_f16(name, got, ref, E, key))


def check32(name, got, ref, E, group=None):
    _own(group, lambda key: check_f32(name, got, ref, E, key))


def f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32)


def ref_device():
    return DEV if torch.cuda.is_available() else 'cpu'


# ------------------------------------------------------------------------------------------------------------------------------------
# launch geometry restated from the host code
# ------------------------------------------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def stem_wgrad_geometry(pixels, nsm):
    """stem7x7_wgrad: (L, grid)."""
    grid = max(1, min(cdiv(pixels, 256), 4 * nsm))
    return 16 * cdiv(cdiv(pixels, 16), grid), grid


def dw_wgrad_geometry(pixels, c, nsm):
    """dw_wgrad: (L, lanes, grid)."""
    lanes = 256 // (c // 8)
    grid = max(1, min(cdiv(pixels, lanes * 16), 4 * nsm))
    return cdiv(pixels, grid * lanes), lanes, grid


def conv0_wgrad_geometry(pixels, nsm):
    """mb_conv0_wgrad and stem3x3_s2_wgrad: (L, lanes, grid)."""
    grid = max(1, min(cdiv(pixels, 256), 6 * nsm))
    return cdiv(pixels, grid * 8), 8, grid


def dw_tx(ow):
    """dwconv3x3: output pixels per thread."""
    return 8 if ow >= 52 else 4


# ------------------------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------------------------
def conv_ref(x, w, stride, pad, groups=1):
    """(acc, S) float64 NCHW of F.conv2d on the exact operands and of their absolute values."""
    x, w = x.double(), w.double()
    return (np64(F.conv2d(x, w, None, stride, pad, 1, groups)), np64(F.conv2d(x.abs(), w.abs(), None, stride, pad, 1, groups)))


def bn_relu_ref(acc, E_acc, scale, shift):
    """(ref, E) of max(acc sc + sh, 0) over NCHW."""
    sc, sh = np64(scale).reshape(1, -1, 1, 1), np64(shift).reshape(1, -1, 1, 1)
    lin = sc * acc + sh
    return np.maximum(lin, 0.0), np.abs(sc) * E_acc + 2 * R32 * (np.abs(sc) * (np.abs(acc) + E_acc) + np.abs(sh))


def wgrad_ref(cols_fn, dz, cout, chunks):
    """float64 weight gradient and S: sum over pixels of cols (x) dz, cols_fn(chunk) -> [b, K, P], dz [B, P, cout] in chunks of images."""
    ref = S = None
    for sl in chunks:
        cols = cols_fn(sl)
        g = dz[sl].double()
        r = torch.einsum('bkp,bpc->ck', cols, g)
        s = torch.einsum('bkp,bpc->ck', cols.abs(), g.abs())
        ref, S = (r, s) if ref is None else (ref + r, S + s)
    return np64(ref), np64(S)


def image_chunks(b, per):
    return [slice(i, min(i + per, b)) for i in range(0, b, per)]


def stem_wgrad_ref(x, dz16, stride, pad, k, cout):
    """dw [cout, 3 k k] float64 of a stride-2 conv of the fp32 image x [B,3,H,W] with dz fp16 NHWC [B,oh,ow,cout]."""
    b = x.shape[0]
    dz = dz16.reshape(b, -1, cout)
    per = max(1, (1 << 28) // (x[0].numel() * k * k * 8))
    return wgrad_ref(lambda sl: F.unfold(x[sl].double(), k, padding=pad, stride=stride), dz, cout, image_chunks(b, per))


def dw_wgrad_ref(a16, dz16, stride):
    """dw [C, 9] float64 of the depthwise conv: a fp16 NHWC [B,H,W,C], dz fp16 NHWC [B,oh,ow,C], summed on a's device in chunks of images."""
    b, h, w, c = a16.shape
    oh, ow = h // stride, w // stride
    ref = torch.zeros(c, 9, dtype=torch.float64, device=a16.device)
    S = torch.zeros_like(ref)
    per = max(1, (1 << 27) // (h * w * c))
    for sl in image_chunks(b, per):
        ap = F.pad(a16[sl].double(), (0, 0, 1, 1, 1, 1))
        g = dz16[sl].double()
        for r in range(3):
            for s in range(3):
                t = ap[:, r:r + stride * (oh - 1) + 1:stride, s:s + stride * (ow - 1) + 1:stride, :]
                ref[:, r * 3 + s] += (t * g).sum((0, 1, 2))
                S[:, r * 3 + s] += (t.abs() * g.abs()).sum((0, 1, 2))
    return np64(ref), np64(S)


def pool_taps(x16):
    """The 3x3 stride-2 pad-1 windows of fp16 NHWC x (numpy float16): [9, B, oh, ow, C] values, [9, oh, ow] in-range mask, [9, oh, ow]
    flat input positions, in scan order (rows, then columns)."""
    b, h, w, c = x16.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    pad = np.zeros((b, 2 * oh + 1, 2 * ow + 1, c), dtype=np.float16)
    pad[:, 1:h + 1, 1:w + 1] = x16
    oy, ox = np.meshgrid(np.arange(oh), np.arange(ow), indexing='ij')
    vals, valid, pos = [], [], []
    for r in range(3):
        for s in range(3):
            iy, ix = 2 * oy - 1 + r, 2 * ox - 1 + s
            vals.append(pad[:, 2 * oy + r, 2 * ox + s])
            valid.append((iy >= 0) & (iy < h) & (ix >= 0) & (ix < w))
            pos.append(iy * w + ix)
    return np.stack(vals), np.stack(valid), np.stack(pos)


def pool_winner(x16, last=False):
    """(value, flat position) of every window's winner: the first in-range element, replaced by a later one that is strictly greater or NaN
    (last=True: greater or equal, the wrong variant)."""
    vals, valid, pos = pool_taps(x16)
    v = vals.astype(np.float32)
    best, arg = v[0].copy(), np.broadcast_to(pos[0][None, :, :, None], v[0].shape).copy()
    have = np.broadcast_to(valid[0][None, :, :, None], v[0].shape).copy()
    bestv = vals[0].copy()
    for t in range(1, 9):
        ok = valid[t][None, :, :, None]
        better = (v[t] >= best) if last else (v[t] > best)
        take = ok & (~have | better | np.isnan(v[t]))
        best = np.where(take, v[t], best)
        bestv = np.where(take, vals[t], bestv)
        arg = np.where(take, pos[t][None, :, :, None], arg)
        have |= ok
    return bestv, arg


def pool_bwd_ref(x16, dy16, last=False):
    """The kernel's max-pool backward restated in fp32: dx (numpy float16)."""
    b, h, w, c = x16.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    _, arg = pool_winner(x16, last)
    dy = dy16.astype(np.float32)
    iy, ix = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    me = (iy * w + ix)[None, :, :, None]
    oy0, ox0 = iy // 2, ix // 2
    oy1, ox1 = np.minimum((iy + 1) // 2, oh - 1), np.minimum((ix + 1) // 2, ow - 1)
    acc = np.zeros((b, h, w, c), dtype=np.float32)
    for a in (0, 1):
        for bb in (0, 1):
            oy, ox = oy0 + a, ox0 + bb
            inside = ((oy <= oy1) & (ox <= ox1))[None, :, :, None]
            oyc, oxc = np.minimum(oy, oh - 1), np.minimum(ox, ow - 1)
            hit = inside & (arg[:, oyc, oxc] == me)
            acc = np.where(hit, acc + dy[:, oyc, oxc], acc)
    return acc.astype(np.float16)


def upsample_ref(x16, h, w, variant=None):
    b, _, _, c = x16.shape
    y = np.zeros((b, h, w, c), dtype=np.float16)
    if variant == 'odd_rows':
        rows = np.arange(1, h, 2)
        y[:, 1::2, ::2] = x16[:, rows // 2, :(w + 1) // 2]
    else:
        y[:, ::2, ::2] = x16
    return y


def residual_ref(y16, ga16, gb16, stride):
    f = ga16.astype(np.float32)
    if gb16 is not None:
        if stride == 2:
            up = np.zeros_like(f)
            up[:, ::2, ::2] = gb16.astype(np.float32)
        else:
            up = gb16.astype(np.float32)
        f = f + up
    if y16 is not None:
        f = np.where(y16.astype(np.float32) > 0, f, np.float32(0))
    return f.astype(np.float16)


# ------------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------------
def bn_params(c, gen):
    """scale with negative channels and one 1e-5 channel (outputs near the fp16 subnormal range), shift around 0."""
    scale = torch.rand(c, generator=gen) + 0.5
    scale[1::3] *= -1
    scale[c // 2] = 1e-5
    shift = torch.randn(c, generator=gen) * 0.1
    shift[c // 2] = 0.0
    return scale, shift


def pool_input(shape, seed, nan=False):
    """ReLU output on a coarse grid (all-zero windows and ties), -0 among the zeros, -inf, and NaN when asked."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.relu(torch.randint(-3, 4, shape, generator=g).float()) * 0.5).numpy().astype(np.float16)
    r = torch.rand(shape, generator=g).numpy()
    x[(x == 0) & (r < 0.3)] = np.float16(-0.0)
    x[r > 0.97] = np.float16(-np.inf)
    if nan:
        x[(r > 0.9) & (r <= 0.93)] = np.float16(np.nan)
    return x


def split16(v):
    """[hi | lo] fp16 of float32 v along the last axis."""
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return np.concatenate([hi, lo], -1)


# ------------------------------------------------------------------------------------------------------------------------------------
# CPU: the bounds accept float32 stand-ins and reject plausible wrong variants
# ------------------------------------------------------------------------------------------------------------------------------------
def dw_standin(x16, w9, stride, variant=None):
    """The depthwise forward (raw) in fp32: the 9-tap fmaf chain in the kernel's (s, r) order, reading x through its flat NHWC index.
    Variants: 'hw_swapped' checks a column against H and a row against W; 'strip_at_2px0' starts every stride-2 strip's window at column
    2 px0 instead of 2 px0 - 1."""
    b, h, w, c = x16.shape
    oh, ow = h // stride, w // stride
    flat = x16.reshape(-1, c).astype(np.float64)
    img, oy, ox = np.meshgrid(np.arange(b), np.arange(oh), np.arange(ow), indexing='ij')
    hc, wc = (w, h) if variant == 'hw_swapped' else (h, w)
    acc = np.zeros((b, oh, ow, c), dtype=np.float32)
    for s in range(3):
        for r in range(3):
            iy, ix = oy * stride - 1 + r, ox * stride - 1 + s
            if variant == 'strip_at_2px0' and stride == 2 and s == 0:
                ix = np.where(ox % dw_tx(ow) == 0, ix + 1, ix)
            idx = (img * h + iy) * w + ix
            ok = (iy >= 0) & (iy < hc) & (ix >= 0) & (ix < wc) & (idx >= 0) & (idx < flat.shape[0])
            v = np.where(ok[..., None], flat[np.clip(idx, 0, flat.shape[0] - 1)], 0.0)
            acc = f32(acc.astype(np.float64) + v * w9[:, r * 3 + s].astype(np.float64))
    return acc.astype(np.float16)


def dw_case(b, h, w, c, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, h, w, c, generator=g).half()
    w9 = torch.randn(c, 9, generator=g) * 0.3
    return x, w9


def dw_raw_bound(x, w9, stride):
    c = w9.shape[0]
    acc, S = conv_ref(nchw(x), w9.view(c, 1, 3, 3), stride, 1, c)
    return acc, sum_err(S, 9, 0)


@pytest.mark.parametrize('shape', [(2, 9, 5, 8, 1), (2, 5, 9, 8, 1), (2, 12, 106, 8, 2), (2, 106, 12, 16, 2), (1, 8, 102, 8, 2)],
                         ids=lambda s: '%dx%dx%d_C%d_s%d' % s)
def test_depthwise_bound_accepts_standin_and_rejects_variants(shape):
    b, h, w, c, stride = shape
    x, w9 = dw_case(b, h, w, c, h * w + c)
    acc, E = dw_raw_bound(x, w9, stride)
    xn, wn = x.numpy(), w9.numpy()
    check16('stand-in', nchw(torch.from_numpy(dw_standin(xn, wn, stride))), acc, E)
    variants = ['hw_swapped'] + (['strip_at_2px0'] if stride == 2 else [])
    for variant in variants:
        got = nchw(torch.from_numpy(dw_standin(xn, wn, stride, variant)))
        with pytest.raises(AssertionError, match='^' + variant):
            check16(variant, got, acc, E)


def test_hw_swap_is_invisible_on_square_shapes():
    """Why every depthwise case has H != W: on a square input the swapped index is the right one."""
    x, w9 = dw_case(2, 10, 10, 8, 3)
    for stride in (1, 2):
        acc, E = dw_raw_bound(x, w9, stride)
        check16('hw_swapped', nchw(torch.from_numpy(dw_standin(x.numpy(), w9.numpy(), stride, 'hw_swapped'))), acc, E)


def test_stem_bound_accepts_fp32_chain():
    """stem7x7 and mb_conv0 as fp32 fmaf chains in (ci, r, s) order, checked against their bounds."""
    g = torch.Generator().manual_seed(7)
    for k, pad, cout in ((7, 3, 64), (3, 1, 32), (3, 0, 32)):
        x = torch.rand(2, 3, 11, 14, generator=g)
        wt = torch.randn(cout, 3, k, k, generator=g) * 0.2
        acc, S = conv_ref(x, wt, 2, pad)
        cols = F.unfold(x.double(), k, padding=pad, stride=2).numpy()                     # [B, 3 k k, P] in (ci, r, s) order
        wf = wt.reshape(cout, -1).double().numpy()
        a = np.zeros((cols.shape[0], cout, cols.shape[2]), dtype=np.float32)
        for t in range(cols.shape[1]):
            a = f32(a.astype(np.float64) + cols[:, t][:, None, :] * wf[:, t][None, :, None])
        check16('stem k%d chain' % k, a.reshape(acc.shape).astype(np.float16), acc, sum_err(S, 3 * k * k, 0))


def test_split_bound_accepts_fp32_split():
    """hi = RN16(v), lo = RN16(v - hi) of an fp32 v within E of ref: both checks pass, and hi + lo is closer to ref than hi alone."""
    g = torch.Generator().manual_seed(9)
    ref = (torch.randn(4000, generator=g).double() * torch.logspace(-7, 1, 4000, dtype=torch.float64)).numpy()
    E = 1e-6 * np.abs(ref)
    v = f32(ref + 0.9 * E * (torch.rand(4000, generator=g).double().numpy() * 2 - 1))      # plus its fp32 rounding: within E
    hl = split16(v[:, None])
    hi, lo = hl[:, 0].astype(np.float64), hl[:, 1].astype(np.float64)
    check_f16('hi', hi, ref, E)
    check_f16('lo', lo, ref - hi, E)
    assert np.all(np.abs(hi + lo - ref) <= np.abs(hi - ref) + 2.0 ** -25)


def test_maxpool_restatement_rejects_last_maximum():
    """The backward restatement is bit-exact: routing ties to the last maximum changes the bits of the tie-heavy inputs."""
    for shape in ((2, 7, 4, 8), (1, 3, 2, 8), (3, 13, 10, 16)):
        x = pool_input(shape, sum(shape))
        dy = (torch.randn((shape[0], (shape[1] + 1) // 2, (shape[2] + 1) // 2, shape[3]), generator=torch.Generator().manual_seed(1))
              .half().numpy())
        good, wrong = pool_bwd_ref(x, dy), pool_bwd_ref(x, dy, last=True)
        assert not np.array_equal(good.view(np.int16), wrong.view(np.int16)), shape


def test_maxpool_restatement_outputs_nan():
    """torch's forward rule on a window holding a NaN: NaN.  A max that drops NaN operands (the pre-fix __hmax2) gives a finite value there."""
    x = pool_input((2, 9, 6, 8), 5, nan=True)
    best, _ = pool_winner(x)
    vals, valid, _ = pool_taps(x)
    has_nan = (np.isnan(vals.astype(np.float32)) & valid[:, None, :, :, None]).any(0)
    assert has_nan.any() and np.array_equal(np.isnan(best.astype(np.float32)), has_nan)
    dropped = np.where(valid[:, None, :, :, None] & ~np.isnan(vals.astype(np.float32)), vals.astype(np.float32), -np.inf).max(0)
    assert not np.isnan(dropped[has_nan]).any()


def test_upsample_restatement_rejects_odd_rows():
    x = torch.randn(2, 4, 5, 8, generator=torch.Generator().manual_seed(2)).half().numpy()
    for h, w in ((7, 9), (8, 10)):
        assert not np.array_equal(upsample_ref(x, h, w), upsample_ref(x, h, w, 'odd_rows'))


def emulated_stem_wgrad_one_weight(pixels, nsm, term):
    """One stem weight's sum in the kernel's order: CTA i walks slabs i, i + grid, ... in fp32 (fmaf, exact product), then the CTA partials
    are added in fp32 (one order of the global atomics).  Every pixel contributes the same product `term`."""
    L, grid = stem_wgrad_geometry(pixels, nsm)
    slabs = cdiv(pixels, 16)
    n = np.zeros(grid, dtype=np.int64)                    # real pixels per CTA
    for cta in range(grid):
        own = np.arange(cta, slabs, grid)
        n[cta] = np.minimum(16, pixels - 16 * own).sum()
    acc = np.zeros(grid, dtype=np.float32)
    t = np.float64(term)
    for k in range(int(n.max())):
        acc = np.where(k < n, f32(acc.astype(np.float64) + t), acc)
    total = np.float32(0)
    for p in acc:
        total = np.float32(total + p)
    return float(total), L, grid


def test_wgrad_bound_needs_the_whole_chain():
    """The stem's weight gradient at 64 x 416^2 on 132 SMs: a thread's chain is 5248 fmaf long.  An fp32 stand-in with that order stays
    within (L + grid + 2) u S but not within the bound of one slab (L = 16): a bound without the chain would fail a correct kernel."""
    pixels = 64 * 208 * 208
    term = float(np.float32(0.9))
    got, L, grid = emulated_stem_wgrad_one_weight(pixels, H100_SMS, term)
    S = pixels * term
    err = abs(got - S)
    assert (L, grid) == (5248, 528)
    assert err <= sum_err(S, L + grid + 2, pixels)
    assert err > sum_err(S, 16 + grid + 2, pixels), (err / S, 16 + grid + 2)
    rec('wgrad_chain_standin', err_over_bound=err / sum_err(S, L + grid + 2, pixels), err_over_one_slab_bound=err / sum_err(S, 18 + grid,
                                                                                                                            pixels))


def test_rel_err_misses_what_the_bound_sees():
    """A 10 % error on an element 1e-4 of the largest output: max|d| / max|ref| <= 1e-3 accepts it, the element-wise bound does not."""
    x, w9 = dw_case(2, 9, 14, 8, 4)
    w9[3] *= 1e-4                                             # channel 3: outputs about 1e-4 of the others
    acc, E = dw_raw_bound(x, w9, 1)
    y = nchw(torch.from_numpy(dw_standin(x.numpy(), w9.numpy(), 1))).numpy().copy()
    check16('stand-in', y, acc, E)
    top = np.abs(acc).max()
    i = np.unravel_index(np.argmax(np.abs(acc[:, 3])), acc[:, 3].shape)
    i = (i[0], 3) + i[1:]
    assert 0.3e-4 * top <= abs(acc[i]) <= 3e-4 * top
    y[i] = np.float16(acc[i] * 1.1)
    assert rel_err(y, acc) <= 1e-3
    with pytest.raises(AssertionError, match='^ten_percent'):
        check16('ten_percent', y, acc, E)


def test_geometry_at_the_training_sizes():
    """The chains the weight-gradient bounds are made of, on 132 SMs."""
    assert stem_wgrad_geometry(64 * 208 * 208, H100_SMS) == (5248, 528)
    assert stem_wgrad_geometry(7, H100_SMS) == (16, 1) and stem_wgrad_geometry(256, H100_SMS) == (256, 1)
    assert stem_wgrad_geometry(256 * 528 + 16, H100_SMS) == (16 * 17, 528)
    assert conv0_wgrad_geometry(32 * 208 * 208, H100_SMS) == (219, 8, 792)
    assert dw_wgrad_geometry(32 * 208 * 208, 32, H100_SMS) == (41, 64, 528)
    assert dw_wgrad_geometry(32 * 13 * 13, 1024, H100_SMS) == (16, 2, 169)
    assert [dw_tx(ow) for ow in (1, 2, 51, 52, 53, 60)] == [4, 4, 4, 8, 8, 8]


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def out16(shape):
    """(buffer, view): an fp16 output of `shape` followed by GUARD elements, all SENTINEL."""
    n = int(np.prod(shape))
    buf = sentinel((n + GUARD,))
    return buf, buf[:n].view(shape)


def out32(shape):
    n = int(np.prod(shape))
    buf = torch.full((n + GUARD,), float('nan'), device=DEV)
    return buf, buf[:n].view(shape)


def guard_kept(buf, shape):
    n = int(np.prod(shape))
    return bool((bits(buf[n:]) == SENTINEL).all())


def untouched16(buf):
    torch.cuda.synchronize()
    return bool((bits(buf) == SENTINEL).all())


def dev(t):
    return torch.as_tensor(t).to(DEV)


def hw_id(c):
    return 'x'.join(str(v) for v in c)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: ResNet stem
# ------------------------------------------------------------------------------------------------------------------------------------
STEM_SHAPES = [
    # b, h, w
    (3, 2, 2),          # a 1 x 1 output: 33 of the 49 taps of each channel are padding
    (2, 32, 96),
    (2, 96, 32),
    (1, 6, 418),
    (2, 30, 46),        # 690 pixels: not a multiple of 128
    (2, 64, 96),
    (2, 32, 48),
    (1, 64, 32),
    (1, 416, 416),
]


def stem_inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, 3, h, w, generator=g)
    wt = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    return x, wt, *bn_params(64, g)


def check_stem_forward(ops, tag, x, wt, scale, shift, b, h, w, group, keep=None):
    """Both forms on x (device); keep = the slice of images checked (all by default)."""
    keep = keep or slice(0, b)
    acc, S = conv_ref(x[keep], wt.to(x.device), 2, 3)
    E_acc = sum_err(S, 147, 0)
    shp = (b, h // 2, w // 2, 64)
    zb, z = out16(shp)
    ops.call('yb_stem7x7_raw_fwd', x, dev(wt), z, b, h, w)
    check16('stem7x7 raw %s' % tag, nchw(z[keep]), acc, E_acc, group + '_raw')
    assert guard_kept(zb, shp), 'stem7x7 raw wrote past its output'
    yb, y = out16(shp)
    ops.call('yb_stem7x7_bn_relu_fwd', x, dev(wt), dev(scale), dev(shift), y, b, h, w)
    ref, E = bn_relu_ref(acc, E_acc, scale, shift)
    check16('stem7x7 bn_relu %s' % tag, nchw(y[keep]), ref, E, group + '_bn_relu')
    assert guard_kept(yb, shp), 'stem7x7 bn_relu wrote past its output'


@gpu
@pytest.mark.parametrize('shape', STEM_SHAPES, ids=hw_id)
def test_stem7x7_forward_vs_float64(ops, shape):
    b, h, w = shape
    x, wt, scale, shift = stem_inputs(b, h, w, b + h * 3 + w)
    check_stem_forward(ops, '%dx%dx%d' % shape, dev(x), wt, scale, shift, b, h, w, 'stem7x7')


@gpu
def test_stem7x7_forward_last_image_of_a_416_batch(ops):
    """64 x 416^2: 2.8 M output pixels, 21632 CTAs; the last image is checked (its pixels are the highest indices of the grid)."""
    b, h, w = 64, 416, 416
    x = torch.rand(b, 3, h, w, generator=torch.Generator(device=DEV).manual_seed(64), device=DEV)
    _, wt, scale, shift = stem_inputs(1, 2, 2, 64)
    check_stem_forward(ops, '64x416x416 last image', x, wt, scale, shift, b, h, w, 'stem7x7_416', keep=slice(b - 1, b))


@gpu
def test_stem7x7_refusals_leave_the_output_untouched(ops):
    wt, one = torch.randn(64, 3, 7, 7, device=DEV), torch.ones(64, device=DEV)
    for h, w in ((33, 32), (32, 33)):
        x = torch.rand(1, 3, h, w, device=DEV)
        yb, y = out16((1, h // 2, w // 2, 64))
        with pytest.raises(RuntimeError):
            ops.call('yb_stem7x7_bn_relu_fwd', x, wt, one, one, y, 1, h, w)
        with pytest.raises(RuntimeError):
            ops.call('yb_stem7x7_raw_fwd', x, wt, y, 1, h, w)
        dz = torch.zeros(1, h // 2, w // 2, 64, dtype=torch.float16, device=DEV)
        dw = torch.full((64 * 147,), 7.0, device=DEV)
        with pytest.raises(RuntimeError):
            ops.call('yb_stem7x7_wgrad', x, dz, dw, 1, h, w)
        assert untouched16(yb) and bool((dw == 7.0).all()), (h, w)


def stem_wgrad_cases():
    cap_plus_one = (1, 32, 2 * (16 * 4 * sms() + 1)) if torch.cuda.is_available() else (1, 32, 2 * (16 * 4 * H100_SMS + 1))
    return [('one_partial_slab', (1, 4, 6)), ('256_pixels', (1, 32, 32)), ('one_slab_past_the_cap', cap_plus_one),
            ('2x32x48', (2, 32, 48)), ('1x64x32', (1, 64, 32)), ('3x30x46', (3, 30, 46))]


def check_stem_wgrad(ops, tag, x, dz, b, h, w, group):
    dwb, dw = out32((64, 3, 7, 7))
    ops.call('yb_stem7x7_wgrad', x, dz, dw, b, h, w)
    pixels = b * (h // 2) * (w // 2)
    L, grid = stem_wgrad_geometry(pixels, sms())
    ref, S = stem_wgrad_ref(x, dz, 2, 3, 7, 64)
    ref, S = ref.reshape(64, 3, 7, 7), S.reshape(64, 3, 7, 7)
    E = sum_err(S, L + grid + 2, pixels)
    check32('stem7x7_wgrad %s' % tag, dw, ref, E, group)
    assert bool(dwb[dw.numel():].isnan().all()), 'stem7x7_wgrad wrote past dw'
    return np.abs(np64(dw) - ref), E, ref


@gpu
@pytest.mark.parametrize('case', range(6), ids=lambda i: stem_wgrad_cases()[i][0])
def test_stem7x7_wgrad_vs_float64(ops, case):
    """dw pre-filled with NaN: the host's memset is what the atomics add to."""
    name, (b, h, w) = stem_wgrad_cases()[case]
    g = torch.Generator().manual_seed(h + w)
    x = torch.rand(b, 3, h, w, generator=g)
    dz = (torch.randn(b, h // 2, w // 2, 64, generator=g) * 0.1).half()
    check_stem_wgrad(ops, name, dev(x), dev(dz), b, h, w, 'stem7x7_wgrad')


@gpu
def test_stem7x7_wgrad_at_training_size(ops):
    """64 x 416^2: grid capped at 4 SMs, a 5248-long fp32 chain per thread on 132 SMs; float64 reference on the device."""
    b, h, w = 64, 416, 416
    gen = torch.Generator(device=DEV).manual_seed(416)
    x = torch.rand(b, 3, h, w, generator=gen, device=DEV)
    dz = (torch.randn(b, h // 2, w // 2, 64, generator=gen, device=DEV) * 0.05).half()
    err, E, ref = check_stem_wgrad(ops, '64x416x416', x, dz, b, h, w, 'stem7x7_wgrad_416')
    L, grid = stem_wgrad_geometry(b * (h // 2) * (w // 2), sms())
    rec('stem7x7_wgrad_416', chain=L, grid=grid, err_over_dw=float((err / np.maximum(np.abs(ref), 1e-30)).max()),
        err_over_dw_median=float(np.median(err / np.maximum(np.abs(ref), 1e-30))))


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: 3x3 stride-2 max-pool, forward and backward
# ------------------------------------------------------------------------------------------------------------------------------------
POOL_SHAPES = [
    # b, h, w, c
    (2, 1, 1, 8), (1, 1, 4, 64), (2, 2, 3, 8), (1, 3, 2, 64), (2, 4, 7, 8), (1, 7, 4, 64), (3, 13, 10, 16), (2, 9, 16, 8),
    (2, 16, 16, 64), (1, 13, 10, 16), (1, 13, 27, 8), (2, 32, 48, 64), (3, 208, 208, 64),
]


def pool_plus_zero(x16):
    """The sign of a zero maximum under an fp16 max that orders -0 below +0: +0 when any in-range element of the window is +0."""
    vals, valid, _ = pool_taps(x16)
    return ((vals.view(np.int16) == 0) & valid[:, None, :, :, None]).any(0)


def check_pool_forward(tag, y, x16, group):
    """Bits against torch's rule; NaN windows by NaN-ness (the payload is the device's); a zero maximum by value, its sign against the
    +0-over--0 rule of the kernel's max (torch keeps the first zero's sign instead; both agreements are recorded)."""
    best, _ = pool_winner(x16)
    got = y.cpu().numpy()
    gb, rb = got.view(np.int16), best.view(np.int16)
    nan = np.isnan(best.astype(np.float32))
    assert np.array_equal(np.isnan(got.astype(np.float32)), nan), '%s: NaN windows differ (%d expected, %d got)' % (
        tag, nan.sum(), np.isnan(got.astype(np.float32)).sum())
    zero = ~nan & (best.astype(np.float32) == 0)
    same = (gb == rb) | nan | zero
    assert same.all(), '%s: %d outputs differ in bits from the first maximum' % (tag, (~same).sum())
    assert np.array_equal(got[zero].astype(np.float32), best[zero].astype(np.float32))
    plus = pool_plus_zero(x16)[zero]
    rec(group, zero_outputs=int(zero.sum()), zero_sign_as_first_max=int((gb[zero] == rb[zero]).sum()),
        zero_sign_plus_over_minus=int(((gb[zero] == 0) == plus).sum()), nan_windows=int(nan.sum()))
    assert np.array_equal(gb[zero] == 0, plus), '%s: the sign of a zero maximum is not +0-over--0' % tag


@gpu
@pytest.mark.parametrize('nan', [False, True], ids=['ties', 'nan'])
@pytest.mark.parametrize('shape', POOL_SHAPES, ids=hw_id)
def test_maxpool3x3_forward_and_backward(ops, shape, nan):
    b, h, w, c = shape
    x = pool_input(shape, h * 31 + w + c, nan)
    oshape = (b, (h + 1) // 2, (w + 1) // 2, c)
    yb, y = out16(oshape)
    ops.call('yb_maxpool3x3_s2_f16', dev(x), y, b, h, w, c)
    assert guard_kept(yb, oshape), 'maxpool3x3_s2 wrote past its output'
    check_pool_forward('maxpool3x3_s2 %s' % hw_id(shape), y, x, 'maxpool3x3_fwd_nan' if nan else 'maxpool3x3_fwd')
    dy = (torch.randn(oshape, generator=torch.Generator().manual_seed(c + h)) * 0.5).half().numpy()
    dxb, dx = out16(shape)
    ops.call('yb_maxpool3x3_s2_bwd_f16', dev(x), dev(dy), dx, b, h, w, c)
    assert guard_kept(dxb, shape), 'maxpool3x3_s2_bwd wrote past its output'
    want = pool_bwd_ref(x, dy)
    got = dx.cpu().numpy()
    assert np.array_equal(got.view(np.int16), want.view(np.int16)), 'maxpool3x3_s2_bwd: %d of %d elements differ' % (
        (got.view(np.int16) != want.view(np.int16)).sum(), got.size)
    rec('maxpool3x3_bwd', elements=got.size, exact=got.size)


@gpu
def test_maxpool3x3_nan_window_outputs_nan_in_every_form(ops):
    """A window holding a NaN gives NaN in the three forms that share the window (plain, channel slice, valid padding)."""
    b, h, w, c = 2, 9, 6, 16
    x = pool_input((b, h, w, c), 77, nan=True)
    oh, ow = (h + 1) // 2, (w + 1) // 2
    yb, y = out16((b, oh, ow, c))
    ops.call('yb_maxpool3x3_s2_f16', dev(x), y, b, h, w, c)
    check_pool_forward('plain', y, x, 'maxpool3x3_fwd_nan')
    ld = sentinel((b, oh, ow, c + 16))
    ops.call('yb_maxpool3x3_s2_ld_f16', dev(x), ld, c + 16, 8, b, h, w, c)
    assert torch.equal(bits(ld[..., 8:8 + c]), bits(y)), 'the channel-slice form differs from the plain one'
    assert bool((bits(ld[..., :8]) == SENTINEL).all()) and bool((bits(ld[..., 8 + c:]) == SENTINEL).all())
    vh, vw = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    yv = sentinel((b, vh, vw, c))
    ops.call('yb_maxpool3x3_s2_valid_f16', dev(x), yv, c, 0, b, h, w, c)
    xt = torch.from_numpy(x.astype(np.float32)).permute(0, 3, 1, 2)
    ref = F.max_pool2d(xt, 3, 2).permute(0, 2, 3, 1).numpy()
    got = yv.float().cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.isnan(ref).any(), 'valid pool: NaN windows differ from torch'
    ok = ~np.isnan(ref)
    assert np.array_equal(got[ok], ref[ok])


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: data movement
# ------------------------------------------------------------------------------------------------------------------------------------
MOVE_SHAPES = [(2, 14, 10, 64), (1, 7, 9, 8), (2, 1, 1, 8), (1, 2, 5, 16), (3, 5, 2, 8), (2, 32, 48, 64), (1, 13, 27, 8), (3, 208, 208, 64)]


@gpu
@pytest.mark.parametrize('shape', MOVE_SHAPES, ids=hw_id)
def test_subsample2_and_upsample2_zero_bit_exact(ops, shape):
    b, h, w, c = shape
    g = torch.Generator().manual_seed(h * w + c)
    x = torch.randn(b, h, w, c, generator=g).half()
    oshape = (b, (h + 1) // 2, (w + 1) // 2, c)
    yb, y = out16(oshape)
    ops.call('yb_subsample2_f16', dev(x), y, b, h, w, c)
    assert torch.equal(bits(y.cpu()), bits(x[:, ::2, ::2])) and guard_kept(yb, oshape), 'subsample2'
    xs = torch.randn(oshape, generator=g).half()
    ub, u = out16(shape)
    ops.call('yb_upsample2_zero_f16', dev(xs), u, b, h, w, c)
    want = upsample_ref(xs.numpy(), h, w)
    assert np.array_equal(u.cpu().numpy().view(np.int16), want.view(np.int16)) and guard_kept(ub, shape), 'upsample2_zero'


RESIDUAL_COMBOS = [(1, True, True), (2, True, True), (1, False, True), (2, True, False), (1, True, False)]     # stride_b, g_b, mask


@gpu
@pytest.mark.parametrize('shape', [(2, 10, 12, 32), (2, 7, 9, 8), (1, 1, 3, 16), (3, 5, 1, 8)], ids=hw_id)
@pytest.mark.parametrize('combo', RESIDUAL_COMBOS, ids=lambda c: 's%d_%s_%s' % (c[0], 'gb' if c[1] else 'nogb', 'mask' if c[2] else 'nomask'))
def test_residual_bwd_bit_exact(ops, shape, combo):
    b, h, w, c = shape
    stride, with_b, with_mask = combo
    g = torch.Generator().manual_seed(h * 7 + w + c + stride)
    y = torch.relu(torch.randn(b, h, w, c, generator=g)).half().numpy()
    y.flat[np.flatnonzero(y == 0)[::2]] = np.float16(-0.0)                               # +0 and -0 both mask
    ga = torch.randn(b, h, w, c, generator=g).half().numpy()
    gb = torch.randn(b, (h + 1) // 2 if stride == 2 else h, (w + 1) // 2 if stride == 2 else w, c, generator=g).half().numpy() if with_b else None
    ob, out = out16(shape)
    ops.call('yb_residual_bwd_f16', dev(y) if with_mask else None, dev(ga), None if gb is None else dev(gb), stride, out, b, h, w, c)
    want = residual_ref(y if with_mask else None, ga, gb, stride)
    assert np.array_equal(out.cpu().numpy().view(np.int16), want.view(np.int16)), 'residual_bwd %s %s' % (shape, combo)
    assert guard_kept(ob, shape), 'residual_bwd wrote past its output'


@gpu
@pytest.mark.parametrize('count', [8, 5 * 13 * 13 * 512, 8 * 1000 + 8])
def test_add_relu_bit_exact_and_in_place(ops, count):
    g = torch.Generator().manual_seed(count)
    a = torch.randn(count, generator=g).half()
    r = torch.randn(count, generator=g).half()
    want = np.maximum(a.numpy().astype(np.float32) + r.numpy().astype(np.float32), np.float32(0)).astype(np.float16)
    ob, out = out16((count,))
    ops.call('yb_add_relu_f16', dev(a), dev(r), out, count)
    assert np.array_equal(out.cpu().numpy().view(np.int16), want.view(np.int16)) and guard_kept(ob, (count,))
    ab, ad = out16((count,))
    ad.copy_(dev(a))
    ops.call('yb_add_relu_f16', ad, dev(r), ad, count)                                  # in place, as the blocks use it
    assert np.array_equal(ad.cpu().numpy().view(np.int16), want.view(np.int16)) and guard_kept(ab, (count,))
    with pytest.raises(RuntimeError):
        ops.call('yb_add_relu_f16', dev(a), dev(r), out, count - 4)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: MobileNet first layer, and Inception's pad-0 stem in training
# ------------------------------------------------------------------------------------------------------------------------------------
CONV0_SHAPES = [(3, 2, 2), (2, 32, 48), (2, 48, 32), (1, 6, 418), (2, 30, 46)]


def conv0_inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, 3, h, w, generator=g)
    wt = torch.randn(32, 3, 3, 3, generator=g) * 0.2
    return x, wt, *bn_params(32, g)


def check_split(name, hl, ref, E, c, group):
    hi, lo = hl[..., :c], hl[..., c:]
    check16(name + ' hi', nchw(hi), ref, E, group + '_hi')
    check16(name + ' lo', nchw(lo), ref - np64(nchw(hi)), E, group + '_lo')
    return hi


@gpu
@pytest.mark.parametrize('shape', CONV0_SHAPES, ids=hw_id)
def test_mb_conv0_forms_vs_float64(ops, shape):
    b, h, w = shape
    x, wt, scale, shift = conv0_inputs(b, h, w, h + w * 5 + b)
    acc, S = conv_ref(x, wt, 2, 1)
    E_acc = sum_err(S, 27, 0)
    oshape = (b, h // 2, w // 2, 32)
    args = (dev(x), dev(wt))
    zb, z = out16(oshape)
    ops.call('yb_mb_conv0_raw_fwd', *args, z, b, h, w)
    check16('mb_conv0 raw', nchw(z), acc, E_acc, 'mb_conv0_raw')
    yb, y = out16(oshape)
    ops.call('yb_mb_conv0_bn_relu_fwd', *args, dev(scale), dev(shift), y, b, h, w)
    ref, E = bn_relu_ref(acc, E_acc, scale, shift)
    check16('mb_conv0 bn_relu', nchw(y), ref, E, 'mb_conv0_bn_relu')
    sshape = (b, h // 2, w // 2, 64)
    sb, s = out16(sshape)
    ops.call('yb_mb_conv0_split_fwd', *args, dev(scale), dev(shift), s, b, h, w)
    hi = check_split('mb_conv0 split', s, ref, E, 32, 'mb_conv0_split')
    assert torch.equal(bits(hi), bits(y)), 'mb_conv0 split: hi differs from the BatchNorm form'
    assert guard_kept(zb, oshape) and guard_kept(yb, oshape) and guard_kept(sb, sshape), 'mb_conv0 wrote past its output'
    # pad 1 of the Inception entries is the same kernel
    zs = sentinel(oshape)
    ops.call('yb_stem3x3_s2_raw_fwd', *args, zs, b, h, w, 1)
    assert torch.equal(bits(zs), bits(z)), 'stem3x3_s2_raw at pad 1 differs from mb_conv0_raw'


@gpu
def test_mb_conv0_refusals_leave_the_output_untouched(ops):
    wt, one = torch.randn(32, 3, 3, 3, device=DEV), torch.ones(32, device=DEV)
    for h, w in ((9, 8), (8, 9)):
        x = torch.rand(1, 3, h, w, device=DEV)
        yb, y = out16((1, h // 2 + 1, w // 2 + 1, 64))
        for name, extra in (('yb_mb_conv0_bn_relu_fwd', (one, one)), ('yb_mb_conv0_split_fwd', (one, one)), ('yb_mb_conv0_raw_fwd', ())):
            with pytest.raises(RuntimeError):
                ops.call(name, x, wt, *extra, y, 1, h, w)
        dw = torch.full((32 * 27,), 7.0, device=DEV)
        with pytest.raises(RuntimeError):
            ops.call('yb_mb_conv0_wgrad', x, torch.zeros(1, 5, 5, 32, dtype=torch.float16, device=DEV), dw, 1, h, w)
        assert untouched16(yb) and bool((dw == 7.0).all()), (h, w)


def check_conv0_wgrad(ops, entry, x, dz, b, h, w, pad, group, extra=()):
    dwb, dw = out32((32, 3, 3, 3))
    ops.call(entry, x, dz, dw, b, h, w, *extra)
    pixels = dz.shape[0] * dz.shape[1] * dz.shape[2]
    L, lanes, grid = conv0_wgrad_geometry(pixels, sms())
    ref, S = stem_wgrad_ref(x, dz, 2, pad, 3, 32)
    ref, S = ref.reshape(32, 3, 3, 3), S.reshape(32, 3, 3, 3)
    check32('%s %dx%dx%d' % (entry, b, h, w), dw, ref, sum_err(S, L + lanes + grid, pixels), group)
    assert bool(dwb[dw.numel():].isnan().all()), '%s wrote past dw' % entry
    return np.abs(np64(dw) - ref), ref, L, grid


@gpu
@pytest.mark.parametrize('shape', [(1, 3, 4), (2, 7, 5), (1, 107, 139), (2, 139, 107)], ids=hw_id)
def test_stem3x3_s2_pad0_raw_and_wgrad(ops, shape):
    """Inception-v3's Conv2d_1a_3x3 in training: the raw output and the weight gradient at pad 0 on odd, non-square inputs."""
    b, h, w = shape
    x, wt, _, _ = conv0_inputs(b, h, w, h * 3 + w)
    acc, S = conv_ref(x, wt, 2, 0)
    oshape = (b, (h - 3) // 2 + 1, (w - 3) // 2 + 1, 32)
    zb, z = out16(oshape)
    ops.call('yb_stem3x3_s2_raw_fwd', dev(x), dev(wt), z, b, h, w, 0)
    check16('stem3x3_s2 raw pad 0', nchw(z), acc, sum_err(S, 27, 0), 'stem3x3_raw_pad0')
    assert guard_kept(zb, oshape)
    dz = (torch.randn(oshape, generator=torch.Generator().manual_seed(h)) * 0.1).half()
    check_conv0_wgrad(ops, 'yb_stem3x3_s2_wgrad', dev(x), dev(dz), b, h, w, 0, 'stem3x3_wgrad_pad0', (0,))


def conv0_wgrad_cases():
    n = sms() if torch.cuda.is_available() else H100_SMS
    return [(3, 2, 2), (2, 32, 48), (2, 48, 32), (1, 34, 2 * (16 * 6 * n + 1))]          # the last: more than 256 pixels per CTA at the cap


@gpu
@pytest.mark.parametrize('case', range(4), ids=lambda i: hw_id(conv0_wgrad_cases()[i]))
def test_mb_conv0_wgrad_vs_float64(ops, case):
    b, h, w = conv0_wgrad_cases()[case]
    g = torch.Generator().manual_seed(h + w)
    x = torch.rand(b, 3, h, w, generator=g)
    dz = (torch.randn(b, h // 2, w // 2, 32, generator=g) * 0.1).half()
    check_conv0_wgrad(ops, 'yb_mb_conv0_wgrad', dev(x), dev(dz), b, h, w, 1, 'mb_conv0_wgrad')


@gpu
def test_mb_conv0_wgrad_at_training_size(ops):
    b, h, w = 32, 416, 416
    gen = torch.Generator(device=DEV).manual_seed(32)
    x = torch.rand(b, 3, h, w, generator=gen, device=DEV)
    dz = (torch.randn(b, h // 2, w // 2, 32, generator=gen, device=DEV) * 0.05).half()
    err, ref, L, grid = check_conv0_wgrad(ops, 'yb_mb_conv0_wgrad', x, dz, b, h, w, 1, 'mb_conv0_wgrad_416')
    rec('mb_conv0_wgrad_416', chain=L, grid=grid, err_over_dw=float((err / np.maximum(np.abs(ref), 1e-30)).max()),
        err_over_dw_median=float(np.median(err / np.maximum(np.abs(ref), 1e-30))))


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: depthwise forward (plain, raw, split)
# ------------------------------------------------------------------------------------------------------------------------------------
OWS = (1, 2, 51, 52, 53, 60)          # tx = 4 below 52, 8 from 52; ragged last strips at 1, 2, 51, 53, 60


def dw_fwd_shapes(stride):
    """(h, w) with output width ow in OWS, taller and wider than ow, never square."""
    out = []
    for ow in OWS:
        out.append(((ow + 3) * stride, ow * stride))
        if ow >= 2:
            out.append(((ow // 2) * stride, ow * stride))
    return out


def dw_fwd_check(ops, tag, b, h, w, c, stride, seed, group):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, h, w, c, generator=g).half()
    w9 = torch.randn(c, 9, generator=g) * 0.3
    scale, shift = bn_params(c, g)
    rd = ref_device()
    acc, S = conv_ref(nchw(x.to(rd)), w9.to(rd).view(c, 1, 3, 3), stride, 1, c)
    E_acc = sum_err(S, 9, 0)
    oshape = (b, h // stride, w // stride, c)
    xd, wd, scd, shd = dev(x), dev(w9), dev(scale), dev(shift)
    zb, z = out16(oshape)
    ops.call('yb_dwconv3x3_raw_fwd', xd, wd, z, b, h, w, c, stride)
    check16('dwconv raw %s' % tag, nchw(z), acc, E_acc, group + '_raw')
    yb, y = out16(oshape)
    ops.call('yb_dwconv3x3_bn_relu_fwd', xd, wd, scd, shd, y, b, h, w, c, stride)
    ref, E = bn_relu_ref(acc, E_acc, scale, shift)
    check16('dwconv bn_relu %s' % tag, nchw(y), ref, E, group + '_bn_relu')
    assert guard_kept(zb, oshape) and guard_kept(yb, oshape), 'dwconv3x3 wrote past its output (%s)' % tag
    # strict form: x = [hi | lo] of an fp32 activation, the sum on the exact hi + lo
    v = (torch.randn(b, h, w, c, generator=g) * 1.3).numpy().astype(np.float32)
    xs = split16(v)
    xe = xs[..., :c].astype(np.float64) + xs[..., c:].astype(np.float64)
    acc2, S2 = conv_ref(nchw(torch.from_numpy(xe).to(rd)), w9.to(rd).view(c, 1, 3, 3), stride, 1, c)
    ref2, E2 = bn_relu_ref(acc2, sum_err(S2, 10, 0), scale, shift)
    sshape = oshape[:3] + (2 * c,)
    sb, s = out16(sshape)
    ops.call('yb_dwconv3x3_split_fwd', dev(xs), wd, scd, shd, s, b, h, w, c, stride)
    check_split('dwconv split %s' % tag, s, ref2, E2, c, group + '_split')
    assert guard_kept(sb, sshape), 'dwconv3x3_split wrote past its output (%s)' % tag


@gpu
@pytest.mark.parametrize('c', [8, 24, 40, 1024])
@pytest.mark.parametrize('stride', [1, 2])
def test_dwconv3x3_forward_strips_vs_float64(ops, stride, c):
    b = 1 if c == 1024 else 2
    for h, w in dw_fwd_shapes(stride):
        dw_fwd_check(ops, '%dx%dx%d C%d s%d' % (b, h, w, c, stride), b, h, w, c, stride, h * 131 + w + c, 'dwconv_fwd')


# the depthwise cases of the plugin's inference and training tests (square, as the model runs them), and non-square ones
DW_CASES = [
    # b, h, w, c, stride
    (2, 13, 13, 1024, 1), (3, 52, 52, 128, 2), (2, 7, 7, 64, 1), (1, 60, 60, 32, 1), (2, 26, 26, 256, 1), (2, 26, 26, 256, 2),
    (1, 104, 104, 64, 2), (2, 12, 12, 64, 1), (2, 12, 12, 64, 2), (1, 26, 26, 256, 2), (3, 13, 13, 1024, 1),
    (2, 2, 2, 16, 2), (2, 6, 14, 32, 2), (2, 14, 6, 32, 2), (2, 9, 5, 8, 1), (1, 5, 11, 128, 1), (2, 1, 3, 8, 1),
]


@gpu
@pytest.mark.parametrize('case', DW_CASES, ids=lambda c: '%dx%dx%d_C%d_s%d' % c)
def test_dwconv3x3_forward_and_gradients_vs_float64(ops, case):
    b, h, w, c, stride = case
    dw_fwd_check(ops, '%dx%dx%d C%d s%d' % case, b, h, w, c, stride, h * w + c + stride, 'dwconv_fwd_cases')
    g = torch.Generator().manual_seed(c + h * 3 + w)
    w9 = torch.randn(c, 9, generator=g) * 0.3
    dz = torch.randn(b, h // stride, w // stride, c, generator=g).half()
    z64, w64 = nchw(dz).double(), w9.double().view(c, 1, 3, 3)
    ref = np64(torch.nn.grad.conv2d_input((b, c, h, w), w64, z64, stride, 1, 1, c))
    S = np64(torch.nn.grad.conv2d_input((b, c, h, w), w64.abs(), z64.abs(), stride, 1, 1, c))
    db, da = out16((b, h, w, c))
    ops.call('yb_dwconv3x3_dgrad', dev(dz), dev(w9), da, b, h, w, c, stride)
    check16('dwconv dgrad %s' % hw_id(case), nchw(da), ref, sum_err(S, 9, 0), 'dwconv_dgrad')
    assert guard_kept(db, (b, h, w, c)), 'dwconv3x3_dgrad wrote past its output'
    if 256 % (c // 8) == 0:
        a = torch.randn(b, h, w, c, generator=g).half()
        check_dw_wgrad(ops, hw_id(case), dev(a), dev(dz), b, h, w, c, stride, 'dwconv_wgrad')


@gpu
def test_dwconv3x3_refusals_leave_the_output_untouched(ops):
    for (h, w, c, stride) in ((8, 8, 12, 1), (5, 8, 16, 2), (8, 7, 16, 2)):
        x = torch.randn(1, h, w, 2 * c, device=DEV).half()
        w9, one = torch.randn(c, 9, device=DEV), torch.ones(c, device=DEV)
        yb, y = out16((1, h, w, 2 * c))
        for name, extra in (('yb_dwconv3x3_bn_relu_fwd', (one, one)), ('yb_dwconv3x3_split_fwd', (one, one)), ('yb_dwconv3x3_raw_fwd', ())):
            with pytest.raises(RuntimeError):
                ops.call(name, x, w9, *extra, y, 1, h, w, c, stride)
        with pytest.raises(RuntimeError):
            ops.call('yb_dwconv3x3_dgrad', x, w9, y, 1, h, w, c, stride)
        assert untouched16(yb), (h, w, c, stride)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: depthwise weight gradient
# ------------------------------------------------------------------------------------------------------------------------------------
def check_dw_wgrad(ops, tag, a, dz, b, h, w, c, stride, group):
    dwb, dw = out32((c, 9))
    ops.call('yb_dwconv3x3_wgrad', a, dz, dw, b, h, w, c, stride)
    pixels = b * (h // stride) * (w // stride)
    L, lanes, grid = dw_wgrad_geometry(pixels, c, sms())
    ref, S = dw_wgrad_ref(a, dz, stride)
    check32('dwconv wgrad %s' % tag, dw, ref, sum_err(S, L + lanes + grid, pixels), group)
    assert bool(dwb[dw.numel():].isnan().all()), 'dwconv3x3_wgrad wrote past dw'
    return np.abs(np64(dw) - ref), ref


@gpu
@pytest.mark.parametrize('c', [8, 16, 32, 64, 128, 256, 512, 1024])
def test_dwconv3x3_wgrad_every_accepted_width(ops, c):
    g = torch.Generator().manual_seed(c)
    for (b, h, w, stride) in ((2, 12, 12, 1), (2, 12, 12, 2), (2, 10, 6, 1), (1, 6, 14, 2), (1, 2, 2, 2), (3, 1, 5, 1)):
        a = torch.randn(b, h, w, c, generator=g).half()
        dz = torch.randn(b, h // stride, w // stride, c, generator=g).half()
        check_dw_wgrad(ops, '%dx%dx%d C%d s%d' % (b, h, w, c, stride), dev(a), dev(dz), b, h, w, c, stride, 'dwconv_wgrad')
    # more pixels than the grid cap covers at 16 per thread
    lanes = 256 // (c // 8)
    pixels = lanes * 16 * 4 * sms() + lanes
    h = 2 * 16
    w = 2 * cdiv(pixels, 16)
    a = torch.randn(1, h, w, c, generator=g).half()
    dz = torch.randn(1, h // 2, w // 2, c, generator=g).half()
    check_dw_wgrad(ops, 'past the cap C%d' % c, dev(a), dev(dz), 1, h, w, c, 2, 'dwconv_wgrad_past_cap')


@gpu
def test_dwconv3x3_wgrad_refusals_leave_dw_untouched(ops):
    for c in (24, 2048, 12):
        a = torch.randn(1, 4, 6, c, device=DEV).half()
        dw = torch.full((c * 9,), 7.0, device=DEV)
        with pytest.raises(RuntimeError):
            ops.call('yb_dwconv3x3_wgrad', a, a, dw, 1, 4, 6, c, 1)
        torch.cuda.synchronize()
        assert bool((dw == 7.0).all()), c
    a = torch.randn(1, 5, 6, 16, device=DEV).half()
    dw = torch.full((16 * 9,), 7.0, device=DEV)
    with pytest.raises(RuntimeError):
        ops.call('yb_dwconv3x3_wgrad', a, a, dw, 1, 5, 6, 16, 2)
    torch.cuda.synchronize()
    assert bool((dw == 7.0).all())


# (C, side, stride) of MobileNet's depthwise layers at 416^2
MOBILENET_DW_416 = [(32, 208, 1), (64, 208, 2), (128, 104, 1), (128, 104, 2), (256, 52, 1), (256, 52, 2), (512, 26, 1), (512, 26, 2), (1024, 13, 1)]


@gpu
def test_dwconv3x3_wgrad_at_training_size(ops):
    """The nine depthwise layers of the MobileNet training step at 32 x 416^2, on ReLU-like activations and a small dz."""
    b = 32
    gen = torch.Generator(device=DEV).manual_seed(13)
    for c, side, stride in MOBILENET_DW_416:
        a = torch.relu(torch.randn(b, side, side, c, generator=gen, device=DEV)).half()
        dz = (torch.randn(b, side // stride, side // stride, c, generator=gen, device=DEV) * 0.05).half()
        err, ref = check_dw_wgrad(ops, '32x%d^2 C%d s%d' % (side, c, stride), a, dz, b, side, side, c, stride, 'dwconv_wgrad_416')
        rel = err / np.maximum(np.abs(ref), 1e-30)
        rec('dwconv_wgrad_416', err_over_dw=float(rel.max()), err_over_dw_median=float(np.median(rel)))
        L, lanes, grid = dw_wgrad_geometry(b * (side // stride) ** 2, c, sms())
        rec('dwconv_wgrad_416', **{'chain_C%d_s%d' % (c, stride): L, 'grid_C%d_s%d' % (c, stride): grid})
        del a, dz
