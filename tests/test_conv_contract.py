"""Contract of the implicit-GEMM conv family, element by element against float64 on the exact fp16 operands each kernel reads:
conv_igemm_kernel (64 x 1, 128 x 1 and 64 x 2 tiles), conv_wide_kernel (128 x 2), conv_c32_kernel (Cin = 32 halo tiles), the split
operands of strict mode, the data gradient (conv_igemm_kernel on yb_pack_weight_dgrad_f16 weights) and conv_wgrad_kernel.

The bound.  For one output element let S = sum |x * w| over the same fp16 operands (a float64 conv of |x| and |w|, zero padding), K
the reduction length (k * k * Cin; for the split forms the concatenated width; for the weight gradient the pixels summed by one split)
and P the number of partial sums combined (stream-K contributors per tile, or weight-gradient splits).  Then

    E_acc = (2 * ceil(K / 16) + P + 2) * 2^-23 * S
    E     = |scale| * E_acc + 2 * 2^-23 * (|scale| * (|acc| + E_acc) + |shift|)  [+ 2^-23 * slope * (|scale * acc + shift| + E) for the slope product]

Model: an fp16 x fp16 product is exact in fp32; one wgmma k16 step adds its 16 products into the fp32 accumulator with an error of at
most 2 fp32 ulps of S (DESIGN 2 measured the weight gradient's biased accumulation at about 1 ulp per step, 4e-9 per pixel); each
partial sum combined costs one more rounding; the epilogue's fma(acc, scale, shift) and the leaky slope product cost one rounding each,
and leaky with a slope in [0, 1] is 1-Lipschitz.  The constant comes from that arithmetic and is not fitted to any measurement.

Assertions (`check_f32`, `check_f16`):
  * fp32 outputs:  |got - ref| <= E;
  * fp16 outputs:  |got - ref| <= E + 1/2 ulp16(|ref| + E) * (1 + 2^-10), which covers the fp16 subnormal range (half an ulp = 2^-25);
  * where no fp16 rounding boundary lies within E of ref (RN16(ref - E) == RN16(ref + E)): got == RN16(ref) exactly; the number of
    such elements is recorded.
The worst err / bound and the worst error in fp16 ulps of each group are recorded (`record`, written to
$YB_PARITY_OUT/conv_measured.json when that is set).  max|d| / max|ref| is never used here: it cannot see an error on an element much
smaller than the largest one, which is what the unmarked tests demonstrate on the GPU tests' own shapes.

Exact relations asserted bit for bit besides the bound: the four tile shapes without stream-K (every accumulator sees the same K-blocks
and k16 steps in the same order; only the partition of M and N differs); the plain store against the TMA store and against RN16 of the
fp32 NCHW output (one epilogue expression); three stream-K launches; a channel slice of a wider output and an input read at x_ld > Cin
against the standalone launch; the halo-tile kernel against conv_igemm_kernel at BK = 32 (same tap order, two k16 steps per tap).
"""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

DEV = 'cuda'
gpu = pytest.mark.gpu
U = 2.0 ** -23              # fp32 spacing at 1
SENTINEL = 0x7C01           # an fp16 NaN payload no kernel writes: guard channels must keep it bit for bit
MEASURED = {}


def record(group, **figs):
    """Keep the worst figure per (group, quantity): maxima, except 'exact' which is summed; mirror to $YB_PARITY_OUT/conv_measured.json."""
    g = MEASURED.setdefault(group, {})
    for k, v in figs.items():
        g[k] = g.get(k, 0) + v if k in ('exact', 'elements') else max(float(v), g.get(k, 0.0))
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'conv_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


# ------------------------------------------------------------------------------------------------------------------------------------
# the reference and the bound
# ------------------------------------------------------------------------------------------------------------------------------------
def np64(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def rn16(a):
    """Round-to-nearest-even float64 -> fp16 (numpy converts directly, without an intermediate fp32 rounding)."""
    return np.asarray(a, dtype=np.float64).astype(np.float16)


def ulp16(a):
    a = np.abs(np.asarray(a, dtype=np.float64))
    with np.errstate(divide='ignore'):
        e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def acc_bound(S, K, P):
    return (2 * math.ceil(K / 16) + P + 2) * U * S


def epilogue(acc, S, K, P, scale, shift, slope):
    """(ref, E) of scale * acc + shift -> leaky(slope) over an NCHW accumulator, with the bound of the module docstring."""
    sc = np64(scale).reshape(1, -1, 1, 1)
    sh = np64(shift).reshape(1, -1, 1, 1)
    e_acc = acc_bound(S, K, P)
    lin = sc * acc + sh
    e_lin = np.abs(sc) * e_acc + 2 * U * (np.abs(sc) * (np.abs(acc) + e_acc) + np.abs(sh))
    ref = np.where(lin > 0, lin, lin * slope)
    return ref, e_lin + U * slope * (np.abs(lin) + e_lin)


def _fail(name, bad, got, ref, bound):
    i = np.unravel_index(np.argmax(bad), bad.shape)
    raise AssertionError('%s: %d of %d elements outside the bound, first at %s: got %r, reference %r, bound %.3e'
                         % (name, bad.sum(), bad.size, i, got[i], ref[i], bound[i]))


def check_f32(name, got, ref, E, group=None):
    got = np64(got)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = np.abs(got - ref)
    bad = ~(err <= E)
    if group:
        record(group, err_over_bound=(err / np.maximum(E, 1e-300)).max(), elements=err.size)
    if bad.any():
        _fail(name, bad, got, ref, E)


def check_f16(name, got, ref, E, group=None):
    """got: fp16 values (any tensor / array).  Bound, then bit equality with RN16(ref) where no rounding boundary is within E."""
    got = np64(got)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    bound = E + 0.5 * ulp16(np.abs(ref) + E) * (1 + 2.0 ** -10)
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    if bad.any():
        _fail(name, bad, got, ref, bound)
    sure = rn16(ref - E) == rn16(ref + E)
    exact = rn16(ref)
    wrong = sure & (got.astype(np.float16) != exact)
    if wrong.any():
        i = np.unravel_index(np.argmax(wrong), wrong.shape)
        raise AssertionError('%s: %d elements differ from RN16(ref) with no rounding boundary within E, first at %s: got %r, RN16 %r'
                             % (name, wrong.sum(), i, got[i], exact[i]))
    if group:
        record(group, err_over_bound=(err / bound).max(), err_ulp16=(err / ulp16(ref)).max(), exact=int(sure.sum()), elements=err.size)
    return int(sure.sum())


def rel_err(got, ref):
    got, ref = np64(got), np64(ref)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def conv64(x, w, k):
    """float64 conv (stride 1, pad (k-1)/2) of NCHW x and OIHW w, and the same conv of |x| and |w|."""
    x, w = x.double(), w.double()
    return F.conv2d(x, w, padding=k // 2), F.conv2d(x.abs(), w.abs(), padding=k // 2)


def ref_device():
    return DEV if torch.cuda.is_available() else 'cpu'


# ------------------------------------------------------------------------------------------------------------------------------------
# forward inputs (shared by the CPU and the GPU tests)
# ------------------------------------------------------------------------------------------------------------------------------------
FWD_SHAPES = [
    # b, h, w, cin, cout, k
    (3, 11, 13, 96, 136, 3),        # BK = 32, ragged M and N
    (2, 13, 13, 512, 1024, 3),
    (5, 13, 13, 1024, 200, 1),      # tiled A, ragged N
    (1, 7, 9, 64, 64, 3),           # M below one tile
    (4, 1, 37, 128, 72, 3),         # one pixel high: the halo above and below in the same K-block
    (4, 37, 1, 128, 72, 3),
    (4, 2, 2, 128, 72, 3),
    (2, 9, 11, 64, 8, 1),           # Cout 8 and 24
    (2, 9, 11, 64, 8, 3),
    (2, 9, 11, 64, 24, 1),
    (2, 9, 11, 64, 24, 3),
    (3, 8, 16, 64, 128, 3),         # M = 384: a multiple of 128, not of 256
    (2, 13, 13, 1280, 1024, 3),
]
SLOPES = (0.1, 0.0, 1.0)            # leaky, ResNet's ReLU, raw / head


def shape_id(s):
    return '%dx%dx%d_%d-%d_k%d' % s


def fwd_inputs(shape, seed=None):
    """x fp16 NCHW, w fp32 OIHW (the kernels pack it), scale with negative channels and one 1e-5 channel (outputs in the fp16
    subnormal range), random shift (0 on the 1e-5 channel), and the case's slope."""
    b, h, w, cin, cout, k = shape
    seed = seed if seed is not None else b * 1000003 + h * 1009 + w * 101 + cin * 7 + cout + k
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=g).half()
    wt = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5
    scale[1::3] *= -1
    shift = torch.randn(cout, generator=g) * 0.1
    scale[cout // 2] = 1e-5
    shift[cout // 2] = 0.0
    slope = SLOPES[FWD_SHAPES.index(shape) % 3] if shape in FWD_SHAPES else 0.1
    return x, wt, scale, shift, slope


_REF = {}


def fwd_reference(shape, x, wt):
    """(acc, S) float64 NCHW on the exact fp16 operands, cached per shape within the module."""
    key = (shape, x.shape)
    if key not in _REF:
        dev = ref_device()
        acc, S = conv64(x.to(dev), wt.half().to(dev), shape[5])
        _REF[key] = (np64(acc), np64(S))
    return _REF[key]


# ------------------------------------------------------------------------------------------------------------------------------------
# CPU: the bound accepts a correct stand-in and rejects deliberately wrong ones
# ------------------------------------------------------------------------------------------------------------------------------------
def standin(x, w16, scale, shift, slope, k, variant=None):
    """A correct kernel's stand-in: torch's fp32 conv of the same fp16 operands, fp32 epilogue, RN16 -- or one deliberately wrong variant."""
    xf, wf = x.float(), w16.float()
    if variant == 'halo_from_neighbour_row' and k == 3:
        # the left / right halo column read from the previous / next pixel in memory order (the neighbouring image row, or the
        # neighbouring image), not zeros
        b, c, h, w = xf.shape
        pad = torch.zeros(b * h * w + 2, c)
        pad[1:-1] = xf.permute(0, 2, 3, 1).reshape(b * h * w, c)
        rows = torch.arange(b * h)
        xp = torch.zeros(b, c, h + 2, w + 2)
        xp[:, :, 1:-1, 1:-1] = xf
        xp[:, :, 1:-1, 0] = pad[rows * w].view(b, h, c).permute(0, 2, 1)             # pixel (r, -1) = flat pixel r * w - 1
        xp[:, :, 1:-1, w + 1] = pad[rows * w + w + 1].view(b, h, c).permute(0, 2, 1)  # pixel (r, w) = flat pixel r * w + w
        acc = F.conv2d(xp, wf)
    else:
        acc = F.conv2d(xf, wf, padding=k // 2)
    if variant == 'channel_dropped':
        # one input channel of one tap left out (the one with the largest weights, so the error is visible at any K)
        tap = (k * k) // 2
        r, s = divmod(tap, k)
        c = int(wf[:, :, r, s].abs().sum(0).argmax())
        wd = torch.zeros_like(wf)
        wd[:, c, r, s] = wf[:, c, r, s]
        acc = acc - F.conv2d(xf, wd, padding=k // 2)
    sc, sh = scale.clone(), shift.clone()
    cout = sc.numel()
    if variant == 'ragged_tile_neighbour_scale':
        n0 = (cout - 1) // 64 * 64                                     # the last (ragged) 64-channel column tile
        sc[n0:], sh[n0:] = torch.roll(scale[n0:], 1), torch.roll(shift[n0:], 1)
    lin = acc * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)
    neg_slope = slope * 1.01 if variant == 'slope_off_by_1pct' else slope
    v = torch.where(lin > 0, lin, lin * neg_slope)
    if variant == 'last_m_tile_rows_duplicated':
        b, c, h, w = v.shape
        rows = v.permute(0, 2, 3, 1).reshape(b * h * w, c).clone()
        m0 = (rows.shape[0] - 1) // 128 * 128                          # the last (partial) 128-pixel M-tile
        lo = max(m0, 1)
        rows[lo:] = rows[lo - 1:-1].clone()                            # every row of it repeats its predecessor
        v = rows.reshape(b, h, w, c).permute(0, 3, 1, 2)
    y = v.half()
    if variant == 'round_toward_zero':
        y64 = y.double()
        over = y64.abs() > v.double().abs()
        y = torch.where(over, torch.from_numpy(np.nextafter(y.numpy(), np.float16(0))), y)
    return y


VARIANTS = ('round_toward_zero', 'slope_off_by_1pct', 'channel_dropped', 'halo_from_neighbour_row', 'ragged_tile_neighbour_scale',
            'last_m_tile_rows_duplicated')
BELOW_THE_BOUND = ('round_toward_zero', 'slope_off_by_1pct')     # errors of about one fp16 rounding
C32_SHAPES = [(2, 16, 8), (3, 21, 19), (1, 1, 37), (2, 37, 1), (1, 2, 2)]
C32_COUTS = [8, 16, 32, 48, 64]
CPU_SHAPES = FWD_SHAPES + [(b, h, w, 32, 48, 3) for b, h, w in C32_SHAPES]


@pytest.mark.parametrize('shape', CPU_SHAPES, ids=shape_id)
def test_bound_accepts_correct_standin(shape):
    x, wt, scale, shift, slope = fwd_inputs(shape)
    acc, S = fwd_reference(shape, x, wt)
    ref, E = epilogue(acc, S, shape[5] ** 2 * shape[3], 1, scale, shift, slope)
    check_f16('stand-in', standin(x, wt.half(), scale, shift, slope, shape[5]), ref, E)


REL_ERR_ACCEPTS = {}


@pytest.mark.parametrize('shape', CPU_SHAPES, ids=shape_id)
def test_bound_rejects_wrong_variants(shape):
    """Each deliberately wrong variant fails check_f16 on this shape (slope 0.1 so that the slope variant is a real error); which of them
    max|d| / max|ref| <= 1e-3 accepts is printed and kept in REL_ERR_ACCEPTS."""
    b, h, w, cin, cout, k = shape
    x, wt, scale, shift, _ = fwd_inputs(shape)
    slope = 0.1
    acc, S = fwd_reference(shape, x, wt)
    ref, E = epilogue(acc, S, k * k * cin, 1, scale, shift, slope)
    accepted = []
    for variant in VARIANTS:
        if variant == 'halo_from_neighbour_row' and (k == 1 or w == 1 or b * h == 1):
            continue                     # no halo column, or its memory neighbours are the pixels above / below, or outside the tensor
        y = standin(x, wt.half(), scale, shift, slope, k, variant)
        if variant in BELOW_THE_BOUND and k * k * cin > 8192:
            # 2 ulps per k16 step over K > 8192 allow more than half an fp16 ulp of an O(1) output: an error of one fp16 rounding
            # is inside the bound by construction.  Asserted, so that this exception stays exact.
            check_f16(variant, y, ref, E)
            continue
        with pytest.raises(AssertionError, match='^' + variant):
            check_f16(variant, y, ref, E)
        if rel_err(y, ref) <= 1e-3:
            accepted.append(variant)
    REL_ERR_ACCEPTS[shape] = accepted
    print('%s: rel_err <= 1e-3 accepts %s' % (shape_id(shape), ', '.join(accepted) or 'none'))


def test_rel_err_misses_what_the_bound_sees():
    """The gap this file closes: on the GPU tests' shapes max|d| / max|ref| <= 1e-3 accepts wrong fp16 rounding, a 1 % slope error and
    a wrong scale on the ragged column tile, all of which the element-wise bound rejects (test_bound_rejects_wrong_variants)."""
    for shape in [(2, 13, 13, 512, 1024, 3), (3, 11, 13, 96, 136, 3), (5, 13, 13, 1024, 200, 1)]:
        x, wt, scale, shift, _ = fwd_inputs(shape)
        acc, S = fwd_reference(shape, x, wt)
        ref, _ = epilogue(acc, S, 1, 1, scale, shift, 0.1)
        y = standin(x, wt.half(), scale, shift, 0.1, shape[5], 'round_toward_zero')
        assert rel_err(y, ref) <= 1e-3, shape
    shape = (2, 13, 13, 512, 1024, 3)
    x, wt, scale, shift, _ = fwd_inputs(shape)
    acc, S = fwd_reference(shape, x, wt)
    ref, _ = epilogue(acc, S, 1, 1, scale, shift, 0.1)
    assert rel_err(standin(x, wt.half(), scale, shift, 0.1, 3, 'slope_off_by_1pct'), ref) <= 1e-3


def test_fp16_rule_in_the_subnormal_range():
    """Half an ulp below 2^-14 is 2^-25: an output one subnormal step off is rejected when E is small, RN16 accepted."""
    ref = np.array([3.0e-6, 1.0e-7, -4.2e-5, 0.0])
    E = np.full_like(ref, 1e-12)
    check_f16('sub', rn16(ref), ref, E)
    with pytest.raises(AssertionError):
        check_f16('sub', rn16(ref) + np.float16(2.0 ** -24), ref, E)


def test_pool_bound_on_standin():
    """Fused 2x2 max-pool: ref = max of the window's references, bound = the window's largest bound (max is 1-Lipschitz)."""
    shape = (2, 16, 8, 32, 48, 3)
    x, wt, scale, shift, slope = fwd_inputs(shape)
    acc, S = fwd_reference(shape, x, wt)
    ref, E = epilogue(acc, S, 9 * 32, 1, scale, shift, slope)
    y = F.max_pool2d(standin(x, wt.half(), scale, shift, slope, 3).float(), 2)
    check_f16('pool', y, pool_np(ref), pool_np(E))


def pool_np(a):
    b, c, h, w = a.shape
    return a.reshape(b, c, h // 2, 2, w // 2, 2).max(axis=(3, 5))


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


@pytest.fixture(scope='module')
def ws(ops):
    return ops.conv_workspace(DEV)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def nchw(y):
    return y.permute(0, 3, 1, 2)


def bits(t):
    return t.contiguous().view(torch.int16)


def sentinel(shape):
    return torch.full(shape, SENTINEL, dtype=torch.int16, device=DEV).view(torch.float16)


def sk_partials(m_total, rows, cout, bn, num_kb):
    """Upper bound of the stream-K contributors of one tile: the iteration space tiles x K-blocks is cut into #SMs ranges of at least
    floor(units / #SMs) K-blocks (WorkIter), so a tile meets at most ceil(num_kb / base) + 1 of them."""
    tiles = -(-m_total // rows) * -(-cout // bn)
    base = max(tiles * num_kb // sms(), 1)
    return -(-num_kb // base) + 1


FORMS = [('64x1', 64, 1), ('128x1', 128, 1), ('64x2', 64, 2), ('128x2', 128, 2)]


def form_flags(ops, bn, mt, sk):
    return ops.conv_force_bn(bn) | ops.conv_force_mt(mt) | (ops.CONV_FORCE_STREAMK if sk else ops.CONV_NO_STREAMK)


def expect_choice(ops, shape, flags, kernel, bk, bn, rows, sk, out_mode=0):
    b, h, w, cin, cout, k = shape
    ch = ops.conv_choice(b, h, w, cin, cout, k, out_mode=out_mode, flags=flags, workspace=sk)
    want = dict(kernel=kernel, bk=bk, bn=bn, rows=rows, streamk=sk)
    assert {q: ch[q] for q in want} == want, 'flags %#x reached %s, not %s' % (flags, ch, want)
    return ch


def to_dev(x, wt, scale, shift, ops):
    x16 = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    w16 = ops.pack_weight_f16(wt.to(DEV))
    assert torch.equal(bits(w16), bits(wt.half().permute(0, 2, 3, 1).to(DEV))), 'pack_weight_f16 differs from w.half()'
    return x16, w16, scale.to(DEV), shift.to(DEV)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: forward, conv_igemm_kernel and conv_wide_kernel
# ------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('shape', FWD_SHAPES, ids=shape_id)
def test_forward_tiles_vs_float64(ops, ws, shape):
    b, h, w, cin, cout, k = shape
    x, wt, scale, shift, slope = fwd_inputs(shape)
    acc, S = fwd_reference(shape, x, wt)
    x16, w16, sc, sh = to_dev(x, wt, scale, shift, ops)
    m_total, K = b * h * w, k * k * cin
    bk = 64 if cin % 64 == 0 else 32
    num_kb = k * k * (cin // bk)
    taken = []
    for name, bn, mt in FORMS:
        wide = bn * mt > 128
        kern = 'conv_wide_kernel' if wide else 'conv_igemm_kernel'
        for sk in (False, True):
            flags = form_flags(ops, bn, mt, sk)
            ch = ops.conv_choice(b, h, w, cin, cout, k, flags=flags, workspace=sk)
            if sk and not ch['streamk']:
                continue                 # conv_choice does not take stream-K here (fewer than 4 K-blocks per CTA or one K-block)
            expect_choice(ops, shape, flags, kern, bk, bn, 128 * mt, sk)
            taken.append(name + ('+sk' if sk else ''))
            P = sk_partials(m_total, 128 * mt, cout, bn, num_kb) if sk else 1
            ref, E = epilogue(acc, S, K, P, scale, shift, slope)
            group = 'fwd_%s%s' % (name, '_sk' if sk else '')
            kw = dict(flags=flags, workspace=ws if sk else None)
            y = ops.conv_bn_act(x16, w16, sc, sh, slope, **kw)
            check_f16('%s tma' % group, nchw(y), ref, E, group)
            if sk:
                for _ in range(2):
                    assert torch.equal(bits(ops.conv_bn_act(x16, w16, sc, sh, slope, **kw)), bits(y)), 'stream-K launches differ'
                torch.cuda.synchronize()
                assert int(ws[:4096].view(torch.int32).abs().sum()) == 0, 'stream-K flags not reset'
            # output slice: channels [8, 8 + Cout) of a wider buffer; every guard channel keeps the sentinel
            buf = sentinel((b, h, w, cout + 24))
            ops.conv_bn_act(x16, w16, sc, sh, slope, out=buf, y_ch_off=8, **kw)
            assert torch.equal(bits(buf[..., 8:8 + cout]), bits(y)), '%s: slice output differs' % group
            assert bool((bits(buf[..., :8]) == SENTINEL).all()) and bool((bits(buf[..., 8 + cout:]) == SENTINEL).all()), \
                '%s: wrote outside its channel slice' % group
            # input slice: the first Cin channels of an x_ld = Cin + 24 buffer whose other channels are NaN
            xw = torch.full((b, h, w, cin + 24), float('nan'), dtype=torch.float16, device=DEV)
            xw[..., :cin] = x16
            assert torch.equal(bits(ops.conv_bn_act(xw, w16, sc, sh, slope, cin=cin, **kw)), bits(y)), '%s: x_ld > Cin differs' % group
            if wide:
                continue                 # the wide tile has neither the plain store nor the fp32 NCHW output
            expect_choice(ops, shape, flags | ops.CONV_PLAIN_STORE, kern, bk, bn, 128 * mt, sk)
            yp = ops.conv_bn_act(x16, w16, sc, sh, slope, flags=flags | ops.CONV_PLAIN_STORE, workspace=ws if sk else None)
            check_f16('%s plain' % group, nchw(yp), ref, E, group + '_plain')
            expect_choice(ops, shape, flags, kern, bk, bn, 128 * mt, sk, out_mode=ops.OUT_F32_NCHW)
            y32 = ops.conv_bn_act(x16, w16, sc, sh, slope, out_mode=ops.OUT_F32_NCHW, **kw)
            check_f32('%s fp32' % group, y32, ref, E, group + '_f32')
            assert torch.equal(bits(nchw(yp)), bits(y32.half())), '%s: plain store != RN16(fp32 output)' % group
            assert torch.equal(bits(yp), bits(y)), '%s: TMA store != plain store' % group
            if sk:
                torch.cuda.synchronize()
                assert int(ws[:4096].view(torch.int32).abs().sum()) == 0, 'stream-K flags not reset'
    # every tile shape without stream-K, at the same BK: the same K-order per accumulator, so the same bits
    ref_y = ops.conv_bn_act(x16, w16, sc, sh, slope, flags=form_flags(ops, 128, 1, False))
    for name, bn, mt in FORMS:
        y = ops.conv_bn_act(x16, w16, sc, sh, slope, flags=form_flags(ops, bn, mt, False))
        assert torch.equal(bits(y), bits(ref_y)), '%s differs from 128x1 without stream-K' % name
    record('forms_reached', **{f: 1 for f in taken})


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: forward, conv_c32_kernel and its alternatives
# ------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('cout', C32_COUTS)
@pytest.mark.parametrize('bhw', C32_SHAPES, ids=lambda s: '%dx%dx%d' % s)
def test_forward_c32_vs_float64(ops, bhw, cout):
    b, h, w = bhw
    shape = (b, h, w, 32, cout, 3)
    x, wt, scale, shift, slope = fwd_inputs(shape)
    acc, S = fwd_reference(shape, x, wt)
    x16, w16, sc, sh = to_dev(x, wt, scale, shift, ops)
    ref, E = epilogue(acc, S, 9 * 32, 1, scale, shift, slope)
    expect_choice(ops, shape, 0, 'conv_c32_kernel', 32, 64, 128, False)
    y = ops.conv_bn_act(x16, w16, sc, sh, slope)
    check_f16('c32 halo', nchw(y), ref, E, 'c32_halo')
    for tag, fl in (('im2col', ops.CONV_C32_IM2COL), ('plain', ops.CONV_C32_IM2COL | ops.CONV_PLAIN_STORE), ('generic', ops.CONV_NO_SMALLK)):
        ch = ops.conv_choice(b, h, w, 32, cout, 3, flags=fl, workspace=False)
        assert ch['kernel'] == 'conv_igemm_kernel' and ch['bk'] == 32, (tag, ch)
        y2 = ops.conv_bn_act(x16, w16, sc, sh, slope, flags=fl)
        check_f16('c32 ' + tag, nchw(y2), ref, E, 'c32_' + tag)
        # same taps in the same order, two k16 steps per tap: the halo tile equals conv_igemm_kernel at BK = 32
        assert torch.equal(bits(y2), bits(y)), 'c32 %s differs from the halo-tile kernel' % tag
    if h % 2 == 0 and w % 2 == 0:
        assert ops.conv_choice(b, h, w, 32, cout, 3, flags=ops.CONV_POOL2X2, workspace=False)['kernel'] == 'conv_c32_kernel'
        yp = ops.conv_bn_act(x16, w16, sc, sh, slope, flags=ops.CONV_POOL2X2)
        check_f16('c32 pool', nchw(yp), pool_np(ref), pool_np(E), 'c32_pool')
        assert torch.equal(bits(yp), bits(ops.maxpool2x2(y)))
    buf = sentinel((b, h, w, cout + 24))
    ops.conv_bn_act(x16, w16, sc, sh, slope, out=buf, y_ch_off=8)
    assert torch.equal(bits(buf[..., 8:8 + cout]), bits(y))
    assert bool((bits(buf[..., :8]) == SENTINEL).all()) and bool((bits(buf[..., 8 + cout:]) == SENTINEL).all())
    xw = torch.full((b, h, w, 40), float('nan'), dtype=torch.float16, device=DEV)
    xw[..., :32] = x16
    assert torch.equal(bits(ops.conv_bn_act(xw, w16, sc, sh, slope, cin=32)), bits(y)), 'x_ld > 32 differs'


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: split operands (strict mode)
# ------------------------------------------------------------------------------------------------------------------------------------
SPLIT_CASES = [     # the shapes of test_gpu_parity.test_conv_split_precision_vs_oracle
    # b, h, w, cin, cout, k, split_a, split_w, src_lo
    (2, 16, 16, 64, 128, 3, True, True, True),
    (3, 13, 13, 128, 256, 3, True, False, True),
    (3, 13, 13, 128, 256, 3, False, True, False),
    (2, 26, 26, 256, 128, 1, True, True, True),
    (2, 26, 26, 256, 128, 1, False, True, True),
    (32, 13, 13, 512, 1024, 3, True, True, True),
    (3, 21, 19, 32, 64, 3, False, True, False),
    (5, 19, 17, 96, 136, 3, True, True, True),
]


def split_operands(b, h, w, cin, cout, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5
    scale[1::3] *= -1
    shift = torch.randn(cout, generator=g) * 0.1
    return x, wt, scale, shift


def split_reference(x, wt, k, split_a, split_w):
    """fp64 sum of the segments the kernel multiplies: a_hi w_hi, a_lo w_hi (activation split), a_hi w_lo (weight split)."""
    dev = ref_device()
    a_hi = x.half()
    a_lo = (x - a_hi.float()).half()
    w_hi = wt.half()
    w_lo = (wt - w_hi.float()).half()
    pairs = [(a_hi, w_hi)] + ([(a_lo, w_hi)] if split_a else []) + ([(a_hi, w_lo)] if split_w else [])
    acc = S = 0
    for a, ww in pairs:
        c, s = conv64(a.to(dev), ww.to(dev), k)
        acc, S = acc + c, S + s
    return np64(acc), np64(S), len(pairs), a_hi, a_lo


@gpu
@pytest.mark.parametrize('case', SPLIT_CASES, ids=lambda c: '%dx%dx%d_%d-%d_k%d_%d%d%d' % c)
def test_split_operands_vs_float64(ops, case):
    b, h, w, cin, cout, k, split_a, split_w, src_lo = case
    x, wt, scale, shift = split_operands(b, h, w, cin, cout, k, cin * 5 + cout + k)
    acc, S, segs, a_hi, a_lo = split_reference(x, wt, k, split_a, split_w)
    ref, E = epilogue(acc, S, segs * k * k * cin, 1, scale, shift, 0.1)
    hi = a_hi.permute(0, 2, 3, 1)
    src = (torch.cat([hi, a_lo.permute(0, 2, 3, 1)], -1) if src_lo else hi).contiguous().to(DEV)
    w16 = ops.pack_weight_split_f16(wt.to(DEV), split_a, split_w)
    assert w16.shape[-1] == segs * cin
    sc, sh = scale.to(DEV), shift.to(DEV)
    a_ch = cin * (2 if split_a else 1)
    flags = form_flags(ops, 128, 1, False)
    out = sentinel((b, h, w, 2 * cout + 8))
    ops.conv_bn_act_split(src, w16, sc, sh, 0.1, out, a_channels=a_ch, y_ch_off=0, lo_ch_off=cout, flags=flags)
    y32 = torch.empty(b, cout, h, w, dtype=torch.float32, device=DEV)
    ops.conv_bn_act_split(src, w16, sc, sh, 0.1, y32, a_channels=a_ch, out_mode=ops.OUT_F32_NCHW, flags=flags)
    assert bool((bits(out[..., 2 * cout:]) == SENTINEL).all()), 'wrote outside its channel slices'
    check_f32('split fp32', y32, ref, E, 'split_f32')
    got_hi, got_lo = nchw(out[..., :cout]), nchw(out[..., cout:2 * cout])
    check_f16('split hi', got_hi, ref, E, 'split_hi')
    # hi = RN16(f), lo = RN16(f - hi) of the fp32 value f the same tile computes (the fp32 output above, checked within E)
    assert torch.equal(bits(got_hi), bits(y32.half())), 'hi != RN16(f)'
    assert torch.equal(bits(got_lo), bits((y32 - got_hi.float()).half())), 'lo != RN16(f - hi)'
    f = np64(y32)
    hl = np64(got_hi) + np64(got_lo)
    check_f32('split hi + lo', hl, ref, E + 0.5 * ulp16(np.abs(f - np64(got_hi))) * (1 + 2.0 ** -10), 'split_hi_plus_lo')


@gpu
@pytest.mark.parametrize('sk', [False, True])
def test_split_operands_wide_tile(ops, ws, sk):
    b, h, w, cin, cout, k = 3, 13, 13, 256, 512, 3
    x, wt, scale, shift = split_operands(b, h, w, cin, cout, k, 23)
    acc, S, segs, a_hi, a_lo = split_reference(x, wt, k, True, True)
    src = torch.cat([a_hi, a_lo], 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    w16 = ops.pack_weight_split_f16(wt.to(DEV), True, True)
    flags = form_flags(ops, 128, 2, sk)
    ch = ops.conv_choice(b, h, w, 3 * cin, cout, k, flags=flags, workspace=sk)
    assert ch['kernel'] == 'conv_wide_kernel' and ch['streamk'] == sk and ch['bn'] == 128 and ch['rows'] == 256, ch
    num_kb = k * k * 3 * cin // 64
    P = sk_partials(b * h * w, 256, cout, 128, num_kb) if sk else 1
    ref, E = epilogue(acc, S, 3 * k * k * cin, P, scale, shift, 0.1)
    out = torch.empty(b, h, w, cout, dtype=torch.float16, device=DEV)
    ops.conv_bn_act_split(src, w16, scale.to(DEV), shift.to(DEV), 0.1, out, a_channels=2 * cin, flags=flags, workspace=ws if sk else None)
    check_f16('split wide', nchw(out), ref, E, 'split_wide' + ('_sk' if sk else ''))
    if not sk:
        out128 = torch.empty_like(out)
        ops.conv_bn_act_split(src, w16, scale.to(DEV), shift.to(DEV), 0.1, out128, a_channels=2 * cin, flags=form_flags(ops, 128, 1, False))
        assert torch.equal(bits(out), bits(out128))


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: weight packing and the data gradient
# ------------------------------------------------------------------------------------------------------------------------------------
def special_weights(cout, cin, k, seed):
    """Random weights plus fp16 edge values: subnormals, -0, a tie between two fp16 neighbours, values just under 65504."""
    w = torch.randn(cout, cin, k, k, generator=torch.Generator().manual_seed(seed)) * 0.05
    flat = w.view(-1)
    flat[:6] = torch.tensor([3e-7, -5.9e-8, -0.0, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 65000.0])
    return w


@gpu
@pytest.mark.parametrize('cout,cin,k,cout_pad', [(125, 1024, 1, 128), (64, 32, 3, 64), (1024, 512, 3, 1024), (72, 64, 3, 96), (8, 32, 1, 24)])
def test_weight_packs_bit_exact(ops, cout, cin, k, cout_pad):
    w = special_weights(cout, cin, k, cout + cin + k)
    wd = w.to(DEV)
    w_hi = w.half()
    rot = w_hi.flip(2, 3).permute(1, 2, 3, 0)                          # [Cin][k][k][Cout], rotated 180 degrees
    out = sentinel((cin, k, k, cout_pad))
    ops.call('yb_pack_weight_dgrad_f16', wd, out, cout, cin, k, cout_pad)
    want = torch.zeros(cin, k, k, cout_pad, dtype=torch.float16)
    want[..., :cout] = rot
    assert torch.equal(bits(out.cpu()), bits(want)), 'yb_pack_weight_dgrad_f16'
    assert torch.equal(bits(ops.pack_weight_f16(wd, 0).cpu()), bits(w_hi.permute(0, 2, 3, 1))), 'pack_weight_f16 mode 0'
    assert torch.equal(bits(ops.pack_weight_f16(wd, 1).cpu()), bits(rot)), 'pack_weight_f16 mode 1'
    w_lo = (w - w_hi.float()).half()
    segs = {(True, False): (w_hi, w_hi), (False, True): (w_hi, w_lo), (True, True): (w_hi, w_hi, w_lo)}
    for (sa, sw), parts in segs.items():
        want = torch.cat([p.permute(0, 2, 3, 1) for p in parts], -1)
        assert torch.equal(bits(ops.pack_weight_split_f16(wd, sa, sw).cpu()), bits(want)), 'pack_weight_split_f16 %s' % ((sa, sw),)


DGRAD_CASES = [
    # b, h, w, cout, cout_pad, cin, k: the data gradient of a conv cin -> cout runs conv_igemm_kernel cout_pad -> cin on dz
    (2, 13, 13, 125, 128, 1024, 1),     # the head
    (2, 16, 12, 64, 64, 32, 3),
    (2, 13, 13, 1024, 1024, 512, 3),
    (3, 11, 9, 72, 96, 64, 3),
]


@gpu
@pytest.mark.parametrize('case', DGRAD_CASES, ids=lambda c: '%dx%dx%d_%d(%d)-%d_k%d' % c)
def test_data_gradient_vs_float64(ops, case):
    b, h, w, cout, cout_pad, cin, k = case
    g = torch.Generator().manual_seed(cout + cin + k)
    wt = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    dz = (torch.randn(b, cout, h, w, generator=g) * 0.1).half()
    wd = torch.empty(cin, k, k, cout_pad, dtype=torch.float16, device=DEV)
    ops.call('yb_pack_weight_dgrad_f16', wt.to(DEV), wd, cout, cin, k, cout_pad)
    dz16 = torch.zeros(b, h, w, cout_pad, dtype=torch.float16, device=DEV)
    dz16[..., :cout] = dz.permute(0, 2, 3, 1).to(DEV)
    ch = ops.conv_choice(b, h, w, cout_pad, cin, k, workspace=False)
    assert ch['kernel'] in ('conv_igemm_kernel', 'conv_wide_kernel') and not ch['streamk'], ch
    one, zero = torch.ones(cin, device=DEV), torch.zeros(cin, device=DEV)
    dx = ops.conv_bn_act(dz16, wd, one, zero, 1.0)
    dev = ref_device()
    w64, dz64 = wt.half().double().to(dev), dz.double().to(dev)
    ref = np64(torch.nn.grad.conv2d_input((b, cin, h, w), w64, dz64, padding=k // 2))
    S = np64(torch.nn.grad.conv2d_input((b, cin, h, w), w64.abs(), dz64.abs(), padding=k // 2))
    refe, E = epilogue(ref, S, k * k * cout_pad, 1, one.cpu(), zero.cpu(), 1.0)
    check_f16('dgrad %s' % ch['kernel'], nchw(dx), refe, E, 'dgrad')
    # the padding channels of dz meet zero weights: large finite values there change no bit
    dz16[..., cout:] = 30000.0
    assert torch.equal(bits(ops.conv_bn_act(dz16, wd, one, zero, 1.0)), bits(dx)), 'dz padding channels leak into dx'
    record('dgrad_kernels', **{ch['kernel'] + '_bn%d_rows%d_bk%d' % (ch['bn'], ch['rows'], ch['bk']): 1})


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: weight gradient
# ------------------------------------------------------------------------------------------------------------------------------------
WGRAD_KP = 128      # pixels per K-block of conv_wgrad_kernel


def wgrad_geometry(m_total, cin, cout, k, env_splits=None, num_sms=None):
    """conv_wgrad_forward's launch geometry restated (accumulator columns N, splits, pixels per split) -- for the bound's K and P and
    to name the form each case reaches."""
    num_sms = num_sms or sms()
    nmax = 96 if cin == 32 else 256
    taps = k * k
    npg = min(256 if cin >= 256 else cin, nmax)
    chunks = -(-cin // npg)
    col_tiles = taps * chunks
    g = nmax // npg
    if taps == 9 and 3 < g < 9:
        g = 3
    g = min(g, col_tiles, 9)
    base_items = -(-cout // 128) * -(-col_tiles // g)
    kb_total = -(-m_total // WGRAD_KP)
    max_splits = (kb_total + 7) // 8
    splits, best = 1, 1e30
    for s in range(1, min(max_splits, 512) + 1):
        waves = -(-base_items * s // num_sms)
        cost = waves * (-(-kb_total // s) + (11.0 if s > 1 else 3.3))
        if cost < best * 0.999:
            best, splits = cost, s
    if env_splits is not None:
        splits = env_splits
    splits = max(1, min(splits, max_splits))
    kbps = -(-kb_total // splits)
    return dict(N=g * npg, splits=-(-kb_total // kbps), pixels=kbps * WGRAD_KP, ragged_chunk=cin % npg != 0, max_splits=max_splits)


WGRAD_CASES = [
    # b, h, w, cin, cout, k, x_ld, dz_ld
    (8, 26, 26, 32, 64, 1, 32, 64),         # N = 32; 43 K-blocks: up to 6 splits
    (8, 52, 52, 32, 64, 3, 32, 64),         # N = 96, 169 K-blocks: up to 22 splits
    (8, 26, 26, 64, 64, 1, 64, 64),         # N = 64
    (4, 26, 26, 128, 64, 1, 128, 64),       # N = 128
    (4, 26, 26, 64, 128, 3, 64, 128),       # N = 192
    (8, 26, 26, 256, 128, 1, 256, 128),     # N = 256
    (2, 13, 13, 128, 128, 3, 128, 128),     # N = 256 from two 128-channel groups
    (2, 13, 13, 320, 64, 1, 320, 64),       # ragged last input-channel chunk (256 + 64)
    (8, 26, 26, 320, 64, 3, 320, 64),
    (8, 26, 26, 384, 64, 1, 384, 64),       # 256 + 128
    (2, 13, 13, 384, 64, 3, 384, 64),
    (3, 11, 13, 64, 8, 3, 64, 8),           # Cout < 64
    (3, 11, 13, 64, 24, 1, 64, 24),
    (2, 13, 13, 1024, 125, 1, 1024, 128),   # the head: dz_ld 128
    (3, 11, 13, 128, 200, 3, 128, 200),
    (2, 7, 9, 64, 24, 3, 72, 40),           # x_ld > Cin, dz_ld > Cout (NaN in the unread channels)
    (3, 1, 1, 64, 64, 3, 64, 64),           # tiny images: one 128-pixel K-block spans many of them
    (5, 2, 2, 128, 64, 3, 136, 64),
    (4, 1, 37, 64, 64, 3, 64, 64),
    (1, 7, 9, 64, 64, 3, 64, 64),           # M < 128
]


@gpu
@pytest.mark.parametrize('case', WGRAD_CASES, ids=lambda c: '%dx%dx%d_%d-%d_k%d_ld%d,%d' % c)
def test_weight_gradient_vs_float64(ops, monkeypatch, case):
    b, h, w, cin, cout, k, x_ld, dz_ld = case
    g = torch.Generator().manual_seed(cin * 3 + cout + k + h)
    x = torch.randn(b, h, w, cin, generator=g).half()
    dz = (torch.randn(b, h, w, cout, generator=g) * 0.1).half()
    xb = torch.full((b, h, w, x_ld), float('nan'), dtype=torch.float16)
    xb[..., :cin] = x
    dzb = torch.full((b, h, w, dz_ld), float('nan'), dtype=torch.float16)
    dzb[..., :cout] = dz
    xb, dzb = xb.to(DEV), dzb.to(DEV)
    dev = ref_device()
    x64, dz64 = x.permute(0, 3, 1, 2).double().to(dev), dz.permute(0, 3, 1, 2).double().to(dev)
    ref = np64(torch.nn.grad.conv2d_weight(x64, (cout, cin, k, k), dz64, padding=k // 2))
    S = np64(torch.nn.grad.conv2d_weight(x64.abs(), (cout, cin, k, k), dz64.abs(), padding=k // 2))
    m_total = b * h * w
    model = wgrad_geometry(m_total, cin, cout, k)
    seen = set()
    for tag, env in (('1', 1), ('3', 3), ('model', None), ('max', 512)):
        if env is None:
            monkeypatch.delenv('YB_WGRAD_SPLITS', raising=False)
        else:
            monkeypatch.setenv('YB_WGRAD_SPLITS', str(env))
        geo = wgrad_geometry(m_total, cin, cout, k, env)
        if geo['splits'] in seen:
            continue
        seen.add(geo['splits'])
        dw = torch.full((cout, k, k, cin), float('nan'), dtype=torch.float32, device=DEV)   # an element never written stays NaN
        ops.call('yb_conv_wgrad', xb, dzb, dw, b, h, w, cin, cout, k, x_ld, dz_ld)
        E = acc_bound(S, geo['pixels'], geo['splits'])
        check_f32('wgrad N=%d splits=%d' % (geo['N'], geo['splits']), dw.permute(0, 3, 1, 2), ref, E,
                  'wgrad_N%d_%s' % (geo['N'], 'direct' if geo['splits'] == 1 else 'atomic'))
    monkeypatch.delenv('YB_WGRAD_SPLITS', raising=False)
    record('wgrad_forms', **{'N%d_splits%d' % (model['N'], s): 1 for s in seen})
    # the reference's OIHW layout times the unscale factor: one fp32 multiply per element
    out = torch.empty(cout, cin, k, k, dtype=torch.float32, device=DEV)
    ops.call('yb_unpack_wgrad', dw, out, cout, cin, k, 0.37)
    assert torch.equal(out, dw.permute(0, 3, 1, 2) * torch.tensor(0.37, dtype=torch.float32, device=DEV))


def test_wgrad_geometry_names_every_width():
    """The restated launch geometry reaches every accumulator width and the ragged chunk that WGRAD_CASES claims (a CPU check of the
    table itself; the GPU test runs them)."""
    geos = [wgrad_geometry(b * h * w, cin, cout, k, num_sms=132) for b, h, w, cin, cout, k, _, _ in WGRAD_CASES]   # an H100 SXM
    assert {g['N'] for g in geos} == {32, 64, 96, 128, 192, 256}
    assert {c[3] for c, g in zip(WGRAD_CASES, geos) if g['ragged_chunk']} == {320, 384}
    assert max(g['max_splits'] for g in geos) >= 8


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: host-side refusals, on buffers that really have the claimed size
# ------------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_refusals_leave_the_output_untouched(ops):
    b, h, w = 2, 6, 5
    one = lambda c: torch.ones(c, device=DEV)                                        # noqa: E731
    cases = {}
    # Cin % 32 != 0
    cases['cin48'] = (torch.zeros(b, h, w, 48, dtype=torch.float16, device=DEV), torch.zeros(64, 3, 3, 48, dtype=torch.float16, device=DEV), 64, {}, None)
    # Cout % 8 != 0 with fp16 output
    cases['cout12'] = (torch.zeros(b, h, w, 64, dtype=torch.float16, device=DEV), torch.zeros(12, 3, 3, 64, dtype=torch.float16, device=DEV), 12, {}, None)
    # x_ld % 8 != 0: the first 32 of 36 channels
    cases['xld36'] = (torch.zeros(b, h, w, 36, dtype=torch.float16, device=DEV), torch.zeros(64, 3, 3, 32, dtype=torch.float16, device=DEV), 64,
                      dict(cin=32), None)
    # x not 16 B aligned: a real buffer viewed one element in
    base = torch.zeros(b * h * w * 64 + 1, dtype=torch.float16, device=DEV)
    cases['misaligned'] = (base[1:].view(b, h, w, 64), torch.zeros(64, 3, 3, 64, dtype=torch.float16, device=DEV), 64, {}, None)
    # the fused max-pool outside the Cin = 32 kernel
    cases['pool_cin64'] = (torch.zeros(b, 6, 6, 64, dtype=torch.float16, device=DEV), torch.zeros(64, 3, 3, 64, dtype=torch.float16, device=DEV), 64,
                           dict(flags=ops.CONV_POOL2X2), (b, 3, 3, 64))
    for name, (x, wt, cout, kw, oshape) in cases.items():
        out = sentinel(oshape or (x.shape[0], x.shape[1], x.shape[2], cout))
        with pytest.raises((RuntimeError, ValueError)):
            ops.conv_bn_act(x, wt, one(cout), one(cout), 0.1, out=out, **kw)
        torch.cuda.synchronize()
        assert bool((bits(out) == SENTINEL).all()), '%s: refused launch wrote its output' % name
    # the weight gradient has no kernel for Cin = 96
    x = torch.zeros(b, h, w, 96, dtype=torch.float16, device=DEV)
    dz = torch.zeros(b, h, w, 64, dtype=torch.float16, device=DEV)
    dw = torch.full((64, 3, 3, 96), float('nan'), dtype=torch.float32, device=DEV)
    with pytest.raises(RuntimeError):
        ops.call('yb_conv_wgrad', x, dz, dw, b, h, w, 96, 64, 3, 96, 64)
    torch.cuda.synchronize()
    assert bool(dw.isnan().all())
