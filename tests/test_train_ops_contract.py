"""Contract of the first-layer conv (conv0_tc.cu) and of the BatchNorm, pool and reorg kernels of the Darknet-19 / Tiny training step
(train_ops.cu, pointwise.cu), element by element against float64 on the exact operands each kernel reads, at the shapes where they go wrong.
Same method and helpers as test_conv_contract.py: fp16 outputs are checked with `check_f16` (the bound, then RN16(ref) bit for bit where no
fp16 rounding boundary lies within it), fp32 outputs with `check_f32`; max|d| / max|ref| is never used.

Operands.  conv0 reads the image as fp16: RN16(x) of the fp32 NCHW image, RN16(RN32(RN32(u8) * RN32(1/255))) of a uint8 NHWC frame, and
RN16(w) of the fp32 weights.  The BatchNorm kernels read the stored fp16 z, da, dap, the fp32 mean, invstd, gamma, beta and the float64 sums
buffer; the references below restate each kernel's operation on exactly those values.  u = 2^-24 (fp32 unit roundoff), v = 2^-53.

Sums (bn_stats, conv0's fused statistics, bn_act_bwd mode 0).  With L the largest number of fp32 additions one term goes through and G the
float64 additions after that, recursive summation gives |S_kernel - S| <= 1.01 (L u + (G + 64) v) A, A = sum |term| (the 64 v also covers
the reference's own float64 reduction).  L and G are restated from the host code.  bn_stats runs rpi = 256 / (C/8) rows per iteration on
blocks = min(ceil(rows / (16 rpi)), 8 SMs); a thread adds each trip's four rows in fp32 and the trips in float64, then the block's threads and
the blocks add in float64: L = 4, G = ceil(rows / (4 blocks rpi)) + rpi + blocks.  conv0_k16_kernel<raw> sums 16 rows of a tile per thread
in fp32, reduces them over a 3-level shuffle tree and adds the warp sums in float64 once per tile: L = 19, G = ceil(tiles / grid) + 4 + grid.
bn_act_bwd mode 0 keeps fp32 throughout: blocks = min(ceil(items C/8 / 4096), 8 SMs), L = nwin ceil(items / (blocks rpi)) + rpi,
G = blocks.  Squares of fp16 values are exact in fp32.

bn_finalize (float64): m = S1 / n, var = max(S2 / n - m^2, 0).  With E1, E2 the sums bounds, dm = E1 / n + v |m| and
dvar = E2 / n + (2 |m| + dm) dm + 4 v (S2 / n + m^2).  For a channel with |mean| / std = r, E2 / n ~ L u var (1 + r^2): the 1 + r^2
amplification.  invstd = 1 / sqrt(var + eps) moves by at most dvar / (2 (max(var - dvar, 0) + eps)^1.5), plus its fp32 rounding u invstd.
The reference variance is the two-pass float64 sum of (z - m)^2, and eps is the fp32 value the kernel receives.  Running statistics:
rm = (1 - mom) rm0 + mom m, rv = (1 - mom) rv0 + mom var n / (n - 1) (var itself for n = 1), each rounded once to fp32.

bn_act_apply and bn_act_bwd mode 1: sc = RN32(gamma invstd), sh = RN32(beta - mean sc), y = fma(z, sc, sh):
|y - lin| <= 1.01 u (|z gi| + 3 |m gi| + |beta| + |lin|) with lin = gi (z - m) + beta, gi = gamma invstd; the slope product costs u slope |lin|.
dz = fma(sc, dy, -fma(k2, xhat, k1)) with xhat = fma(z, invstd, RN32(-m invstd)), k1 = RN32(sc RN32(RN32(S1) RN32(1 / RN32(n)))), k2 likewise
(1 / rows is rounded twice once rows > 2^24), dy = the (da + dap) sum and slope product in fp32.  To first order
|dz - dz_ref| <= 1.01 u (3 |gi dy| + 7 |k1| + |k2| (|m invstd| + 8 |xhat|) + |dz_ref|), k1 = gi S1 / n, k2 = gi S2 / n on the kernel's sums.
The slope decision and each pool window's winner are the kernel's own: taken from y recomputed in fp32 from the stored z (as
test_train_units_darknet.gpu_y), the first maximum in scan order (0,0), (0,1), (1,0), (1,1); bn_act_apply<1> and bn_act_bwd are also checked
to pick the same winner directly.  The fused max-pool's reference is the window's maximum of the references, bounded by the largest bound.

Weight gradients (mma.sync, fp32 accumulators): test_conv_contract.acc_bound with K = the pixels one warp accumulator sums (32 per tile times
the block's tiles) and P = 8 warps + the blocks' fp32 atomics.  conv0_wgrad_bn forms dz in shared memory and rounds it to fp16 before the
MMAs: its bound adds sum |x| (E_dz + half an fp16 ulp of |dz|).

Pools, reorg, reorg backward and head_grad_prepare's dz are bit-exact.  maxpool2x2_s1_bwd adds up to four fp16 gradients in fp32 and rounds
once: E = 3 u sum |g|.  head_grad_prepare's dbias: ceil(n / 256) terms per thread, a 5-level shuffle tree and 8 warp partials in order:
L = ceil(n / 256) + 13, G = 0.

The CPU tests check the bounds themselves: a float32 stand-in of each kernel (its summation order emulated) passes, and each plausible wrong
variant is rejected.  The figures of each group (worst err / bound, worst invstd error per |mean| / std) are recorded with `record` and
written to $YB_PARITY_OUT/train_ops_measured.json.
"""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_conv_contract import (MEASURED, SENTINEL, acc_bound, bits, check_f16, check_f32, epilogue, nchw, np64, pool_np, record,
                                sentinel, sms, ulp16)

DEV = 'cuda'
gpu = pytest.mark.gpu
R32 = 2.0 ** -24            # fp32 unit roundoff
R64 = 2.0 ** -53
EPS = float(np.float32(1e-5))
MOM = float(np.float32(0.01))
H100_SMS = 132


TRAIN_MEASURED = {}


def _own(group, fn):
    """Run a recording helper of test_conv_contract for `group`, keeping the figures in TRAIN_MEASURED (written to
    $YB_PARITY_OUT/train_ops_measured.json) and out of conv_measured.json."""
    if not group:
        return fn(None)
    key = 'train_ops.' + group
    if group in TRAIN_MEASURED:
        MEASURED[key] = TRAIN_MEASURED[group]
    try:
        return fn(key)
    finally:
        if key in MEASURED:
            TRAIN_MEASURED[group] = MEASURED.pop(key)
        out = os.environ.get('YB_PARITY_OUT')
        if out:
            os.makedirs(out, exist_ok=True)
            for name, d in (('conv_measured.json', MEASURED), ('train_ops_measured.json', TRAIN_MEASURED)):
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


# ------------------------------------------------------------------------------------------------------------------------------------
# launch geometry restated from the host code
# ------------------------------------------------------------------------------------------------------------------------------------
def stats_geometry(rows, c, nsm):
    """bn_stats: (L, G) of the module docstring."""
    rpi = 256 // (c // 8)
    blocks = min(-(-rows // (rpi * 16)), 8 * nsm)
    return 4, -(-rows // (4 * blocks * rpi)) + rpi + blocks


def bwd_geometry(items, c, nwin, nsm):
    """bn_act_bwd mode 0 (grid_for_groups with 16 items per thread)."""
    c8 = c // 8
    rpi = 256 // c8
    blocks = max(1, min(-(-items * c8 // 4096), 8 * nsm))
    return nwin * -(-items // (blocks * rpi)) + rpi, blocks


def conv0_stats_geometry(tiles, nsm):
    grid = min(tiles, 2 * nsm)
    return 19, -(-tiles // grid) + 4 + grid


def conv_epilogue_stats_geometry(rows, nsm):
    """conv_igemm_kernel (a 5-level shuffle tree over a warp's 32 rows, at most 8 warps per column of a tile in fp32, each tile in float64)
    and conv_c32_kernel_v1 (the tree, then float64): at most L = 13, G = rows / 32 + 8 SMs."""
    return 13, rows // 32 + 8 * nsm


def sum_err(A, L, G):
    return 1.01 * (L * R32 + (G + 64) * R64) * np.asarray(A, dtype=np.float64)


# ------------------------------------------------------------------------------------------------------------------------------------
# references and bounds
# ------------------------------------------------------------------------------------------------------------------------------------
def finalize_ref(S1, S2, var_ref, n, E1, E2, rm0, rv0, eps=EPS, mom=MOM):
    """(refs, bounds) of bn_finalize's mean, invstd, running mean, running var from the exact sums' bounds E1, E2."""
    S1, S2, var = (np.asarray(t, dtype=np.float64) for t in (S1, S2, var_ref))
    rm0, rv0 = np64(rm0), np64(rv0)
    m = S1 / n
    dm = E1 / n + R64 * np.abs(m)
    dvar = E2 / n + (2 * np.abs(m) + dm) * dm + 4 * R64 * (np.abs(S2) / n + m * m)
    inv = 1.0 / np.sqrt(var + eps)
    lo = np.maximum(var - dvar, 0.0) + eps
    dinv = 0.5 * dvar / lo ** 1.5 + 1.01 * R32 * inv
    unb = var * n / (n - 1) if n > 1 else var
    dunb = dvar * n / (n - 1) if n > 1 else dvar
    rm = (1 - mom) * rm0 + mom * m
    rv = (1 - mom) * rv0 + mom * unb
    e_rm = mom * dm + 1.01 * R32 * (np.abs(rm) + mom * dm) + 4 * R64 * (np.abs(rm0) + np.abs(m))
    e_rv = mom * dunb + 1.01 * R32 * (np.abs(rv) + mom * dunb) + 4 * R64 * (np.abs(rv0) + np.abs(unb))
    ref = dict(mean=m, invstd=inv, rm=rm, rv=rv)
    bound = dict(mean=dm + 1.01 * R32 * (np.abs(m) + dm), invstd=dinv, rm=e_rm, rv=e_rv)
    return ref, bound


def fold32(mean, invstd, gamma, beta):
    """The kernels' per-channel constants: sc = RN32(gamma invstd), sh = RN32(beta - mean sc) (one rounding: fmaf)."""
    sc = f32(np64(gamma) * np64(invstd))
    sh = f32(np64(beta) - np64(mean) * sc.astype(np.float64))
    return sc, sh


def y32(z16, sc, sh):
    """fmaf(z, sc, sh) in fp32 (the fp16 x fp32 product is exact in float64)."""
    return f32(np64(z16) * sc.astype(np.float64) + sh.astype(np.float64))


def win4(a):
    """[B,H,W,C] -> [B,H/2,W/2,C,4], window elements in scan order (0,0), (0,1), (1,0), (1,1)."""
    b, h, w, c = a.shape
    return a.reshape(b, h // 2, 2, w // 2, 2, c).transpose(0, 1, 3, 5, 2, 4).reshape(b, h // 2, w // 2, c, 4)


def unwin4(a):
    b, oh, ow, c, _ = a.shape
    return a.reshape(b, oh, ow, c, 2, 2).transpose(0, 1, 4, 2, 5, 3).reshape(b, 2 * oh, 2 * ow, c)


def first_max_onehot(y, last=False):
    w = win4(y)
    idx = (3 - np.argmax(w[..., ::-1], -1)) if last else np.argmax(w, -1)
    return unwin4((np.arange(4) == idx[..., None]).astype(np.float64)), idx


def apply_ref(z16, mean, invstd, gamma, beta, slope, pool):
    """(ref, E, the kernel's fp32 y) of bn_act_apply over [B,H,W,C] (channels last)."""
    z = np64(z16)
    m, gi, bt = np64(mean), np64(gamma) * np64(invstd), np64(beta)
    lin = gi * (z - m) + bt
    e_lin = 1.01 * R32 * (np.abs(z * gi) + 3 * np.abs(m * gi) + np.abs(bt) + np.abs(lin))
    yk = y32(z16, *fold32(mean, invstd, gamma, beta))
    pos = yk > 0
    ref = np.where(pos, lin, lin * slope)
    E = np.where(pos, e_lin, slope * e_lin + R32 * slope * (np.abs(lin) + e_lin))
    if pool:
        ref, E = win4(ref).max(-1), win4(E).max(-1)
    return ref, E, yk


def bwd_ref(z16, mean, invstd, gamma, beta, slope, da16, dap16, window, has_bn, last_max=False):
    """fp64 dy (the kernel's slope and routing decisions), xhat and the per-element bound terms of bn_act_bwd."""
    z = np64(z16)
    if has_bn:
        yk = y32(z16, *fold32(mean, invstd, gamma, beta))
        gi = np64(gamma) * np64(invstd)
        xhat = (z - np64(mean)) * np64(invstd)
        mi = np.abs(np64(mean) * np64(invstd)) * np.ones_like(z)
    else:
        yk = z16.astype(np.float32) if isinstance(z16, np.ndarray) else np64(z16).astype(np.float32)
        gi, xhat, mi = np.ones(z.shape[-1]), np.zeros_like(z), np.zeros_like(z)
    g = np64(da16) if da16 is not None else np.zeros_like(z)
    if dap16 is not None:
        oh, idx = first_max_onehot(yk, last_max)
        g = g + oh * np.repeat(np.repeat(np64(dap16), 2, 1), 2, 2)
    dy = np.where(yk > 0, g, g * slope)
    return dict(dy=dy, xhat=xhat, mi=mi, gi=gi * np.ones(z.shape[-1]), yk=yk, has_bn=has_bn)


def bwd_sums_ref(r, L, G):
    dy, xhat = r['dy'], r['xhat']
    e_dy = 2 * R32 * np.abs(dy)
    e_x = 1.01 * R32 * (r['mi'] + np.abs(xhat))
    ax = tuple(range(dy.ndim - 1))
    S1, S2 = dy.sum(ax), (dy * xhat).sum(ax)
    E1 = sum_err(np.abs(dy).sum(ax), L, G) + e_dy.sum(ax)
    E2 = sum_err(np.abs(dy * xhat).sum(ax), L, G) + (np.abs(dy) * e_x + np.abs(xhat) * e_dy).sum(ax)
    return S1, S2, E1, E2


def dz_ref(r, S1k, S2k, n, missing_inv_rows=False):
    gi = r['gi']
    scale = (1.0 if missing_inv_rows else 1.0 / n) if r['has_bn'] else 0.0        # without BatchNorm k1 = k2 = 0
    k1, k2 = gi * np64(S1k) * scale, gi * np64(S2k) * scale
    dz = gi * r['dy'] - k1 - k2 * r['xhat']
    E = 1.01 * R32 * (3 * np.abs(gi * r['dy']) + 7 * np.abs(k1) + np.abs(k2) * (r['mi'] + 8 * np.abs(r['xhat'])) + np.abs(dz))
    return dz, E


def dz_kernel32(r, sums, n, has_bn, sc):
    """A float32 stand-in of bn_act_bwd mode 1 (fmaf emulated in float64)."""
    c = r['dy'].shape[-1]
    dy = f32(r['dy'])
    if not has_bn:
        return dy.astype(np.float16)
    inv_rows = np.float32(1.0) / np.float32(n)
    k1 = f32(sc.astype(np.float64) * f32(np.float64(f32(sums[:c])) * np.float64(inv_rows)))
    k2 = f32(sc.astype(np.float64) * f32(np.float64(f32(sums[c:])) * np.float64(inv_rows)))
    xh = f32(r['xhat'])          # within u of the fma the kernel computes: the stand-in's own rounding
    inner = f32(k2.astype(np.float64) * xh + k1)
    return f32(sc.astype(np.float64) * dy - inner).astype(np.float16)


# ------------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------------
# (mean, std) per channel, cycled over C: |mean| / std of 0, 1, 30 and 300 at two scales, a constant channel and an all-zero channel
CHANNELS = [(0.0, 1.0), (0.5, 0.5), (3.0, 0.1), (30.0, 0.1), (0.0, 0.05), (-0.05, 0.05), (-1.5, 0.05), (15.0, 0.05),
            (1.5, 0.0), (0.0, 0.0), (0.2, 2.0), (-0.7, 0.3)]


def offset_of(c):
    m, s = CHANNELS[c % len(CHANNELS)]
    return ('zero' if m == 0 else 'const') if s == 0 else 'r%g' % round(abs(m) / s)


def stats_input(rows, c, ld, gen, device):
    ms = torch.tensor([CHANNELS[i % len(CHANNELS)] for i in range(c)], dtype=torch.float32, device=device)
    z = torch.full((rows, ld), float('nan'), dtype=torch.float16, device=device)
    z[:, :c] = (torch.randn(rows, c, generator=gen, device=device) * ms[:, 1] + ms[:, 0]).half()
    return z


def exact_stats(z, c, chunk=1 << 22):
    """float64 S1, S2, A1 (= sum |z|), two-pass variance of the stored z, chunked on the device."""
    S1 = torch.zeros(c, dtype=torch.float64, device=z.device)
    S2, A1 = torch.zeros_like(S1), torch.zeros_like(S1)
    for i in range(0, z.shape[0], chunk):
        t = z[i:i + chunk, :c].double()
        S1 += t.sum(0)
        S2 += (t * t).sum(0)
        A1 += t.abs().sum(0)
    n = z.shape[0]
    m = S1 / n
    V = torch.zeros_like(S1)
    for i in range(0, n, chunk):
        V += ((z[i:i + chunk, :c].double() - m) ** 2).sum(0)
    return np64(S1), np64(S2), np64(A1), np64(V / n)


def bn_params(c, gen):
    gamma = torch.rand(c, generator=gen) + 0.5
    gamma[1::3] *= -1                       # a negative gamma reverses the order inside each window
    gamma[c // 2] = 1e-3
    beta = torch.randn(c, generator=gen) * 0.2
    return gamma, beta


# ------------------------------------------------------------------------------------------------------------------------------------
# CPU: the bounds accept float32 stand-ins and reject plausible wrong variants
# ------------------------------------------------------------------------------------------------------------------------------------
def emulated_bn_stats(z16, c, nsm):
    """bn_stats' summation order: each thread's trips of four grid-stride rows in float32, everything after that in float64."""
    rows = z16.shape[0]
    rpi = 256 // (c // 8)
    blocks = min(-(-rows // (rpi * 16)), 8 * nsm)
    stride = blocks * rpi
    per = -(-rows // stride)
    zz = np.zeros((per * stride, c), dtype=np.float32)
    zz[:rows] = z16[:, :c].astype(np.float32)
    zz = zz.reshape(per, blocks, rpi, c)
    s = np.zeros((blocks, rpi, c))
    q = np.zeros_like(s)
    for k0 in range(0, per, 4):
        ts = np.zeros((blocks, rpi, c), dtype=np.float32)
        tq = np.zeros_like(ts)
        for k in range(k0, min(k0 + 4, per)):
            ts += zz[k]
            tq += zz[k] * zz[k]
        s += ts
        q += tq
    return np.concatenate([s.sum((0, 1)), q.sum((0, 1))])


def finalize_standin(sums, n, c, rm0, rv0, variant=None):
    m = sums[:c] / n
    var = np.maximum(sums[c:] / n - m * m, 0)
    inv = 1.0 / (np.sqrt(var) + EPS) if variant == 'eps_outside_sqrt' else 1.0 / np.sqrt(var + EPS)
    unb = var if (variant == 'biased_running_var' or n == 1) else var * n / (n - 1)
    return dict(mean=f32(m), invstd=f32(inv), rm=f32((1 - MOM) * rm0 + MOM * m), rv=f32((1 - MOM) * rv0 + MOM * unb))


def check_stats(tag, got, ref, bound, group=None):
    for q in ('mean', 'invstd', 'rm', 'rv'):
        check32('%s %s' % (tag, q), got[q], ref[q], bound[q], group and group + '_' + q)


def cpu_stats_case(rows, c=32, seed=0):
    gen = torch.Generator().manual_seed(seed)
    z = stats_input(rows, c, c, gen, 'cpu').numpy()
    S1, S2, A1, var = exact_stats(torch.from_numpy(z), c)
    L, G = stats_geometry(rows, c, H100_SMS)
    E1, E2 = sum_err(A1, L, G), sum_err(S2, L, G)
    rm0, rv0 = np.linspace(-0.5, 0.5, c), np.linspace(0.5, 2.0, c)
    ref, bound = finalize_ref(S1, S2, var, rows, E1, E2, rm0, rv0)
    return z, (S1, S2, E1, E2), rm0, rv0, ref, bound


@pytest.mark.parametrize('rows', [1, 2, 777, 100003])
def test_stats_bound_accepts_float32_standin(rows):
    c = 32
    z, (S1, S2, E1, E2), rm0, rv0, ref, bound = cpu_stats_case(rows, c, rows)
    sums = emulated_bn_stats(z, c, H100_SMS)
    assert np.all(np.abs(sums[:c] - S1) <= E1) and np.all(np.abs(sums[c:] - S2) <= E2)
    check_stats('float32 stand-in', finalize_standin(sums, rows, c, rm0, rv0), ref, bound)
    check_stats('float64 stand-in', finalize_standin(np.concatenate([S1, S2]), rows, c, rm0, rv0), ref, bound)
    if rows == 1:
        assert np.all(ref['invstd'] == 1 / np.sqrt(EPS)) and np.all(ref['rv'] == (1 - MOM) * rv0)


@pytest.mark.parametrize('variant', ['biased_running_var', 'eps_outside_sqrt'])
def test_stats_bound_rejects_wrong_variants(variant):
    rows, c = 777, 32
    z, (S1, S2, E1, E2), rm0, rv0, ref, bound = cpu_stats_case(rows, c, 5)
    got = finalize_standin(emulated_bn_stats(z, c, H100_SMS), rows, c, rm0, rv0, variant)
    with pytest.raises(AssertionError, match='^stand-in (rv|invstd)'):
        check_stats('stand-in', got, ref, bound)


def apply_case(seed=3, b=2, h=6, w=10, c=32):
    gen = torch.Generator().manual_seed(seed)
    z = (torch.randn(b, h, w, c, generator=gen) * 1.5).half()
    z[0, :2, :2, :] = 0.75                                          # a tied window in every channel
    z[1, 2:4, 4:6, :8] = z[1, 2, 4, :8]
    gamma, beta = bn_params(c, gen)
    mean = (torch.randn(c, generator=gen) * 0.3).float()
    invstd = (torch.rand(c, generator=gen) + 0.5).float()
    return z.numpy(), mean.numpy(), invstd.numpy(), gamma.numpy(), beta.numpy()


def apply_standin(z16, mean, invstd, gamma, beta, slope, pool, variant=None):
    if variant == 'channel_group_offset_8':
        mean, invstd, gamma, beta = (np.roll(t, -8) for t in (mean, invstd, gamma, beta))
    y = y32(z16, *fold32(mean, invstd, gamma, beta))
    if variant == 'slope_on_wrong_side':
        a = np.where(y > 0, f32(y * np.float32(slope)), y)
    else:
        a = np.where(y > 0, y, f32(y * np.float32(slope)))
    if pool:
        a = win4(a).max(-1)
    a = a.astype(np.float16)
    if variant == 'one_ulp_on_small_elements':
        small = np.abs(a) < np.float16(0.25)
        a = np.where(small, np.nextafter(a, np.float16(np.inf)), a)
    return a


@pytest.mark.parametrize('pool', [False, True])
def test_apply_bound_accepts_standin_and_rejects_variants(pool):
    z, mean, invstd, gamma, beta = apply_case()
    ref, E, _ = apply_ref(z, mean, invstd, gamma, beta, 0.1, pool)
    check16('stand-in', apply_standin(z, mean, invstd, gamma, beta, 0.1, pool), ref, E)
    for variant in ('channel_group_offset_8', 'slope_on_wrong_side', 'one_ulp_on_small_elements'):
        with pytest.raises(AssertionError, match='^' + variant):
            check16(variant, apply_standin(z, mean, invstd, gamma, beta, 0.1, pool, variant), ref, E)


@pytest.mark.parametrize('has_bn', [1, 0])
def test_bwd_bound_accepts_standin_and_rejects_variants(has_bn):
    z, mean, invstd, gamma, beta = apply_case(7)
    gen = torch.Generator().manual_seed(8)
    b, h, w, c = z.shape
    dap = (torch.randn(b, h // 2, w // 2, c, generator=gen) * 0.1).half().numpy()
    n = b * h * w
    r = bwd_ref(z, mean, invstd, gamma, beta, 0.1, None, dap, 1, has_bn)
    L, G = bwd_geometry(b * h * w // 4, c, 4, H100_SMS)
    S1, S2, E1, E2 = bwd_sums_ref(r, L, G)
    sums = np.concatenate([S1, S2])                 # the stand-in's sums: exact
    sc = fold32(mean, invstd, gamma, beta)[0] if has_bn else None
    ref, E = dz_ref(r, S1, S2, n)
    check16('stand-in', dz_kernel32(r, sums, n, has_bn, sc), ref, E)
    wrong = {'last_max_instead_of_first': dz_kernel32(bwd_ref(z, mean, invstd, gamma, beta, 0.1, None, dap, 1, has_bn, last_max=True), sums, n,
                                                      has_bn, sc)}
    if has_bn:
        wrong['missing_inv_rows'] = dz_kernel32(r, sums, 1, has_bn, sc)
    for variant, got in wrong.items():
        with pytest.raises(AssertionError, match='^' + variant):
            check16(variant, got, ref, E)


def c3_offsets():
    """Per-unit |mean| / std of the batch statistics of the reference's C3 training step (64 x 416^2, tests/golden/c3_train64.npz), read
    back from the running statistics it stores after the step: rm = 0.99 rm0 + 0.01 mean, rv = 0.99 rv0 + 0.01 var_unbiased."""
    from oracle import yolo2_oracle as O
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'c3_train64.npz'))
    sd = O.make_state_dict(0)
    out = {}
    for k in g.files:
        if k.startswith('buf_') and k.endswith('.running_mean'):
            key = k[4:-len('.running_mean')]
            mean = (g[k].astype(np.float64) - 0.99 * np64(sd[key + '.running_mean'])) / 0.01
            var = (g[k.replace('_mean', '_var')].astype(np.float64) - 0.99 * np64(sd[key + '.running_var'])) / 0.01
            out[key] = float((np.abs(mean) / np.sqrt(var)).max())
    return out


def invstd_bound_at(r, rows, L, G):
    """Relative invstd bound of summed statistics + bn_finalize for a channel of variance 1 and |mean| / std = r over `rows` rows
    (A1 <= n sqrt(1 + r^2)), with the summation depth (L, G) of the kernel that forms the sums."""
    A1, S2 = rows * math.sqrt(1 + r * r), rows * (1 + r * r)
    _, bound = finalize_ref(np.array([r * rows]), np.array([S2]), np.array([1.0]), rows, sum_err(A1, L, G), sum_err(S2, L, G),
                            np.zeros(1), np.ones(1))
    return float(bound['invstd'][0] * math.sqrt(1 + EPS))


def test_statistics_bound_at_the_c3_offsets():
    """The offsets the Darknet chain reaches on the C3 batch keep the derived invstd bound of every statistics path the chain runs below half
    an fp16 ulp of the normalised activation (2^-11 relative), at 64 x 416^2 and at 64 x 608^2: conv0_k16_kernel's fused statistics for
    layers1.0, the conv epilogue's for the other units, and bn_stats (the unfused form).  The old form of conv0's statistics, fp32 over all of
    a CTA's tiles (L = 16 ceil(tiles / grid) + 7), is shown above it."""
    offs = c3_offsets()
    worst, r0 = max(offs.values()), offs['layers1.0.bn']
    figs = {}
    for size in (416, 608):
        rows0 = 64 * size * size
        tiles = 64 * (size // 32) * (size // 16)
        figs['conv0_%d' % size] = invstd_bound_at(r0, rows0, *conv0_stats_geometry(tiles, H100_SMS))
        figs['bn_stats_%d' % size] = invstd_bound_at(worst, rows0, *stats_geometry(rows0, 32, H100_SMS))
        figs['conv_epilogue_%d' % size] = invstd_bound_at(worst, rows0 // 4, *conv_epilogue_stats_geometry(rows0 // 4, H100_SMS))
        grid = min(tiles, 2 * H100_SMS)
        figs['conv0_fp32_over_tiles_%d' % size] = invstd_bound_at(r0, rows0, 16 * -(-tiles // grid) + 7, grid)
    rec('c3_offsets', worst_mean_over_std=worst, layers1_0_mean_over_std=r0, **figs)
    print('C3 |mean| / std: worst %.2f (%s), layers1.0 %.2f; invstd bounds %s' % (worst, max(offs, key=offs.get), r0,
                                                                                 ', '.join('%s %.2e' % kv for kv in figs.items())))
    assert len(offs) == 22 and 1 < worst < 10
    for k, v in figs.items():
        assert (v > 2.0 ** -11) if k.startswith('conv0_fp32') else (v < 2.0 ** -11), (k, v)


def test_geometry_at_the_c3_batch():
    """bn_stats at layers1.0 of the C3 batch on 132 SMs: the grid is capped at 1056 blocks, each thread runs 41 trips of four rows."""
    assert stats_geometry(64 * 416 * 416, 32, H100_SMS) == (4, 41 + 64 + 8 * H100_SMS)
    assert conv0_stats_geometry(64 * 13 * 26, H100_SMS) == (19, 82 + 4 + 2 * H100_SMS)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


def guarded(shape_lead, c, ld, off, fill=None):
    """A [..., ld] fp16 buffer whose channels outside [off, off + c) hold the sentinel."""
    buf = sentinel(tuple(shape_lead) + (ld,))
    if fill is not None:
        buf[..., off:off + c] = fill
    return buf


def guards_kept(buf, off, c):
    return bool((bits(buf[..., :off]) == SENTINEL).all()) and bool((bits(buf[..., off + c:]) == SENTINEL).all())


def dev(t):
    return torch.as_tensor(t).to(DEV)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: conv0, both forms
# ------------------------------------------------------------------------------------------------------------------------------------
CONV0_CASES = [
    # b, h, w, kernel
    (1, 48, 32, 'conv0_tc_kernel'),
    (3, 16, 64, 'conv0_tc_kernel'),
    (2, 32, 16, 'conv0_k16_kernel'),
    (1, 64, 96, 'conv0_k16_kernel'),
    (5, 96, 160, 'conv0_k16_kernel'),
    (100, 48, 32, 'conv0_tc_kernel'),         # 300 tiles and 3 x 224^2 (294 tiles): more than the 2 x 132 persistent CTAs
    (3, 224, 224, 'conv0_k16_kernel'),
]


def conv0_inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, 3, h, w, generator=g)
    x[0, :, 0, :5] = torch.tensor([1e-6, 3e-5, 0.99999, 0.5 + 2.0 ** -12, 65.0])[:5]       # fp16 subnormal, rounding ties, > 1
    frames = torch.randint(0, 256, (b, h, w, 3), dtype=torch.uint8, generator=g)
    wt = torch.randn(32, 3, 3, 3, generator=g) * 0.3
    scale = torch.rand(32, generator=g) + 0.5
    scale[1::3] *= -1
    shift = torch.randn(32, generator=g) * 0.1
    scale[16], shift[16] = 1e-5, 0.0
    return x, frames, wt, scale, shift


def conv0_ref(x16_nchw, wt):
    return np64(F.conv2d(x16_nchw.double(), wt.half().double(), padding=1)), np64(F.conv2d(x16_nchw.double().abs(), wt.half().double().abs(), padding=1))


@gpu
@pytest.mark.parametrize('case', CONV0_CASES, ids=lambda c: '%dx%dx%d_%s' % c)
def test_conv0_vs_float64(ops, case):
    b, h, w, kern = case
    x, frames, wt, scale, shift = conv0_inputs(b, h, w, h * 7 + w + b)
    u8_16 = (frames.float() * torch.tensor(1 / 255, dtype=torch.float32)).half().permute(0, 3, 1, 2)
    wd, sc, sh = dev(wt), dev(scale), dev(shift)
    K = 48                                   # at most three k16 steps per output (two in conv0_tc_kernel)
    for form, xin, x16 in (('f32', dev(x), x.half()), ('u8', dev(frames), u8_16)):
        acc, S = conv0_ref(x16, wt)
        fn = 'yb_conv0_bn_leaky_pool_fwd' if form == 'f32' else 'yb_conv0_u8_bn_leaky_pool_fwd'
        for slope in (0.1, 0.0, 1.0):
            ref, E = epilogue(acc, S, K, 1, scale, shift, slope)
            y = sentinel((b, h // 2, w // 2, 32))
            ops.call(fn, xin, wd, sc, sh, slope, y, b, h, w, 32)
            check16('%s %s slope %g' % (kern, form, slope), nchw(y), pool_np(ref), pool_np(E), 'conv0_%s_%s' % (kern, form))
    if kern == 'conv0_tc_kernel':
        with pytest.raises(RuntimeError):                             # the raw / statistics form needs the 32 x 16 tiles
            ops.call('yb_conv0_raw_stats_fwd', dev(x), wd, torch.empty(b, h, w, 32, dtype=torch.float16, device=DEV),
                     torch.zeros(64, dtype=torch.float64, device=DEV), b, h, w, 32)
        return
    acc, S = conv0_ref(x.half(), wt)
    z = sentinel((b, h, w, 32))
    ops.call('yb_conv0_raw_fwd', dev(x), wd, z, b, h, w, 32)
    check16('%s raw' % kern, nchw(z), acc, acc_bound(S, K, 1), 'conv0_raw')
    zs = sentinel((b, h, w, 32))
    sums = torch.zeros(64, dtype=torch.float64, device=DEV)
    ops.call('yb_conv0_raw_stats_fwd', dev(x), wd, zs, sums, b, h, w, 32)
    assert torch.equal(bits(zs), bits(z)), 'raw_stats output differs from raw'
    zz = np64(z).reshape(-1, 32)
    L, G = conv0_stats_geometry(b * (h // 32) * (w // 16), sms())
    ref_s = np.concatenate([zz.sum(0), (zz * zz).sum(0)])
    E_s = sum_err(np.concatenate([np.abs(zz).sum(0), (zz * zz).sum(0)]), L, G)
    check32('conv0 raw_stats sums', sums, ref_s, E_s, 'conv0_raw_stats')


@gpu
def test_conv0_raw_stats_over_many_tiles(ops):
    """The fused statistics where every CTA loops over many tiles (24 x 416^2: 8112 tiles, 31 per CTA on 132 SMs), and bn_stats of the same z,
    against float64 sums of the stored z; then both through bn_finalize at layers1.0's offsets (a mean near 2.5 std on some channels)."""
    b, h, w = 24, 416, 416
    g = torch.Generator(device=DEV).manual_seed(24)
    x = torch.rand(b, 3, h, w, generator=g, device=DEV)
    wt = torch.randn(32, 3, 3, 3, generator=torch.Generator().manual_seed(5)) * 0.3
    wt[::4] = wt[::4].abs()                                                  # positive filters: channels with a large mean / std
    z = torch.empty(b, h, w, 32, dtype=torch.float16, device=DEV)
    sums = torch.zeros(64, dtype=torch.float64, device=DEV)
    ops.call('yb_conv0_raw_stats_fwd', x, dev(wt), z, sums, b, h, w, 32)
    rows = b * h * w
    S1, S2, A1, var = exact_stats(z.view(rows, 32), 32)
    L, G = conv0_stats_geometry(b * (h // 32) * (w // 16), sms())
    assert G - 4 - min(b * (h // 32) * (w // 16), 2 * sms()) > 16, 'fewer than 16 tiles per CTA'
    check32('conv0 raw_stats sum z', sums[:32], S1, sum_err(A1, L, G), 'conv0_raw_stats_long')
    check32('conv0 raw_stats sum z^2', sums[32:], S2, sum_err(S2, L, G), 'conv0_raw_stats_long')
    rec('c3_offsets', conv0_long_max_mean_over_std=float((np.abs(S1 / rows) / np.sqrt(var)).max()))
    check_stats_gpu('bn_stats of conv0 z', ops, z.view(rows, 32), 32, rows, 'stats_conv0_z')
    ref, bound = finalize_ref(S1, S2, var, rows, sum_err(A1, L, G), sum_err(S2, L, G), np.zeros(32), np.ones(32))
    mean, invstd = torch.empty(32, device=DEV), torch.empty(32, device=DEV)
    rm, rv = torch.zeros(32, device=DEV), torch.ones(32, device=DEV)
    ops.call('yb_bn_finalize', sums, rows, 32, EPS, MOM, rm, rv, mean, invstd)
    check_stats('conv0 fused statistics', dict(mean=mean, invstd=invstd, rm=rm, rv=rv), ref, bound, 'stats_conv0_fused')


@gpu
def test_conv0_refusals_leave_the_output_untouched(ops):
    x = torch.rand(1, 3, 40, 32, device=DEV)
    wt = torch.randn(32, 3, 3, 3, device=DEV)
    one = torch.ones(32, device=DEV)
    for name, (h, w, cout) in {'h40': (40, 32, 32), 'w24': (32, 24, 32), 'cout16': (32, 32, 16)}.items():
        y = sentinel((1, h // 2, w // 2, 32))
        z = sentinel((1, h, w, 32))
        with pytest.raises(RuntimeError):
            ops.call('yb_conv0_bn_leaky_pool_fwd', torch.rand(1, 3, h, w, device=DEV), wt, one, one, 0.1, y, 1, h, w, cout)
        with pytest.raises(RuntimeError):
            ops.call('yb_conv0_raw_fwd', torch.rand(1, 3, h, w, device=DEV), wt, z, 1, h, w, cout)
        torch.cuda.synchronize()
        assert bool((bits(y) == SENTINEL).all()) and bool((bits(z) == SENTINEL).all()), name
    del x


WGRAD0_CASES = [(1, 8, 32), (2, 64, 96), (12, 160, 160), (3, 40, 64)]     # one tile; several; 1200 tiles: more than 8 blocks per SM


def wgrad0_bound(b, h, w, S):
    tiles = b * (h // 8) * (w // 32)
    grid_min = min(tiles, sms())
    return acc_bound(S, 32 * -(-tiles // grid_min), 8 + min(tiles, 8 * sms()))


@gpu
@pytest.mark.parametrize('case', WGRAD0_CASES, ids=lambda c: '%dx%dx%d' % c)
def test_conv0_wgrad_vs_float64(ops, case):
    """conv0_wgrad on a given dz, and conv0_wgrad_bn (dz formed from z, the pooled gradient and the reduce pass's sums) against the fp64
    restatement of the whole tail: dW = sum x16 (x) dz_ref."""
    b, h, w = case
    g = torch.Generator().manual_seed(b * 100 + h + w)
    x = torch.rand(b, 3, h, w, generator=g)
    x16 = x.half().double()
    dz = (torch.randn(b, h, w, 32, generator=g) * 0.1).half()
    ref = np64(torch.nn.grad.conv2d_weight(x16, (32, 3, 3, 3), dz.double().permute(0, 3, 1, 2), padding=1))
    S = np64(torch.nn.grad.conv2d_weight(x16.abs(), (32, 3, 3, 3), dz.double().abs().permute(0, 3, 1, 2), padding=1))
    dw = torch.full((32, 3, 3, 3), float('nan'), device=DEV)
    ops.call('yb_conv0_wgrad', dev(x), dev(dz), dw, b, h, w)
    check32('conv0_wgrad', dw, ref, wgrad0_bound(b, h, w, S), 'conv0_wgrad')
    # fused form
    z = (torch.randn(b, h, w, 32, generator=g) * 0.7).half()
    z[0, :2, :2, :] = 0.25                                                 # tied windows
    gamma, beta = bn_params(32, g)
    mean = (z.double().mean((0, 1, 2))).float()
    invstd = (1 / (z.double().var((0, 1, 2), unbiased=False) + EPS).sqrt()).float()
    dap = guarded((b, h // 2, w // 2), 32, 48, 8, (torch.randn(b, h // 2, w // 2, 32, generator=g) * 0.05).half().to(DEV))
    zd, md, idd, gd, bd = dev(z), dev(mean), dev(invstd), dev(gamma), dev(beta)
    sums = torch.zeros(64, dtype=torch.float64, device=DEV)
    ops.call('yb_bn_act_bwd', 0, zd, 32, md, idd, gd, bd, 0.1, None, 0, 0, dap, 48, 8, b, h, w, 32, 1, sums, None, 0, 1)
    ops.call('yb_conv0_wgrad_bn', dev(x), zd, dap, 48, 8, md, idd, gd, bd, 0.1, sums, dw, b, h, w)
    r = bwd_ref(z.numpy(), mean.numpy(), invstd.numpy(), gamma.numpy(), beta.numpy(), 0.1, None, dap[..., 8:40].cpu().numpy(), 1, 1)
    sk = np64(sums)
    dzr, E_dz = dz_ref(r, sk[:32], sk[32:], b * h * w)
    ed16 = E_dz + 0.5 * ulp16(np.abs(dzr) + E_dz) * (1 + 2.0 ** -10)
    t = lambda a: torch.from_numpy(a).permute(0, 3, 1, 2)                                       # noqa: E731
    ref = np64(torch.nn.grad.conv2d_weight(x16, (32, 3, 3, 3), t(dzr), padding=1))
    S = np64(torch.nn.grad.conv2d_weight(x16.abs(), (32, 3, 3, 3), t(np.abs(dzr) + ed16), padding=1))
    Ex = np64(torch.nn.grad.conv2d_weight(x16.abs(), (32, 3, 3, 3), t(ed16), padding=1))
    check32('conv0_wgrad_bn', dw, ref, wgrad0_bound(b, h, w, S) + Ex, 'conv0_wgrad_bn')
    # the two-kernel path: bn_act_bwd mode 1 writes the same dz within the same bound
    dzk = torch.empty(b, h, w, 32, dtype=torch.float16, device=DEV)
    ops.call('yb_bn_act_bwd', 1, zd, 32, md, idd, gd, bd, 0.1, None, 0, 0, dap, 48, 8, b, h, w, 32, 1, sums, dzk, 32, 1)
    check16('bn_act_bwd pooled dz', dzk, dzr, E_dz, 'bwd_pooled_only_dz')


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: BatchNorm statistics
# ------------------------------------------------------------------------------------------------------------------------------------
def run_stats(ops, z, c, rows, rm0, rv0):
    sums = torch.zeros(2 * c, dtype=torch.float64, device=DEV)
    ops.call('yb_bn_stats', z, z.shape[-1], rows, c, sums)
    out = dict(sums=sums.clone())
    rm, rv = dev(rm0).float(), dev(rv0).float()
    mean, invstd = torch.empty(c, device=DEV), torch.empty(c, device=DEV)
    ops.call('yb_bn_finalize', sums, rows, c, EPS, MOM, rm, rv, mean, invstd)
    torch.cuda.synchronize()
    assert int((sums != 0).sum()) == 0, 'bn_finalize left the sums non-zero'
    out.update(mean=mean, invstd=invstd, rm=rm, rv=rv)
    return out


def check_stats_gpu(tag, ops, z, c, rows, group):
    rm0, rv0 = np.linspace(-0.5, 0.5, c).astype(np.float32), np.linspace(0.5, 2.0, c).astype(np.float32)
    got = run_stats(ops, z, c, rows, rm0, rv0)
    S1, S2, A1, var = exact_stats(z, c)
    L, G = stats_geometry(rows, c, sms())
    E1, E2 = sum_err(A1, L, G), sum_err(S2, L, G)
    check32(tag + ' sum z', got['sums'][:c], S1, E1, group + '_sums')
    check32(tag + ' sum z^2', got['sums'][c:], S2, E2, group + '_sums')
    ref, bound = finalize_ref(S1, S2, var, rows, E1, E2, rm0, rv0)
    check_stats(tag, got, ref, bound, group)
    err = np.abs(np64(got['invstd']) - ref['invstd']) / ref['invstd']
    for ch in range(c):
        rec('invstd_by_offset', **{offset_of(ch) + '_rel_err': err[ch], offset_of(ch) + '_bound': bound['invstd'][ch] / ref['invstd'][ch]})
    return got, ref


STATS_CS = [8, 16, 32, 64, 128, 256, 512, 1024, 2048]


@gpu
@pytest.mark.parametrize('c', STATS_CS)
def test_bn_stats_every_accepted_width(ops, c):
    """rows = 2^20 / C + 7 (not a multiple of 4 rpi), ld = C + 8 with NaN in the unread channels, and rows = 1."""
    gen = torch.Generator(device=DEV).manual_seed(c)
    rows = (1 << 20) // c + 7
    z = stats_input(rows, c, c + 8, gen, DEV)
    check_stats_gpu('C=%d' % c, ops, z, c, rows, 'stats')
    got, ref = check_stats_gpu('C=%d rows=1' % c, ops, z[:1], c, 1, 'stats_rows1')
    assert torch.equal(got['invstd'], torch.full((c,), 1 / math.sqrt(EPS), device=DEV).float()), 'rows = 1: invstd != 1 / sqrt(eps)'


@gpu
@pytest.mark.parametrize('c', [24, 96])
def test_bn_refusals_leave_the_output_untouched(ops, c):
    b, h, w = 2, 4, 6
    z = torch.randn(b, h, w, c, device=DEV).half()
    sums = torch.full((2 * c,), 7.0, dtype=torch.float64, device=DEV)
    with pytest.raises(RuntimeError):
        ops.call('yb_bn_stats', z, c, b * h * w, c, sums)
    p = torch.ones(c, device=DEV)
    a = sentinel((b, h, w, c))
    with pytest.raises(RuntimeError):
        ops.call('yb_bn_act_apply', z, c, p, p, p, p, 0.1, a, c, 0, b, h, w, c, 0)
    dz = sentinel((b, h, w, c))
    for mode in (0, 1):
        with pytest.raises(RuntimeError):
            ops.call('yb_bn_act_bwd', mode, z, c, p, p, p, p, 0.1, z, c, 0, None, 0, 0, b, h, w, c, 0, sums, dz, c, 1)
    torch.cuda.synchronize()
    assert bool((sums == 7.0).all()) and bool((bits(a) == SENTINEL).all()) and bool((bits(dz) == SENTINEL).all())


@gpu
def test_bn_stats_at_the_c3_length(ops):
    """layers1.0 of the C3 batch: 64 x 416^2 rows of 32 channels, the grid capped and every thread looping over 164 rows."""
    gen = torch.Generator(device=DEV).manual_seed(416)
    rows = 64 * 416 * 416
    z = stats_input(rows, 32, 32, gen, DEV)
    check_stats_gpu('C3 layers1.0', ops, z, 32, rows, 'stats_c3')


@gpu
def test_statistics_and_backward_above_2_24_rows(ops):
    """C = 8 over 17,000,003 rows (> 2^24: rows is not exact in fp32 and 1 / rows is rounded twice): bn_stats, bn_finalize and bn_act_bwd
    mode 1 once each; dz checked on the first and last million rows."""
    rows, c = 17000003, 8
    gen = torch.Generator(device=DEV).manual_seed(17)
    z = stats_input(rows, c, c, gen, DEV)
    got, _ = check_stats_gpu('rows > 2^24', ops, z, c, rows, 'stats_2_24')
    da = (torch.randn(rows, c, generator=gen, device=DEV) * 0.1).half()
    gamma, beta = bn_params(c, torch.Generator().manual_seed(3))
    gd, bd = dev(gamma), dev(beta)
    sums = torch.tensor(np.linspace(-0.3, 0.4, 2 * c) * rows, dtype=torch.float64, device=DEV)
    dz = torch.empty(rows, c, dtype=torch.float16, device=DEV)
    ops.call('yb_bn_act_bwd', 1, z, c, got['mean'], got['invstd'], gd, bd, 0.1, da, c, 0, None, 0, 0, 1, 1, rows, c, 0, sums, dz, c, 1)
    for sl in (slice(0, 1 << 20), slice(rows - (1 << 20), rows)):
        r = bwd_ref(z[sl].cpu().numpy(), got['mean'].cpu().numpy(), got['invstd'].cpu().numpy(), gamma.numpy(), beta.numpy(), 0.1,
                    da[sl].cpu().numpy(), None, 0, 1)
        sk = np64(sums)
        ref, E = dz_ref(r, sk[:c], sk[c:], rows)
        check16('dz rows > 2^24', dz[sl], ref, E, 'bwd_plain_dz_2_24')


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: apply and backward
# ------------------------------------------------------------------------------------------------------------------------------------
BWD_CASES = [
    # b, h, w, C, extra channels of every buffer, channel offset of a / da / dap
    (2, 6, 10, 32, 16, 8),
    (3, 4, 4, 8, 8, 8),
    (1, 2, 2, 2048, 8, 8),
    (4, 26, 26, 64, 0, 0),
    (2, 14, 12, 1024, 24, 16),
]


def bwd_inputs(case, seed):
    b, h, w, c, extra, off = case
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(b, h, w, c, generator=g) * 1.5 + 0.2).half()
    z[0, :2, :2, :] = 0.75                                                  # ties inside windows
    z[-1, -2:, -2:, ::2] = z[-1, -2, -2, ::2]
    gamma, beta = bn_params(c, g)
    mean = (z.double().mean((0, 1, 2)) + 0.01).float()
    invstd = (1 / (z.double().var((0, 1, 2), unbiased=False) + EPS).sqrt()).float()
    da = (torch.randn(b, h, w, c, generator=g) * 0.1).half()
    dap = (torch.randn(b, h // 2, w // 2, c, generator=g) * 0.1).half()
    return z, mean, invstd, gamma, beta, da, dap


def case_id(c):
    return '%dx%dx%d_C%d_ld+%d_off%d' % c


@gpu
@pytest.mark.parametrize('case', BWD_CASES, ids=case_id)
def test_bn_act_apply_vs_float64(ops, case):
    b, h, w, c, extra, off = case
    z, mean, invstd, gamma, beta, _, _ = bwd_inputs(case, c + h)
    zb = guarded((b, h, w), c, c + extra, 0, z.to(DEV))
    prm = [dev(t) for t in (mean, invstd, gamma, beta)]
    plain = None
    for pool in (0, 1):
        for slope in (0.1, 0.0, 1.0):
            oh, ow = (h // 2, w // 2) if pool else (h, w)
            a = guarded((b, oh, ow), c, c + extra + off, off)
            ops.call('yb_bn_act_apply', zb, c + extra, *prm, slope, a, c + extra + off, off, b, h, w, c, pool)
            ref, E, yk = apply_ref(z.numpy(), mean.numpy(), invstd.numpy(), gamma.numpy(), beta.numpy(), slope, pool)
            got = a[..., off:off + c]
            check16('apply pool=%d slope=%g' % (pool, slope), got, ref, E, 'apply_pool' if pool else 'apply')
            assert guards_kept(a, off, c), 'apply wrote outside its channel slice'
            if slope == 0.1 and not pool:
                plain = got.clone()
            if slope == 0.1 and pool:
                # the same winner as bn_act_bwd: the pixel the pooled-only backward routes the gradient to holds the pooled value
                sums = torch.zeros(2 * c, dtype=torch.float64, device=DEV)
                gp = torch.ones(b, h // 2, w // 2, c, dtype=torch.float16, device=DEV)
                dz = torch.empty(b, h, w, c, dtype=torch.float16, device=DEV)
                ops.call('yb_bn_act_bwd', 1, zb, c + extra, *prm, 0.1, None, 0, 0, gp, c, 0, b, h, w, c, 1, sums, dz, c, 1)
                wn = win4(np64(dz) != 0)
                assert bool((wn.sum(-1) == 1).all()), 'pooled gradient not routed to exactly one pixel per window'
                _, idx = first_max_onehot(yk)
                assert np.array_equal(np.argmax(wn, -1), idx), 'bn_act_bwd winner differs from the first maximum of the fp32 y'
                pv = np.take_along_axis(win4(np64(plain)), idx[..., None], -1)[..., 0]
                assert np.array_equal(pv, np64(got)), 'bn_act_apply<1> and bn_act_bwd pick different winners'


BWD_KINDS = ['plain', 'window', 'pooled']


@gpu
@pytest.mark.parametrize('has_bn', [1, 0])
@pytest.mark.parametrize('kind', BWD_KINDS)
@pytest.mark.parametrize('case', BWD_CASES, ids=case_id)
def test_bn_act_bwd_vs_float64(ops, case, kind, has_bn):
    """Mode 0 (sums of dy and dy xhat), bn_param_grad, mode 1 (dz): plain units (da), branch points (da and dap) and pooled-only units."""
    b, h, w, c, extra, off = case
    z, mean, invstd, gamma, beta, da, dap = bwd_inputs(case, c + w)
    ld = c + extra + off
    zb = guarded((b, h, w), c, c + extra, 0, z.to(DEV))
    dab = guarded((b, h, w), c, ld, off, da.to(DEV)) if kind != 'pooled' else None
    dapb = guarded((b, h // 2, w // 2), c, ld, off, dap.to(DEV)) if kind != 'plain' else None
    window = int(kind != 'plain')
    prm = [dev(t) for t in (mean, invstd, gamma, beta)] if has_bn else [None] * 4
    sums = torch.zeros(2 * c, dtype=torch.float64, device=DEV)
    args = (zb, c + extra, *prm, 0.1, dab, ld if dab is not None else 0, off, dapb, ld if dapb is not None else 0, off, b, h, w, c, window, sums)
    ops.call('yb_bn_act_bwd', 0, *args, None, 0, has_bn)
    r = bwd_ref(z.numpy(), mean.numpy(), invstd.numpy(), gamma.numpy(), beta.numpy(), 0.1, da.numpy() if dab is not None else None,
                dap.numpy() if dapb is not None else None, window, has_bn)
    items = b * h * w // (4 if window else 1)
    L, G = bwd_geometry(items, c, 4 if window else 1, sms())
    S1, S2, E1, E2 = bwd_sums_ref(r, L, G)
    group = 'bwd_%s%s' % (kind, '' if has_bn else '_nobn')
    check32('%s sum dy' % group, sums[:c], S1, E1, group + '_sums')
    if has_bn:
        check32('%s sum dy xhat' % group, sums[c:], S2, E2, group + '_sums')
    else:
        assert bool((sums[c:] == 0).all()), 'has_bn = 0: sum dy xhat must stay 0'
    # bn_param_grad: one float64 product and one fp32 rounding, bit for bit; reset off keeps the sums, reset on zeroes them
    sk = np64(sums)
    dgamma, dbeta = torch.full((c,), float('nan'), device=DEV), torch.full((c,), float('nan'), device=DEV)
    scale = 1.0 / 384
    ops.call('yb_bn_param_grad', sums, c, dgamma, dbeta, 0, scale)
    s64 = np.float64(np.float32(scale))
    assert np.array_equal(np64(dbeta), f32(sk[:c] * s64)) and np.array_equal(np64(dgamma), f32(sk[c:] * s64)), 'bn_param_grad'
    assert np.array_equal(np64(sums), sk), 'bn_param_grad with reset = 0 changed the sums'
    # mode 1 on the kernel's own sums
    dz = guarded((b, h, w), c, c + 16, 0)
    ops.call('yb_bn_act_bwd', 1, *args, dz, c + 16, has_bn)
    ref, E = dz_ref(r, sk[:c], sk[c:], b * h * w)
    check16('%s dz' % group, dz[..., :c], ref, E, group + '_dz')
    assert guards_kept(dz, 0, c), 'dz written outside its C channels'
    if not has_bn:
        assert np.array_equal(np64(dz[..., :c]), np64(f32(r['dy']).astype(np.float16))), 'has_bn = 0: dz != RN16(dy)'
    ops.call('yb_bn_param_grad', sums, c, dgamma, dbeta, 1, 1.0)
    torch.cuda.synchronize()
    assert bool((sums == 0).all()), 'bn_param_grad with reset = 1 left the sums non-zero'


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: pools, reorg, head gradient
# ------------------------------------------------------------------------------------------------------------------------------------
def tie_heavy(shape, seed):
    """fp16 values on a coarse grid (many ties across overlapping windows), no zeros."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-3, 4, shape, generator=g).float() + 0.5).half()


POOL_S1_SHAPES = [(2, 1, 7, 16), (2, 7, 1, 8), (1, 1, 1, 8), (3, 5, 9, 24), (2, 13, 13, 64)]


@gpu
@pytest.mark.parametrize('shape', POOL_S1_SHAPES, ids=lambda s: '%dx%dx%d_C%d' % s)
def test_maxpool2x2_s1_forward_and_backward(ops, shape):
    b, h, w, c = shape
    x = tie_heavy(shape, h * w + c)
    xn = np64(x)
    pad = np.full((b, h + 1, w + 1, c), -np.inf)
    pad[:, :h, :w] = xn
    win = np.stack([pad[:, :h, :w], pad[:, :h, 1:], pad[:, 1:, :w], pad[:, 1:, 1:]], -1)      # scan order of window (y, x)
    ref = win.max(-1)
    xb = guarded((b, h, w), c, c + 8, 0, x.to(DEV))
    y = sentinel((b, h, w, c))
    ops.call('yb_maxpool2x2_s1_f16', xb, y, b, h, w, c, c + 8)
    assert np.array_equal(np64(y), ref), 'maxpool2x2_s1 (x_ld > C)'
    # backward: each window's first maximum takes its gradient, the frame acting as -inf
    g = (torch.randn(shape, generator=torch.Generator().manual_seed(c)) * 0.3).half()
    arg = np.argmax(win, -1)
    gn = np64(g)
    dx = np.zeros((b, h + 1, w + 1, c))
    S = np.zeros_like(dx)
    for k, (oy, ox) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        sel = np.where(arg == k, gn, 0.0)
        dx[:, oy:oy + h, ox:ox + w] += sel
        S[:, oy:oy + h, ox:ox + w] += np.abs(sel)
    assert not dx[:, h].any() and not dx[:, :, w].any(), 'a pad element won a window'
    out = sentinel(shape)
    ops.call('yb_maxpool2x2_s1_bwd_f16', x.to(DEV), g.to(DEV), out, b, h, w, c)
    check16('maxpool2x2_s1_bwd', out, dx[:, :h, :w], 3 * R32 * S[:, :h, :w], 'maxpool_s1_bwd')


@gpu
def test_maxpool2x2_at_x_ld_above_c(ops):
    b, h, w, c = 3, 6, 10, 24
    x = tie_heavy((b, h, w, c), 11)
    xb = guarded((b, h, w), c, 40, 0, x.to(DEV))
    y = sentinel((b, h // 2, w // 2, c))
    ops.call('yb_maxpool2x2_f16', xb, y, b, h, w, c, 40)
    assert np.array_equal(np64(y), win4(np64(x)).max(-1))


@gpu
@pytest.mark.parametrize('shape', [(2, 6, 4, 8, 16, 8, 24), (1, 26, 26, 64, 64, 0, 256), (3, 2, 2, 16, 24, 8, 16)],
                         ids=lambda s: '%dx%dx%d_C%d_ld%d_xoff%d_yoff%d' % s)
def test_reorg_and_its_backward_bit_exact(ops, shape):
    b, h, w, c, x_ld, x_off, y_off = shape
    x = torch.randn(b, h, w, c, generator=torch.Generator().manual_seed(h + c)).half()
    xb = guarded((b, h, w), c, x_ld, x_off, x.to(DEV))
    y_ld = y_off + 4 * c + 8
    y = sentinel((b, h // 2, w // 2, y_ld))
    ops.reorg_f16(xb, y, y_ch_off=y_off, channels=c, x_ch_off=x_off)
    want = win4(np64(x)).transpose(0, 1, 2, 4, 3).reshape(b, h // 2, w // 2, 4 * c)          # channel (sh * 2 + sw) * C + c
    assert np.array_equal(np64(y[..., y_off:y_off + 4 * c]), want), 'reorg_f16'
    assert guards_kept(y, y_off, 4 * c), 'reorg_f16 wrote outside its channel slice'
    # backward: the transpose, read from channels [y_off, y_off + 4C) of a y_ld-wide gradient
    dx = sentinel((b, h, w, c))
    ops.call('yb_reorg_bwd_f16', y, y_ld, y_off, dx, b, h, w, c)
    assert torch.equal(bits(dx.cpu()), bits(x)), 'reorg_bwd is not the inverse of reorg'


@gpu
@pytest.mark.parametrize('case', [(2, 125, 128, 13, 13), (3, 30, 40, 5, 7), (1, 8, 8, 1, 1), (4, 125, 136, 19, 19)],
                         ids=lambda c: '%dx%d(%d)_%dx%d' % c)
def test_head_grad_prepare(ops, case):
    b, c, cpad, sh, sw = case
    g = torch.Generator().manual_seed(c + cpad)
    df = torch.randn(b, c, sh, sw, generator=g) * torch.logspace(-6, 1, c).view(1, c, 1, 1)
    df.view(-1)[:3] = torch.tensor([1e-9, -7e-8, 70000.0])                                   # fp16 underflow and overflow
    dz = sentinel((b, sh, sw, cpad))
    dbias = torch.full((cpad,), float('nan'), device=DEV)
    ops.call('yb_head_grad_prepare', df.to(DEV), dz, dbias, b, c, cpad, sh * sw)
    assert torch.equal(bits(dz[..., :c].cpu()), bits(df.permute(0, 2, 3, 1).half())), 'dz != RN16(dfeature)'
    assert bool((bits(dz[..., c:]) == 0).all()), 'pad channels not written as +0'
    d = np64(df)
    n = b * sh * sw
    E = sum_err(np.abs(d).sum((0, 2, 3)), -(-n // 256) + 13, 0)
    check32('head dbias', dbias[:c], d.sum((0, 2, 3)), E, 'head_dbias')
    assert bool(dbias[c:].isnan().all()), 'dbias written past C'
