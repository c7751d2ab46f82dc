"""Inception-v3 training on the GPU (b200.train_engine.InceptionTrainer) and the kernels it adds.

Kernels, element by element on their own fp16 operands: the general weight gradient (yb_conv2d_wgrad) against float64 with the bound of
test_conv_contract.py, and bit for bit against yb_conv_wgrad on the square same-padded form; the kh x kw data-gradient pack and the data
gradient, stride 2 included; the stem's raw form and weight gradient; the valid max-pool backward, the average pool as its own transpose,
and the join.  Then every Mixed block kind and the stem on an fp64 teacher's operands (inception_train_oracle.py), the whole step against the
fp64 restatement, loss descent, eval() after training, and GraphedStep against the eager step.  Measured figures go to
$YB_PARITY_OUT/inception_train_measured.json."""
import configparser
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception_oracle as I
import inception_train_oracle as T
import test_conv_contract as C
from oracle import yolo2_oracle as O
from test_inception import avg_pool_check, avg_pool_reference

DEV = 'cuda'
gpu = pytest.mark.gpu
MEASURED = {}
SENTINEL = -12345.0


def record(name, value):
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'inception_train_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def rel_l2(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def cosine(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                      'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    return config


def make_net(sd):
    import model
    import model.inception3
    net = model.inception3.Inception3(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    return net


@pytest.fixture(scope='module')
def ops():
    from b200 import ops as _ops
    return _ops


# ------------------------------------------------------------------------------------------------------------------------------------
# weight gradient
# ------------------------------------------------------------------------------------------------------------------------------------
def wgrad2_geometry(m_total, cin, cout, kh, kw, env_splits=None):
    """conv2d_wgrad_forward's launch geometry restated: accumulator columns N, splits and pixels per split (for the bound's K and P)."""
    narrow = cin % 64 != 0
    nmax = 96 if narrow else 256
    taps = kh * kw
    npg = (96 if cin % 96 == 0 else 32) if narrow else min(256 if cin >= 256 else cin, nmax)
    col_tiles = taps * -(-cin // npg)
    g = nmax // npg
    if taps == 9 and 3 < g < 9:
        g = 3
    g = min(g, col_tiles, 9)
    base_items = -(-cout // 128) * -(-col_tiles // g)
    kb_total = -(-m_total // C.WGRAD_KP)
    max_splits = (kb_total + 7) // 8
    splits, best = 1, 1e30
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for s in range(1, min(max_splits, 512) + 1):
        cost = -(-base_items * s // sms) * (-(-kb_total // s) + (11.0 if s > 1 else 3.3))
        if cost < best * 0.999:
            best, splits = cost, s
    if env_splits is not None:
        splits = env_splits
    splits = max(1, min(splits, max_splits))
    kbps = -(-kb_total // splits)
    return dict(N=g * npg, splits=-(-kb_total // kbps), pixels=kbps * C.WGRAD_KP)


GEOMS = {  # name: (kh, kw, stride, pad_h, pad_w)
    '1x1': (1, 1, 1, 0, 0), '3x3same': (3, 3, 1, 1, 1), '3x3valid': (3, 3, 1, 0, 0), '3x3s2': (3, 3, 2, 0, 0), '5x5': (5, 5, 1, 2, 2),
    '1x7': (1, 7, 1, 0, 3), '7x1': (7, 1, 1, 3, 0), '1x3': (1, 3, 1, 0, 1), '3x1': (3, 1, 1, 1, 0)}
WGRAD2_CASES = [
    # geometry, b, h, w, cin, cout, x_ld, dz_ld
    ('1x1', 2, 17, 13, 2048, 320, 2048, 320),
    ('1x1', 2, 35, 31, 288, 64, 288, 64),
    ('1x1', 2, 17, 15, 768, 192, 768, 192),      # Mixed_6b .. 6e and 7a inputs
    ('1x7', 2, 17, 15, 768, 160, 776, 160),
    ('1x1', 3, 9, 7, 160, 160, 168, 168),        # x_ld > Cin, dz_ld > Cout with NaN in the unread channels
    ('3x3same', 2, 35, 33, 96, 96, 96, 96),
    ('3x3same', 2, 8, 9, 448, 384, 448, 384),
    ('3x3valid', 2, 53, 69, 32, 32, 32, 32),      # Conv2d_2a_3x3 at 107 x 139
    ('3x3valid', 2, 25, 33, 96, 192, 96, 192),    # Conv2d_4a_3x3 (80 channels read as 96)
    ('3x3s2', 2, 35, 33, 288, 384, 288, 384),     # Mixed_6a.branch3x3
    ('3x3s2', 2, 17, 15, 96, 96, 104, 96),
    ('3x3s2', 2, 17, 17, 192, 320, 192, 328),     # Mixed_7a.branch3x3_2
    ('5x5', 2, 13, 11, 64, 64, 64, 64),
    ('1x7', 2, 17, 15, 128, 128, 128, 128),
    ('7x1', 2, 17, 15, 160, 192, 160, 192),
    ('1x7', 2, 13, 11, 192, 192, 192, 192),
    ('1x3', 2, 8, 9, 384, 384, 392, 384),
    ('3x1', 2, 8, 9, 384, 384, 384, 384),
    ('3x3same', 1, 5, 7, 64, 96, 64, 96),         # M below one tile
    ('7x1', 1, 7, 3, 32, 64, 40, 72),
]


def wgrad_operands(case):
    geo, b, h, w, cin, cout, x_ld, dz_ld = case
    kh, kw, stride, ph, pw = GEOMS[geo]
    oh, ow = (h + 2 * ph - kh) // stride + 1, (w + 2 * pw - kw) // stride + 1
    g = torch.Generator().manual_seed(cin + 7 * cout + kh * 10 + kw + h)
    x = torch.randn(b, h, w, cin, generator=g).half()
    dz = (torch.randn(b, oh, ow, cout, generator=g) * 0.1).half()
    xb = torch.full((b, h, w, x_ld), float('nan'), dtype=torch.float16)
    xb[..., :cin] = x
    dzb = torch.full((b, oh, ow, dz_ld), float('nan'), dtype=torch.float16)
    dzb[..., :cout] = dz
    return (kh, kw, stride, ph, pw), x, dz, xb.to(DEV), dzb.to(DEV)


@gpu
@pytest.mark.parametrize('case', WGRAD2_CASES, ids=lambda c: '%s_%dx%dx%d_%d-%d_ld%d,%d' % c)
def test_conv2d_wgrad_vs_float64(ops, monkeypatch, case):
    geo, b, h, w, cin, cout, x_ld, dz_ld = case
    (kh, kw, stride, ph, pw), x, dz, xb, dzb = wgrad_operands(case)
    x64, dz64 = x.permute(0, 3, 1, 2).double().to(DEV), dz.permute(0, 3, 1, 2).double().to(DEV)
    shape = (cout, cin, kh, kw)
    ref = C.np64(torch.nn.grad.conv2d_weight(x64, shape, dz64, stride=stride, padding=(ph, pw)))
    S = C.np64(torch.nn.grad.conv2d_weight(x64.abs(), shape, dz64.abs(), stride=stride, padding=(ph, pw)))
    m_total = dz.shape[0] * dz.shape[1] * dz.shape[2]
    for env in (1, None):
        if env is None:
            monkeypatch.delenv('YB_WGRAD_SPLITS', raising=False)
        else:
            monkeypatch.setenv('YB_WGRAD_SPLITS', str(env))
        gm = wgrad2_geometry(m_total, cin, cout, kh, kw, env)
        dw = torch.full((cout, kh, kw, cin), float('nan'), dtype=torch.float32, device=DEV)
        ops.call('yb_conv2d_wgrad', xb, dzb, dw, b, h, w, cin, cout, kh, kw, stride, ph, pw, x_ld, dz_ld)
        E = C.acc_bound(S, gm['pixels'], gm['splits'])
        C.check_f32('wgrad %s N=%d splits=%d' % (geo, gm['N'], gm['splits']), dw.permute(0, 3, 1, 2), ref, E, None)
        err = np.abs(C.np64(dw.permute(0, 3, 1, 2)) - ref) / np.maximum(E, 1e-300)
        record('wgrad_%s_N%d_splits%d' % (geo, gm['N'], gm['splits']), float(err.max()))
    monkeypatch.delenv('YB_WGRAD_SPLITS', raising=False)
    # OIHW times a scale, with the weight's Cin below the activation's (the padded-channel layout)
    cw = cin - 16
    out = torch.empty(cout, cw, kh, kw, dtype=torch.float32, device=DEV)
    ops.call('yb_unpack_wgrad_khw', dw, out, cout, cw, kh, kw, cin, 0.37)
    assert torch.equal(out, dw.permute(0, 3, 1, 2)[:, :cw] * torch.tensor(0.37, dtype=torch.float32, device=DEV))


@gpu
def test_conv2d_wgrad_refusals_leave_the_output_untouched(ops):
    b, h, w = 2, 9, 9
    x = torch.zeros(b, h, w, 64, dtype=torch.float16, device=DEV)
    for kh, kw, ph, pw, cin in ((8, 1, 0, 0, 64), (1, 8, 0, 0, 64), (3, 3, 3, 0, 64), (1, 3, 0, 3, 64), (3, 3, 1, 1, 48)):
        dz = torch.zeros(b, h, w, 64, dtype=torch.float16, device=DEV)
        dw = torch.full((64, kh, kw, 64), float('nan'), dtype=torch.float32, device=DEV)
        with pytest.raises(RuntimeError):
            ops.call('yb_conv2d_wgrad', x, dz, dw, b, h, w, cin, 64, kh, kw, 1, ph, pw, 64, 64)
        torch.cuda.synchronize()
        assert bool(dw.isnan().all()), (kh, kw, ph, pw, cin)


@gpu
def test_batched_khw_pack_equals_the_single_unit_packs(ops):
    """yb_pack_weights_khw_batch over every unit of the trainer (and the head): both operands bit for bit those of yb_pack_weight_khw_f16 and
    yb_pack_weight_dgrad_khw_f16, in one launch."""
    net = make_net(I.make_inception_state_dict(2)).to(DEV).train()
    tr = net.trainer
    n0 = ops.launch_count
    tr._repack(torch.device(DEV))
    assert ops.launch_count - n0 == 1
    plan = tr._pack_plan
    units = [u for k, u in tr._plan().items() if k != 'Conv2d_1a_3x3']
    assert plan.count == len(units) + 1
    for u in units:
        w = u.conv.weight.detach()
        f = ops.pack_weight_khw_f16(w, u.cout_pad, u.cin_pad)
        d = ops.pack_weight_dgrad_khw_f16(w, u.cout_pad, u.cin_pad)
        assert torch.equal(plan.fwd[u.key].view(torch.int16), f.view(torch.int16)), u.key
        assert torch.equal(plan.dgrad[u.key].view(torch.int16), d.view(torch.int16)), u.key
    head = tr._head
    assert torch.equal(head.w16.view(torch.int16), ops.pack_weight_khw_f16(head.conv.weight.detach()).view(torch.int16))
    d = torch.empty(2048, 1, 1, 128, dtype=torch.float16, device=DEV)
    ops.call('yb_pack_weight_dgrad_f16', head.conv.weight.detach(), d, 125, 2048, 1, 128)
    assert torch.equal(plan.dgrad[head.key].view(torch.int16), d.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------------------------------
# data gradient
# ------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('geo', sorted(GEOMS))
def test_data_gradient_khw_vs_float64(ops, geo):
    kh, kw, stride, ph, pw = GEOMS[geo]
    b, h, w, cin, cin_pad, cout, cout_pad = 2, 17, 15, 80, 96, 48, 64
    g = torch.Generator().manual_seed(kh * 10 + kw + stride)
    wt = torch.randn(cout, cin, kh, kw, generator=g) * (2.0 / (cin * kh * kw)) ** 0.5
    oh, ow = (h + 2 * ph - kh) // stride + 1, (w + 2 * pw - kw) // stride + 1
    dz = (torch.randn(b, oh, ow, cout, generator=g) * 0.1).half()
    # the pack: bit-exact against flip + transpose + zero pad
    wd = ops.pack_weight_dgrad_khw_f16(wt.to(DEV), cout_pad, cin_pad)
    exp = torch.zeros(cin_pad, kh, kw, cout_pad, dtype=torch.float16)
    exp[:cin, :, :, :cout] = torch.flip(wt, (2, 3)).permute(1, 2, 3, 0).half()
    assert torch.equal(wd.cpu().view(torch.int16), exp.view(torch.int16))
    dz16 = torch.zeros(b, oh, ow, cout_pad, dtype=torch.float16, device=DEV)
    dz16[..., :cout] = dz.to(DEV)
    if stride == 2:
        fh, fw = h + 2 * ph - kh + 1, w + 2 * pw - kw + 1
        dzf = torch.empty(b, fh, fw, cout_pad, dtype=torch.float16, device=DEV)
        ops.call('yb_upsample2_zero_f16', dz16, dzf, b, fh, fw, cout_pad)
    else:
        dzf = dz16
    one, zero = torch.ones(cin_pad, device=DEV), torch.zeros(cin_pad, device=DEV)
    dx = ops.conv2d_bn_act(dzf, wd, one, zero, 1.0, pad=(kh - 1 - ph, kw - 1 - pw))
    assert tuple(dx.shape) == (b, h, w, cin_pad)
    assert bool((dx[..., cin:] == 0).all()) and not bool(torch.signbit(dx[..., cin:]).any()), 'padded input channels are not exact zeros'
    w64, dz64 = wt.half().double().to(DEV), dz.permute(0, 3, 1, 2).double().to(DEV)
    ref = C.np64(torch.nn.grad.conv2d_input((b, cin, h, w), w64, dz64, stride=stride, padding=(ph, pw)))
    S = C.np64(torch.nn.grad.conv2d_input((b, cin, h, w), w64.abs(), dz64.abs(), stride=stride, padding=(ph, pw)))
    refe, E = C.epilogue(ref, S, kh * kw * cout_pad, 1, one[:cin].cpu(), zero[:cin].cpu(), 1.0)
    C.check_f16('dgrad %s' % geo, dx[..., :cin].permute(0, 3, 1, 2), refe, E, None)


# ------------------------------------------------------------------------------------------------------------------------------------
# stem, pools, join
# ------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('hw', [(107, 139), (75, 76)])
def test_stem_raw_and_weight_gradient(ops, hw):
    h, w = hw
    b = 2
    x = O.synth_images(b, h, w, seed=5).to(DEV)
    g = torch.Generator().manual_seed(h)
    wt = (torch.randn(32, 3, 3, 3, generator=g) * 0.2).to(DEV)
    z = ops.stem3x3_s2_raw(x, wt, pad=0)
    one, zero = torch.ones(32, device=DEV), torch.zeros(32, device=DEV)
    a = ops.stem3x3_s2(x, wt, one, zero, pad=0)
    pos = z > 0
    assert torch.equal(z[pos].view(torch.int16), a[pos].view(torch.int16)) and bool((a[~pos] == 0).all())
    ref = F.conv2d(x.double(), wt.double(), stride=2).permute(0, 2, 3, 1)
    assert C.rel_err(z, ref) <= 1e-3
    dz = (torch.randn(b, z.shape[1], z.shape[2], 32, generator=g) * 0.1).half().to(DEV)
    dw = ops.stem3x3_s2_wgrad(x, dz, pad=0)
    ref = torch.nn.grad.conv2d_weight(x.double(), (32, 3, 3, 3), dz.permute(0, 3, 1, 2).double(), stride=2)
    e = rel_l2(dw, ref)
    record('stem_wgrad_rel_l2_%dx%d' % hw, e)
    assert e <= 2e-6, e


@gpu
@pytest.mark.parametrize('hw', [(17, 17), (35, 33), (8, 9)])
def test_valid_maxpool_backward_bit_exact(ops, hw):
    h, w = hw
    b, c, ld, off = 2, 48, 80, 16
    g = torch.Generator().manual_seed(h * w)
    x = (torch.randint(0, 4, (b, c, h, w), generator=g).float() * 0.5).half()      # few levels: many ties
    oh, ow = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    dy = torch.randn(b, c, oh, ow, generator=g).half()
    xr = x.float().requires_grad_(True)
    F.max_pool2d(xr, 3, 2).backward(dy.float())
    exp = xr.grad.half().permute(0, 2, 3, 1)
    dyb = torch.full((b, oh, ow, ld), SENTINEL, dtype=torch.float16)
    dyb[..., off:off + c] = dy.permute(0, 2, 3, 1)
    dx = ops.maxpool3x3_s2_valid_bwd(x.permute(0, 2, 3, 1).contiguous().to(DEV), dyb.to(DEV), off)
    assert torch.equal(dx.cpu().view(torch.int16), exp.contiguous().view(torch.int16))


@gpu
def test_avgpool_is_its_own_transpose(ops):
    g = torch.Generator().manual_seed(9)
    b, h, w, c = 2, 17, 15, 64
    dy = torch.randn(b, h, w, c, generator=g).half()
    xr = torch.zeros(b, c, h, w, dtype=torch.float64, requires_grad=True)
    F.avg_pool2d(xr, 3, 1, 1, count_include_pad=True).backward(dy.permute(0, 3, 1, 2).double())
    got = ops.avgpool3x3_s1(dy.to(DEV))
    _, E = avg_pool_reference(dy)
    exact = avg_pool_check(got.cpu(), xr.grad.permute(0, 2, 3, 1).numpy(), E)
    assert exact > 0.9 * got.numel()


@gpu
@pytest.mark.parametrize('n', [2, 3, 4])
def test_join_rounds_the_sum_once(ops, n):
    g = torch.Generator().manual_seed(n)
    terms = [(torch.randn(3, 9, 7, 64, generator=g) * (1 + i)).half() for i in range(n)]
    got = ops.join([t.to(DEV) for t in terms])
    ref = sum(C.np64(t) for t in terms)
    E = (n - 1) * C.U * sum(np.abs(C.np64(t)) for t in terms)
    sure = C.rn16(ref - E) == C.rn16(ref + E)
    assert (C.np64(got).astype(np.float16)[sure] == C.rn16(ref)[sure]).all() and sure.any()


# ------------------------------------------------------------------------------------------------------------------------------------
# each block on an fp64 teacher's operands
# ------------------------------------------------------------------------------------------------------------------------------------
BLOCK_TOL = 3e-3
IN_SHAPE = {  # block -> channels of its input
    'Mixed_5b': 192, 'Mixed_6a': 288, 'Mixed_6b': 768, 'Mixed_7a': 768, 'Mixed_7b': 1280}


def block_input_hw(h, w, name):
    # Conv2d_1a (stride 2), 2a (valid), max-pool, 4a (valid), max-pool; then the stride-2 blocks Mixed_6a and Mixed_7a
    hh = (((h - 3) // 2 + 1 - 2 - 3) // 2 + 1 - 2 - 3) // 2 + 1
    ww = (((w - 3) // 2 + 1 - 2 - 3) // 2 + 1 - 2 - 3) // 2 + 1
    if name >= 'Mixed_6b':
        hh, ww = (hh - 3) // 2 + 1, (ww - 3) // 2 + 1
    if name >= 'Mixed_7b':
        hh, ww = (hh - 3) // 2 + 1, (ww - 3) // 2 + 1
    return hh, ww


class Recorder(object):
    """What the trainer's units read and wrote during one block's forward and backward (test-side hooks on the trainer's unit methods)."""

    def __init__(self, monkeypatch):
        from b200 import train_engine as TE
        self.fwd, self.bwd, self.dgrad = {}, {}, {}
        f0, b0, d0 = TE.InceptionTrainer._bn_unit_forward, TE.InceptionTrainer._bn_unit_backward, TE.InceptionTrainer._dgrad_khw

        def fwd(tr, u, z, ain, out=None, a_off=0, **extra):
            a, s = f0(tr, u, z, ain, out, a_off, **extra)
            self.fwd[u.key] = (a, a_off)
            return a, s

        def bwd(tr, s, da, da_off, grads):
            dz = b0(tr, s, da, da_off, grads)
            self.bwd[s.u.key] = (da, da_off, dz)
            return dz

        def dgrad(tr, s, dz):
            gi = d0(tr, s, dz)
            self.dgrad[s.u.key] = gi
            return gi
        monkeypatch.setattr(TE.InceptionTrainer, '_bn_unit_forward', fwd)
        monkeypatch.setattr(TE.InceptionTrainer, '_bn_unit_backward', bwd)
        monkeypatch.setattr(TE.InceptionTrainer, '_dgrad_khw', dgrad)


def nchw64(t, c=None):
    t = t if c is None else t[..., :c]
    return t.permute(0, 3, 1, 2).double()


def unit_vs_teacher(s, rec, grads, sd, scale, image=None):
    """One unit against an fp64 recomputation from exactly the operands the GPU unit read: its input (fp16, or the fp32 image), its z for
    the BatchNorm, and the gradient at its output.  Returns {quantity: relative L2 error}."""
    u = s.u
    key, c = u.key, u.cout
    w64 = sd[key + '.conv.weight'].double().to(DEV)
    ain = image.double() if s.ain is None else nchw64(s.ain, u.cin)
    err = {}
    z_ref = F.conv2d(ain, w64.half().double() if s.ain is not None else w64, stride=u.stride, padding=u.pad)
    err['z'] = rel_l2(nchw64(s.z, c), z_ref)
    zg = nchw64(s.z, c).requires_grad_(True)
    gamma = sd[key + '.bn.weight'].double().to(DEV).requires_grad_(True)
    beta = sd[key + '.bn.bias'].double().to(DEV).requires_grad_(True)
    rm, rv = sd[key + '.bn.running_mean'].double().to(DEV).clone(), sd[key + '.bn.running_var'].double().to(DEV).clone()
    a_ref = F.relu(F.batch_norm(zg, rm, rv, gamma, beta, True, 0.1, 1e-3))
    a, a_off = rec.fwd[key]
    err['activation'] = rel_l2(nchw64(a[..., a_off:a_off + c]), a_ref)
    err['running'] = max(rel_l2(u.bn.running_mean, rm), rel_l2(u.bn.running_var, rv))
    da, da_off, dz = rec.bwd[key]
    G = nchw64(da[..., da_off:da_off + c]) / scale
    (a_ref * G).sum().backward()
    err['dz'] = rel_l2(nchw64(dz, c) / scale, zg.grad)
    err['dgamma'] = rel_l2(grads[key + '.bn.weight'], gamma.grad)
    err['dbeta'] = rel_l2(grads[key + '.bn.bias'], beta.grad)
    if u.cout_pad != c:
        assert bool((dz[..., c:] == 0).all()), '%s: padded dz channels' % key
    dz64 = nchw64(dz, c) / scale
    err['dw'] = rel_l2(grads[key + '.conv.weight'], torch.nn.grad.conv2d_weight(ain, tuple(w64.shape), dz64, stride=u.stride, padding=u.pad))
    if key in rec.dgrad:
        gi = rec.dgrad[key]
        ref = torch.nn.grad.conv2d_input(tuple(ain.shape), w64.half().double(), dz64, stride=u.stride, padding=u.pad)
        err['dgrad'] = rel_l2(nchw64(gi, u.cin) / scale, ref)
        if gi.shape[-1] > u.cin:
            assert bool((gi[..., u.cin:] == 0).all()), '%s: padded input channels of the data gradient' % key
    return err, (dz64 if key in rec.dgrad else None)


@gpu
@pytest.mark.parametrize('name', ['stem', 'Mixed_5b', 'Mixed_6a', 'Mixed_6b', 'Mixed_7a', 'Mixed_7b'])
@pytest.mark.parametrize('hw', [(107, 139), (416, 416)])
def test_block_vs_fp64_teacher(monkeypatch, name, hw):
    """Every unit of the block on the operands the GPU read (test_train_units.py's method: no chain, so no amplification), and the gradient
    at the block input against the fp64 transpose of the block from the GPU's dz: the branch data gradients, the average pool's transpose and
    the max-pool's, summed once."""
    h, w = hw
    b = 2
    sd = I.make_inception_state_dict(3)
    net = make_net(sd).to(DEV).train()
    tr = net.trainer
    dev = torch.device(DEV)
    tr._plan()
    tr._repack(dev)
    tr._start_backward(dev)
    rec = Recorder(monkeypatch)
    g = torch.Generator().manual_seed(len(name) + h)
    grads = {}
    image = None
    if name == 'stem':
        image = O.synth_images(b, h, w, seed=4).to(DEV)
        out, st = tr.stem_forward(image)
        gy = (torch.randn(*out.shape, generator=g) * 1e-3).half().to(DEV)
        tr.stem_backward(st, gy * tr.grad_scale, grads)
        recs = st.units
    else:
        hh, ww = block_input_hw(h, w, name)
        xin = torch.randn(b, hh, ww, IN_SHAPE[name], generator=g).abs().half().to(DEV)
        out, blk = tr.block_forward(name, xin)
        gy = (torch.randn(*out.shape, generator=g) * 1e-3).half().to(DEV)
        gin = tr.block_backward(blk, gy * tr.grad_scale, grads)
        recs = blk.units
    torch.cuda.synchronize()
    worst, terms = {}, {}
    for s in recs:
        err, dz64 = unit_vs_teacher(s, rec, grads, sd, tr.grad_scale, image)
        for k, v in err.items():
            worst[k] = max(worst.get(k, 0.0), v)
        if dz64 is not None and name != 'stem' and s.src in ('x', 'pool'):
            u = s.u
            w64 = sd[u.key + '.conv.weight'].double().to(DEV).half().double()
            gx = torch.nn.grad.conv2d_input((b, u.cin, s.in_h, s.in_w), w64, dz64, stride=u.stride, padding=u.pad)
            terms[s.src] = terms.get(s.src, 0) + gx
    # the gradient each intermediate unit was handed against the fp64 transpose of what reads its output, from the GPU's dz: the sum of its
    # consumers' data gradients (branch3x3_1 <- 2a + 2b and branch3x3dbl_2 <- 3a + 3b in Mixed_7b), or in the stem the max-pool transpose
    scale = tr.grad_scale

    def dgrad64(c):
        u = c.u
        w64 = sd[u.key + '.conv.weight'].double().to(DEV).half().double()
        return torch.nn.grad.conv2d_input((b, u.cin, c.in_h, c.in_w), w64, nchw64(rec.bwd[u.key][2], u.cout) / scale, stride=u.stride,
                                          padding=u.pad)

    def maxpool_t(a, g64):
        am = nchw64(a).contiguous().requires_grad_(True)
        F.max_pool2d(am, 3, 2).backward(g64.contiguous())
        return am.grad

    expect = {}
    if name == 'stem':
        s1, s2a, s2b, s3b, s4a = recs
        expect[s4a.u.key] = maxpool_t(st.a5, nchw64(gy))
        expect[s3b.u.key] = dgrad64(s4a)
        expect[s2b.u.key] = maxpool_t(st.a3, dgrad64(s3b))
        expect[s2a.u.key] = dgrad64(s2b)
        expect[s1.u.key] = dgrad64(s2a)
    else:
        for s in recs:
            if not s.to_out:
                expect[s.u.key] = sum(dgrad64(c) for c in recs if c.src == s.name)
        assert len(expect) == sum(1 for s in recs if not s.to_out)
    for s in recs:
        if s.u.key in expect:
            da, da_off, _ = rec.bwd[s.u.key]
            worst['da_join'] = max(worst.get('da_join', 0.0), rel_l2(nchw64(da[..., da_off:da_off + s.u.cout]) / scale, expect[s.u.key]))
    if name != 'stem':
        # contiguous NCHW operands for torch's pools: its CUDA avg_pool2d backward on channels-last float64 tensors returned wrong values
        # here (1.06 relative L2 against the CPU result, while the contiguous CUDA result equals the CPU one)
        x64 = nchw64(xin).contiguous()
        ref = terms['x']
        if 'pool' in terms:
            xp = torch.zeros(x64.shape, dtype=torch.float64, device=DEV, requires_grad=True)
            F.avg_pool2d(xp, 3, 1, 1, count_include_pad=True).backward(terms['pool'].contiguous())
            ref = ref + xp.grad
        mp = {'Mixed_6a': 480, 'Mixed_7a': 512}.get(name)
        if mp is not None:
            xm = x64.clone().requires_grad_(True)
            F.max_pool2d(xm, 3, 2).backward(nchw64(gy[..., mp:]).contiguous())
            ref = ref + xm.grad
        worst['grad_input'] = rel_l2(nchw64(gin) / tr.grad_scale, ref)
    record('block_%s_%dx%d' % (name, h, w), worst)
    for k, v in worst.items():
        assert v <= BLOCK_TOL, (name, k, v, worst)


# ------------------------------------------------------------------------------------------------------------------------------------
# whole step
# ------------------------------------------------------------------------------------------------------------------------------------
def block_of(name):
    return name.split('.')[0]


@gpu
@pytest.mark.parametrize('shape', [(4, 107, 139), (2, 416, 416)], ids=lambda s: '%dx%dx%d' % s)
def test_training_step_vs_fp64_restatement(shape):
    """The whole step against the fp64 restatement, held to the error budget of the GPU path's fp16 roundings alone
    (inception_train_oracle.Rounding, tools/inception_train_error_budget.py), computed here on the same batch: ~94 train-mode BatchNorms
    amplify those roundings into a feature error of about 0.2 and gradient cosines of about 0.6, so a fixed tolerance could not tell a
    wrong block from amplification.  The step must be no further from fp64 than the budget, overall and block by block: a block whose
    gradients were zero or wrong would fall far below the budget's cosine there (the budget's per-block medians are 0.49 to 0.99)."""
    b, h, w = shape
    sd = I.make_inception_state_dict(0)
    net = make_net(sd).to(DEV).train()
    x = O.synth_images(b, h, w, seed=12)
    f = net(x.to(DEV))
    R = T.loss_weights(tuple(f.shape)).to(DEV)
    (f * R).sum().backward()
    torch.cuda.synchronize()
    for k, v in net.state_dict().items():
        if k.endswith('num_batches_tracked'):
            assert int(v) == 1, k
    f_ref, _, g_ref, s_ref = T.train_step(sd, x, device=DEV)
    f_b, _, g_b, s_b = T.train_step(sd, x, rnd=T.Rounding(net.trainer.grad_scale), device=DEV)
    names = sorted(g_ref)
    grads = {n: q.grad for n, q in net.named_parameters()}
    stats = {k: v for k, v in net.state_dict().items() if 'running' in k}
    gpu = T.step_errors(f, grads, stats, f_ref, g_ref, s_ref, names)
    bud = T.step_errors(f_b, g_b, s_b, f_ref, g_ref, s_ref, names)
    blocks = sorted({block_of(n) for n in names})
    per = {}
    for blk in blocks:
        sel = [n for n in names if block_of(n) == blk]
        per[blk] = (T.step_errors(f, grads, stats, f_ref, g_ref, s_ref, sel)['grad_cosine'][0],
                    T.step_errors(f_b, g_b, s_b, f_ref, g_ref, s_ref, sel)['grad_cosine'][0])
    record('step_%dx%dx%d' % shape, dict(gpu=gpu, budget=bud, block_median_cosine=per))
    assert gpu['feature'] <= 1.5 * bud['feature'], (gpu, bud)
    assert gpu['grad_rel_l2'][0] <= 1.25 * bud['grad_rel_l2'][0], (gpu, bud)
    assert gpu['grad_cosine'][0] >= bud['grad_cosine'][0] - 0.1, (gpu, bud)
    assert gpu['running'] <= 2 * bud['running'] + 1e-3, (gpu, bud)
    for blk, (c_gpu, c_bud) in per.items():
        assert c_gpu >= c_bud - (0.1 if blk in ('conv', 'Mixed_7c') else 0.2), (blk, per)


@gpu
def test_padded_activation_channels_are_zero():
    net = make_net(I.make_inception_state_dict(1)).to(DEV).train()
    _, saved = net.trainer.forward(O.synth_images(2, 107, 139, seed=3).to(DEV))
    a4 = saved.stem.units[4].ain                  # Conv2d_3b_1x1's output, 80 channels in 96
    assert a4.shape[-1] == 96 and bool((a4[..., 80:] == 0).all()) and not bool(torch.signbit(a4[..., 80:]).any())
    blk = saved.blocks[0]
    a5 = [s for s in blk.units if s.name == 'branch5x5_2'][0].ain       # branch5x5_1's output, 48 channels in 64
    assert a5.shape[-1] == 64 and bool((a5[..., 48:] == 0).all())


# ------------------------------------------------------------------------------------------------------------------------------------
# after training
# ------------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_loss_descent_and_eval_after_training():
    sd = I.make_inception_state_dict(6)
    net = make_net(sd).to(DEV).train()
    x = O.synth_images(4, 107, 139, seed=11).to(DEV)
    target = T.loss_weights((4, 125, 2, 3), seed=1).to(DEV) * 30
    opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9)
    losses = []
    for _ in range(8):
        opt.zero_grad(set_to_none=True)
        loss = ((net(x) - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    record('descent', losses)
    assert all(np.isfinite(losses)) and losses[-1] < 0.97 * losses[0], losses      # measured: 0.831 -> 0.795 after 6 steps
    net.eval()
    with torch.no_grad():
        y = net(x)
    trained = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    ref = I.inception_forward(trained, x.cpu())
    e = ((y.cpu().double() - ref.double()).abs().max() / ref.abs().max()).item()
    record('eval_after_train', e)
    assert e <= 2.5e-2, e        # measured 1.25e-2 on an H100 (700 W): eight steps on four images leave small running variances


@gpu
def test_graphed_training_step_matches_eager():
    import model
    import train as yb_train
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    sd0 = I.make_inception_state_dict(7)
    b, h, w = 2, 107, 139
    batches = []
    for i in range(2):
        t = O.synth_targets(b, h, w, slots=6, seed=61 + i)
        batches.append(dict(tensor=O.synth_images(b, h, w, seed=71 + i).to(DEV), yx_min=t['yx_min'].to(DEV), yx_max=t['yx_max'].to(DEV),
                            cls=t['cls'].to(DEV)))

    def run(graphed):
        net = make_net(sd0).to(DEV).train()
        inference = model.Inference(cfg, net, anchors).train()
        opt = torch.optim.SGD(net.parameters(), 1e-3, momentum=0.9)
        step = yb_train.GraphedStep(inference, opt, anchors, cfg) if graphed else (lambda d: yb_train.iterate(inference, opt, anchors, cfg, d))
        losses = [float(step(batches[i % 2])['loss_total'].item()) for i in range(3)]
        if graphed:
            assert step.launches > 0 and len(step.graphs) == 1
        return losses, {k: v.detach().float().cpu().clone() for k, v in net.state_dict().items()}

    l_e, sd_e = run(False)
    l_e2, sd_e2 = run(False)
    l_g, sd_g = run(True)
    for sd in (sd_e, sd_e2, sd_g):
        assert all(int(v) == 3 for k, v in sd.items() if k.endswith('num_batches_tracked'))

    def spread(a, b):
        """How far run b is from run a: the first loss, all running statistics together (relative L2), the median cosine of the
        parameter updates."""
        run = [k for k in a if 'running' in k]
        ra, rb = torch.cat([a[k].flatten() for k in run]), torch.cat([b[k].flatten() for k in run])
        coss = []
        for k in a:
            if 'running' in k or k.endswith('num_batches_tracked'):
                continue
            da, db = (a[k] - sd0[k].float()).flatten(), (b[k] - sd0[k].float()).flatten()
            if da.norm().item() > 0:
                coss.append((torch.dot(da, db) / (da.norm() * db.norm() + 1e-30)).item())
        return dict(running=((ra - rb).norm() / ra.norm()).item(), update_cosine=float(np.median(coss)))

    ee = dict(loss=abs(l_e[0] - l_e2[0]) / abs(l_e[0]), **spread(sd_e, sd_e2))
    ge = dict(loss=abs(l_e[0] - l_g[0]) / abs(l_e[0]), **spread(sd_e, sd_g))
    record('graphed_vs_eager', dict(losses=dict(eager=l_e, eager_again=l_e2, graphed=l_g), eager_vs_eager=ee, graphed_vs_eager=ge))
    # At batch 2 the train-mode BatchNorms make the step chaotic: the batch statistics are summed with atomics, so their last bits vary from
    # run to run, and two eager runs from the same state differed by 0.1 % to 2.6 % in the first loss (three runs on an H100).  The graphed
    # step is held to that spread, not to a fixed tolerance.
    assert ge['loss'] <= max(3 * ee['loss'], 5e-2), (ee, ge)
    assert ge['running'] <= 3 * ee['running'] + 1e-2, (ee, ge)
    assert ge['update_cosine'] >= min(ee['update_cosine'], 1.0) - 0.3, (ee, ge)
