"""Inception-v4 training on the GPU (b200.train_engine.Inception4Trainer), with BatchNorm on and off, and the kernel it adds.

The count-exclusive average pool's backward (yb_avgpool3x3_s1_excl_bwd_f16) bit for bit against a float32 restatement of its contract and
within fp16 rounding of float64 autograd; every block kind and the stem on an fp64 teacher's operands (inception4_train_oracle.py); the whole
step against the fp64 restatement held to the error budget of the GPU path's fp16 roundings; the loss scale's headroom; the smallest input;
loss descent and eval() after training; GraphedStep against the eager step.  Measured figures go to
$YB_PARITY_OUT/inception4_train_measured.json."""
import configparser
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception4_oracle as I
import inception4_train_oracle as T4
from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu
MEASURED = {}
SENTINEL = -12345.0
MODES = ('bn', 'nobn')


def record(name, value):
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'inception4_train_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def rel_l2(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def make_config(bn=True):
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': str(int(bn))}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                      'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    return config


def make_sd(seed, mode):
    return I.make_state_dict(seed, bn=mode == 'bn')


def make_net(sd, mode):
    import model
    import model.inception4
    net = model.inception4.Inception4(model.ConfigChannels(make_config(mode == 'bn')), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net


@pytest.fixture(scope='module')
def ops():
    from b200 import ops as _ops
    return _ops


# ------------------------------------------------------------------------------------------------------------------------------------
# count-exclusive average pool backward
# ------------------------------------------------------------------------------------------------------------------------------------
def excl_counts(h, w):
    """n(o) of every output o: the in-range taps of its 3x3 window."""
    rows = torch.full((h,), 3.0)
    cols = torch.full((w,), 3.0)
    rows[0] -= 1
    rows[-1] -= 1
    cols[0] -= 1
    cols[-1] -= 1
    return rows[:, None] * cols[None, :]


def excl_bwd_f32(dy):
    """The contract in float32 on the CPU: dx[i] = fp16(sum over i's in-range neighbours o, row-major, of dy[o] / n(o)); each term one
    round-to-nearest fp32 division, summed in fp32 in that order (an out-of-range term is +0 and leaves the sum's bits unchanged)."""
    b, h, w, c = dy.shape
    q = dy.float() / excl_counts(h, w)[None, :, :, None]
    qp = F.pad(q.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    acc = torch.zeros(b, h, w, c, dtype=torch.float32)
    for r in range(3):
        for s in range(3):
            acc = acc + qp[:, r:r + h, s:s + w, :]
    return acc.half()


@gpu
@pytest.mark.parametrize('c', [384, 1024, 1536])
@pytest.mark.parametrize('hw', [(1, 13), (13, 1), (2, 2), (11, 11), (24, 24), (49, 49)], ids=lambda t: '%dx%d' % t)
def test_excl_pool_backward(ops, hw, c):
    h, w = hw
    b = 2
    g = torch.Generator().manual_seed(h * 100 + w + c)
    dy = torch.randn(b, h, w, c, generator=g).half()
    dx = ops.avgpool3x3_s1_excl_bwd(dy.to(DEV)).cpu()
    assert torch.equal(dx.view(torch.int16), excl_bwd_f32(dy).view(torch.int16))
    # within fp16 rounding of float64 autograd of the module (contiguous NCHW: torch's channels-last CUDA float64 avg-pool backward is wrong)
    xr = torch.zeros(b, c, h, w, dtype=torch.float64, device=DEV, requires_grad=True)
    F.avg_pool2d(xr, 3, 1, 1, count_include_pad=False).backward(dy.permute(0, 3, 1, 2).double().contiguous().to(DEV))
    ref = xr.grad.permute(0, 2, 3, 1).cpu()
    xa = torch.zeros(b, c, h, w, dtype=torch.float64, device=DEV, requires_grad=True)
    F.avg_pool2d(xa, 3, 1, 1, count_include_pad=False).backward(dy.permute(0, 3, 1, 2).double().abs().contiguous().to(DEV))
    S = xa.grad.permute(0, 2, 3, 1).cpu()
    E = 2.0 ** -11 * ref.abs() + 2.0 ** -21 * S + 2.0 ** -25
    err = (dx.double() - ref).abs()
    record('excl_pool_bwd_%dx%d_c%d' % (h, w, c), float((err / E).max()))
    assert bool((err <= E).all())


@gpu
def test_excl_pool_backward_refusals_leave_the_output_untouched(ops):
    from b200 import lib
    dy = torch.ones(2, 5, 5, 16, dtype=torch.float16, device=DEV)
    dx = torch.full((2, 5, 5, 16), SENTINEL, dtype=torch.float16, device=DEV)
    for args in ((dy, dx, 2, 5, 5, 12), (dy, dx, 2, 5, 5, 0), (dy, dx, 0, 5, 5, 16), (dy[..., 1:], dx, 2, 5, 5, 8), (dy, None, 2, 5, 5, 16)):
        with pytest.raises(RuntimeError):
            ops.call('yb_avgpool3x3_s1_excl_bwd_f16', *args)
    torch.cuda.synchronize()
    assert bool((dx == SENTINEL).all())
    assert 'yb_avgpool3x3_s1_excl_bwd_f16' in lib.SIGNATURES


# ------------------------------------------------------------------------------------------------------------------------------------
# each block on an fp64 teacher's operands
# ------------------------------------------------------------------------------------------------------------------------------------
BLOCK_TOL = 3e-3
BLOCKS = ('stem', 3, 4, 5, 6, 10, 11, 18, 19)      # the stem, Mixed_3a, 4a, 5a, Inception_A, Reduction_A, Inception_B, Reduction_B, Inception_C
IN_CHANNELS = {3: 64, 4: 160, 5: 192, 6: 384, 10: 384, 11: 1024, 18: 1024, 19: 1536}


def block_input_hw(h, w, index):
    """The input grid of block features.`index` for an h x w image."""
    def s2(n):
        return (n - 3) // 2 + 1
    h, w = s2(h) - 2, s2(w) - 2                     # features.0 (stride 2), features.1 (valid); features.2 keeps the size
    for i in range(3, index):
        if i in (3, 5, 10, 18):
            h, w = s2(h), s2(w)
        elif i == 4:
            h, w = h - 2, w - 2
    return h, w


class Recorder(object):
    """What the trainer's units wrote and read during one forward and backward (test-side hooks on the trainer's unit methods): every unit's
    activation buffer and channel offset, the gradient it received, its dz and its data gradient; the largest |gradient| stored per block."""

    def __init__(self, monkeypatch):
        from b200 import train_engine as TE
        cls = TE.Inception4Trainer
        self.fwd, self.bwd, self.dgrad, self.peak, self.zero_dz = {}, {}, {}, {}, []
        f0, b0, d0, k0 = cls._unit_forward, cls._bn_unit_backward, cls._dgrad_khw, cls.block_backward

        def peak(key, t):
            blk = '.'.join(key.split('.')[:2])
            self.peak[blk] = max(self.peak.get(blk, 0.0), float(t.float().abs().max()))

        def fwd(tr, u, src, out=None, a_off=0):
            a, s = f0(tr, u, src, out, a_off)
            self.fwd[u.key] = (a, a_off)
            return a, s

        def bwd(tr, s, da, da_off, grads):
            dz = b0(tr, s, da, da_off, grads)
            self.bwd[s.u.key] = (da, da_off, dz)
            peak(s.u.key, dz)
            peak(s.u.key, da[..., da_off:da_off + s.u.cout])
            if not bool(dz.ne(0).any()):
                self.zero_dz.append(s.u.key)
            return dz

        def dgrad(tr, s, dz):
            gi = d0(tr, s, dz)
            self.dgrad[s.u.key] = gi
            peak(s.u.key, gi)
            return gi

        def block(tr, blk, g, grads):
            gi = k0(tr, blk, g, grads)
            peak('features.%d' % blk.index, gi)
            return gi
        monkeypatch.setattr(cls, '_unit_forward', fwd)
        monkeypatch.setattr(cls, '_bn_unit_backward', bwd)
        monkeypatch.setattr(cls, '_dgrad_khw', dgrad)
        monkeypatch.setattr(cls, 'block_backward', block)


def nchw64(t, c=None):
    t = t if c is None else t[..., :c]
    return t.permute(0, 3, 1, 2).double()


def unit_vs_teacher(s, a, a_off, rec, grads, sd, scale, image=None):
    """One unit against an fp64 recomputation from exactly the operands the GPU unit read: its input (fp16, or the fp32 image), its z for the
    BatchNorm (or its own activation as the ReLU mask without one), and the gradient at its output.  Returns {quantity: relative L2 error}."""
    u = s.u
    key, c = u.key, u.cout
    w64 = sd[key + '.conv.weight'].double().to(DEV)
    ain = image.double() if s.ain is None else nchw64(s.ain, u.cin)
    wr = w64 if s.ain is None else w64.half().double()
    err = {}
    conv = F.conv2d(ain, wr, stride=u.stride, padding=u.pad)
    act = nchw64(a[..., a_off:a_off + c])
    da, da_off, dz = rec.bwd[key]
    G = nchw64(da[..., da_off:da_off + c]) / scale
    if u.bn is not None:
        err['z'] = rel_l2(nchw64(s.z, c), conv)
        zg = nchw64(s.z, c).requires_grad_(True)
        gamma = sd[key + '.bn.weight'].double().to(DEV).requires_grad_(True)
        beta = sd[key + '.bn.bias'].double().to(DEV).requires_grad_(True)
        rm, rv = sd[key + '.bn.running_mean'].double().to(DEV).clone(), sd[key + '.bn.running_var'].double().to(DEV).clone()
        a_ref = F.relu(F.batch_norm(zg, rm, rv, gamma, beta, True, 0.1, 1e-3))
        err['activation'] = rel_l2(act, a_ref)
        err['running'] = max(rel_l2(u.bn.running_mean, rm), rel_l2(u.bn.running_var, rv))
        (a_ref * G).sum().backward()
        err['dz'] = rel_l2(nchw64(dz, c) / scale, zg.grad)
        err['dgamma'] = rel_l2(grads[key + '.bn.weight'], gamma.grad)
        err['dbeta'] = rel_l2(grads[key + '.bn.bias'], beta.grad)
    else:
        bias = sd[key + '.conv.bias'].double().to(DEV)
        err['activation'] = rel_l2(act, F.relu(conv + bias[None, :, None, None]))
        dz_ref = G * (act > 0)                                   # the ReLU mask of the activation the GPU kept
        err['dz'] = rel_l2(nchw64(dz, c) / scale, dz_ref)
        err['dbias'] = rel_l2(grads[key + '.conv.bias'], dz_ref.sum((0, 2, 3)))
    dz64 = nchw64(dz, c) / scale
    err['dw'] = rel_l2(grads[key + '.conv.weight'], torch.nn.grad.conv2d_weight(ain, tuple(w64.shape), dz64, stride=u.stride, padding=u.pad))
    if key in rec.dgrad:
        ref = torch.nn.grad.conv2d_input(tuple(ain.shape), w64.half().double(), dz64, stride=u.stride, padding=u.pad)
        err['dgrad'] = rel_l2(nchw64(rec.dgrad[key], u.cin) / scale, ref)
    return err


@gpu
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name', BLOCKS, ids=str)
@pytest.mark.parametrize('hw', [(107, 139), (416, 416)], ids=lambda t: '%dx%d' % t)
def test_block_vs_fp64_teacher(monkeypatch, name, hw, mode):
    """Every unit of the block on the operands the GPU read (no chain, so no amplification); the gradient each intermediate unit received
    against the fp64 sum of its consumers' data gradients from the GPU's dz (Inception_C's two fan-outs included); the gradient at the block
    input against the fp64 transpose: the branches, plus the count-exclusive pool, plus the max-pool."""
    h, w = hw
    b = 2
    sd = make_sd(3, mode)
    net = make_net(sd, mode).to(DEV).train()
    tr = net.trainer
    dev = torch.device(DEV)
    tr._plan()
    tr._repack(dev)
    tr._start_backward(dev)
    rec = Recorder(monkeypatch)
    g = torch.Generator().manual_seed(len(str(name)) + h)
    grads = {}
    image = None
    scale = tr.grad_scale
    if name == 'stem':
        image = O.synth_images(b, h, w, seed=4).to(DEV)
        out, st = tr.stem_forward(image)
        gy = (torch.randn(*out.shape, generator=g) * 1e-3).half().to(DEV)
        tr.stem_backward(st, gy * scale, grads)
        recs = st.units
    else:
        hh, ww = block_input_hw(h, w, name)
        xin = torch.randn(b, hh, ww, IN_CHANNELS[name], generator=g).abs().half().to(DEV)
        out, blk = tr.block_forward(name, xin)
        gy = (torch.randn(*out.shape, generator=g) * 1e-3).half().to(DEV)
        gin = tr.block_backward(blk, gy * scale, grads)
        recs = blk.units
    torch.cuda.synchronize()
    worst = {}
    for s in recs:
        if s.u.key == 'features.0':
            a, a_off = recs[1].ain, 0
        else:
            a, a_off = rec.fwd[s.u.key]
        for k, v in unit_vs_teacher(s, a, a_off, rec, grads, sd, scale, image).items():
            worst[k] = max(worst.get(k, 0.0), v)

    def dgrad64(c):
        u = c.u
        w64 = sd[u.key + '.conv.weight'].double().to(DEV).half().double()
        return torch.nn.grad.conv2d_input((b, u.cin, c.in_h, c.in_w), w64, nchw64(rec.bwd[u.key][2], u.cout) / scale, stride=u.stride,
                                          padding=u.pad)
    expect = {}
    if name == 'stem':
        s0, s1, s2 = recs
        expect[s2.u.key] = nchw64(gy)
        expect[s1.u.key] = dgrad64(s2)
        expect[s0.u.key] = dgrad64(s1)
    else:
        for s in recs:
            if not s.to_out:
                expect[s.u.key] = sum(dgrad64(c) for c in recs if c.src == s.name)
        fan = {s.name: sum(1 for c in recs if c.src == s.name) for s in recs if not s.to_out}
        if name == 19:
            assert fan['branch1_0'] == fan['branch2_2'] == 2, fan
    for s in recs:
        if s.u.key in expect:
            da, da_off, _ = rec.bwd[s.u.key]
            worst['da_join'] = max(worst.get('da_join', 0.0), rel_l2(nchw64(da[..., da_off:da_off + s.u.cout]) / scale, expect[s.u.key]))
    if name != 'stem':
        x64 = nchw64(xin).contiguous()
        ref = sum(dgrad64(s) for s in recs if s.src == 'x')
        pool = [s for s in recs if s.src == 'pool']
        if pool:
            xp = torch.zeros(x64.shape, dtype=torch.float64, device=DEV, requires_grad=True)
            F.avg_pool2d(xp, 3, 1, 1, count_include_pad=False).backward(sum(dgrad64(s) for s in pool).contiguous())
            ref = ref + xp.grad
        if blk.maxpool is not None:
            xm = x64.clone().requires_grad_(True)
            F.max_pool2d(xm, 3, 2).backward(nchw64(gy[..., blk.maxpool:blk.maxpool + xin.shape[-1]]).contiguous())
            ref = ref + xm.grad
        worst['grad_input'] = rel_l2(nchw64(gin) / scale, ref)
    record('block_%s_%s_%dx%d' % (name, mode, h, w), worst)
    for k, v in worst.items():
        assert v <= BLOCK_TOL, (name, k, v, worst)


# ------------------------------------------------------------------------------------------------------------------------------------
# whole step
# ------------------------------------------------------------------------------------------------------------------------------------
def block_of(name):
    return '.'.join(name.split('.')[:2])


def step_errors(f, grads, stats, f_ref, g_ref, s_ref, names):
    if not s_ref:                  # BatchNorm off: no running statistics
        stats = s_ref = {'-': torch.ones(1)}
    return T4.step_errors(f, grads, stats, f_ref, g_ref, s_ref, names)


@gpu
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('shape', [(4, 107, 139), (2, 416, 416)], ids=lambda s: '%dx%dx%d' % s)
def test_training_step_vs_fp64_restatement(monkeypatch, shape, mode):
    """The whole step against the fp64 restatement, held to the error budget of the GPU path's fp16 roundings alone
    (inception4_train_oracle.Rounding, tools/inception4_train_error_budget.py) computed here on the same batch, overall and block by block.
    The same step measures the loss scale's headroom: the gradient guard does not fire, the largest stored |gradient| stays below 65504 / 8,
    and no unit's dz is all zero.

    Without BatchNorm the budget is small (feature 1e-3, median gradient cosine 0.995) and every block is held to it.  With BatchNorm, 149
    train-mode BatchNorms over grids down to 2 x 3 amplify the fp16 roundings until the budget itself is a feature error of about 0.8 and a
    median gradient cosine near 0 (H100, both shapes): the GPU step measures the same, and a block's cosine is noise (about +-0.15) wherever
    the budget's is.  The per-block floors therefore apply where the budget keeps a correlation of at least 0.3 (the head and the last
    block with BatchNorm, every block without); the unit-level correctness is test_block_vs_fp64_teacher's."""
    b, h, w = shape
    sd = make_sd(0, mode)
    net = make_net(sd, mode).to(DEV).train()
    rec = Recorder(monkeypatch)
    x = O.synth_images(b, h, w, seed=12)
    f = net(x.to(DEV))
    R = T4.loss_weights(tuple(f.shape)).to(DEV)
    (f * R).sum().backward()
    torch.cuda.synchronize()
    tr = net.trainer
    for k, v in net.state_dict().items():
        if k.endswith('num_batches_tracked'):
            assert int(v) == 1, k
    f_ref, _, g_ref, s_ref = T4.train_step(sd, x, device=DEV)
    f_b, _, g_b, s_b = T4.train_step(sd, x, rnd=T4.Rounding(tr.grad_scale), device=DEV)
    names = sorted(g_ref)
    grads = {n: q.grad for n, q in net.named_parameters()}
    stats = {k: v for k, v in net.state_dict().items() if 'running' in k}
    gpu = step_errors(f, grads, stats, f_ref, g_ref, s_ref, names)
    bud = step_errors(f_b, g_b, s_b, f_ref, g_ref, s_ref, names)
    per = {}
    for blk in sorted({block_of(n) for n in names}):
        sel = [n for n in names if block_of(n) == blk]
        per[blk] = (step_errors(f, grads, stats, f_ref, g_ref, s_ref, sel)['grad_cosine'][0],
                    step_errors(f_b, g_b, s_b, f_ref, g_ref, s_ref, sel)['grad_cosine'][0])
    head_peak = rec.peak.get('features.21', 0.0)
    growth = max(rec.peak.values()) / max(head_peak, 1e-30)
    record('step_%s_%dx%dx%d' % ((mode,) + shape), dict(gpu=gpu, budget=bud, block_median_cosine=per, found_inf=float(tr.found_inf),
                                                        peak_grad=rec.peak, growth_from_last_block=growth, zero_dz=rec.zero_dz))
    assert float(tr.found_inf) == 0.0
    assert max(rec.peak.values()) < 65504.0 / 8, rec.peak
    assert not rec.zero_dz, rec.zero_dz
    assert gpu['feature'] <= 1.5 * bud['feature'], (gpu, bud)
    assert gpu['grad_rel_l2'][0] <= 1.25 * bud['grad_rel_l2'][0], (gpu, bud)
    assert gpu['grad_cosine'][0] >= bud['grad_cosine'][0] - 0.1, (gpu, bud)
    assert gpu['running'] <= 2 * bud['running'] + 1e-3, (gpu, bud)
    for blk, (c_gpu, c_bud) in per.items():
        if c_bud >= 0.3:
            assert c_gpu >= c_bud - (0.1 if blk in ('features.22', 'features.21') else 0.2), (blk, per)


@gpu
@pytest.mark.parametrize('mode', MODES)
def test_smallest_input_step_is_finite(mode):
    """75 x 75: Reduction_B's output, and every Inception_C's grid, is 1 x 1.  The step runs and everything it leaves is finite.  With BatchNorm
    each Inception_C channel is normalised over the batch's 2 values, whose backward multiplies the gradient by up to 1 / sqrt(eps) per unit,
    so at this size the gradient may exceed fp16: then the guard raises found_inf and zeroes the gradients instead of passing on inf."""
    net = make_net(make_sd(5, mode), mode).to(DEV).train()
    f = net(O.synth_images(2, 75, 75, seed=3).to(DEV))
    assert tuple(f.shape) == (2, 125, 1, 1)
    (f * T4.loss_weights(tuple(f.shape)).to(DEV)).sum().backward()
    torch.cuda.synchronize()
    found = float(net.trainer.found_inf)
    record('smallest_input_found_inf_%s' % mode, found)
    assert bool(torch.isfinite(f).all())
    assert all(bool(torch.isfinite(p.grad).all()) for p in net.parameters())
    assert all(bool(torch.isfinite(v).all()) for k, v in net.state_dict().items() if 'running' in k)
    if mode == 'nobn':
        assert found == 0.0
    elif found:
        assert all(not bool(p.grad.any()) for p in net.parameters())


# ------------------------------------------------------------------------------------------------------------------------------------
# after training
# ------------------------------------------------------------------------------------------------------------------------------------
# mode -> (batch, H, W, SGD learning rate).  With BatchNorm the descent needs larger grids: at 4 x 107 x 139 the last blocks normalise over 24
# values per channel and the step's fp16 noise (see test_training_step_vs_fp64_restatement) hides an 8-step descent; at 4 x 256 x 256 (144
# values) it measured 0.586 -> 0.561 (H100).  Without BatchNorm the gradients are small and a larger rate descends cleanly: 0.355 -> 0.310.
DESCENT = {'bn': (4, 256, 256, 1e-3), 'nobn': (4, 107, 139, 1e-2)}


@gpu
@pytest.mark.parametrize('mode', MODES)
def test_loss_descent_and_eval_after_training(mode):
    b, h, w, lr = DESCENT[mode]
    sd = make_sd(6, mode)
    net = make_net(sd, mode).to(DEV).train()
    x = O.synth_images(b, h, w, seed=11).to(DEV)
    oh, ow = block_input_hw(h, w, 22)
    target = T4.loss_weights((b, 125, oh, ow), seed=1).to(DEV) * 30
    opt = torch.optim.SGD(net.parameters(), lr=lr, momentum=0.9)
    losses = []
    for _ in range(8):
        opt.zero_grad(set_to_none=True)
        loss = ((net(x) - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    record('descent_%s' % mode, losses)
    net.eval()
    with torch.no_grad():
        y = net(x)
    trained = {k: v.detach().cpu() for k, v in net.state_dict().items() if not k.endswith('num_batches_tracked')}
    ref = I.inception4_forward(trained, x.cpu())
    e = ((y.cpu().double() - ref.double()).abs().max() / ref.abs().max()).item()
    e2 = rel_l2(y, ref)
    record('eval_after_train_%s' % mode, dict(max_abs=e, rel_l2=e2))
    assert all(np.isfinite(losses)) and sum(losses[-2:]) < 0.97 * sum(losses[:2]), losses
    # eight steps on four images leave small running variances in some channels, which the fp16 inference path amplifies: the relative L2
    # error is held, not the worst element (measured 1.4e-3 to 1.3e-1 max-abs over runs with BatchNorm)
    assert e2 <= 2.5e-2, (e, e2)


@gpu
@pytest.mark.parametrize('mode', MODES)
def test_graphed_training_step_matches_eager(mode):
    import model
    import train as yb_train
    cfg = make_config(mode == 'bn')
    anchors = O.anchors_yolo_voc()
    sd0 = make_sd(7, mode)
    b, h, w = 2, 107, 139
    batches = []
    for i in range(2):
        t = O.synth_targets(b, h, w, slots=6, seed=61 + i)
        batches.append(dict(tensor=O.synth_images(b, h, w, seed=71 + i).to(DEV), yx_min=t['yx_min'].to(DEV), yx_max=t['yx_max'].to(DEV),
                            cls=t['cls'].to(DEV)))

    def run(graphed):
        net = make_net(sd0, mode).to(DEV).train()
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
        run = [k for k in a if 'running' in k] or ['features.22.bias']
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
    record('graphed_vs_eager_%s' % mode, dict(losses=dict(eager=l_e, eager_again=l_e2, graphed=l_g), eager_vs_eager=ee, graphed_vs_eager=ge))
    # The graphed step is held to the eager-vs-eager spread.  With BatchNorm the step is chaotic at batch 2: the batch statistics are summed
    # with atomics, so their last bits vary from run to run, and 149 train-mode BatchNorms over grids down to 2 x 3 amplify that (the fp16
    # error budget of this step is a feature error of about 0.8).  Two eager runs' first losses differed by 2.5 %, graphed and eager by up to
    # 12.6 % (H100), so the loss bound there is 0.25; without BatchNorm the step is stable and the bound is Inception-v3's.
    assert ge['loss'] <= max(3 * ee['loss'], 5e-2 if mode == 'nobn' else 0.25), (ee, ge)
    assert ge['running'] <= 3 * ee['running'] + 1e-2, (ee, ge)
    assert ge['update_cosine'] >= min(ee['update_cosine'], 1.0) - 0.3, (ee, ge)
