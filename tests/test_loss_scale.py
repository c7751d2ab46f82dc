"""Dynamic loss scaling (`[train] loss_scale = dynamic`) on the GPU.

yb_grad_unscale_guard: the factor and growth tracker move exactly as torch's GradScaler rule (torch._amp_update_scale_ on the CPU), clamped
to [2^-24, 2^24]; the arena pass multiplies by 1 / f bit for bit, zeroes the buffer on a non-finite value anywhere, and leaves it alone at
f = 1.  On every training chain a dynamic step at factor f issues the same library launches as a static step at grad_scale * f, with the
same arguments except the inverse loss scale, which differs by exactly f; its gradients agree with the static step's within the spread of
two static steps (the chains' BatchNorm and weight-gradient reductions use float atomics, so two static steps from the same state already
differ in the last bits, and the step amplifies that).  Recovery from an overflow, growth, the CUDA-graph step, the launches of the default
path, and two ranks in lockstep.
"""
import configparser
import copy
import os
import socket
import time

import pytest
import torch

from oracle import yolo2_oracle as O

pytestmark = pytest.mark.gpu

DEV = 'cuda'
GUARDS = ('yb_grad_guard', 'yb_grad_unscale_guard')


@pytest.fixture(scope='module')
def ops():
    from b200 import ops as _ops
    return _ops


def make_config(loss_scale=None, interval=None, bn=True, hparam_mult=1.0):
    cfg = configparser.ConfigParser()
    train = {'cross_entropy': '1'}
    if loss_scale is not None:
        train['loss_scale'] = loss_scale
    if interval is not None:
        train['loss_scale_growth_interval'] = str(interval)
    cfg.read_dict({'batch_norm': {'enable': str(int(bn))}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                   'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                   'hparam': {k: repr(float(v) * hparam_mult) for k, v in O.HPARAM_DEFAULT.items()}, 'train': train})
    return cfg


def make_batch(b, size, seed):
    t = O.synth_targets(b, size, size, slots=4, seed=seed)
    return dict(tensor=O.synth_images(b, size, size, seed=seed + 1).to(DEV), yx_min=t['yx_min'].to(DEV), yx_max=t['yx_max'].to(DEV),
                cls=t['cls'].to(DEV))


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def assert_agree(d, s1, spread, what):
    """d (a dynamic step's gradient arena) against s1 (the static step it must equal): the least-squares scale of d on s1 is 1.  A wrong
    factor anywhere in the bookkeeping moves it to 0.5 or 2; the float-atomic reductions move it by a few percent at most (DESIGN §6).  The
    distance itself is printed beside the relative spread of two static steps, but not asserted: one pair of steps does not estimate that
    spread (two pairs of the same chain measured 8e-4 and 9e-2 apart)."""
    alpha = (torch.dot(d.double(), s1.double()) / torch.dot(s1.double(), s1.double())).item()
    err = rel_l2(d, s1)
    print('%s: scale %.6f, rel L2 %.3e, static spread %.3e, bit-identical %s' % (what, alpha, err, spread, torch.equal(d, s1)))
    assert abs(alpha - 1.0) <= 0.25, (what, alpha, err, spread)


class Recorder(object):
    """Wraps b200.ops.call: the name and the arguments of every library call (tensors as shape and dtype)."""

    def __init__(self, ops):
        self.real = ops.call
        self.calls = []

    def __call__(self, name, *args):
        self.calls.append((name, tuple(self._arg(a) for a in args)))
        return self.real(name, *args)

    @staticmethod
    def _arg(a):
        if torch.is_tensor(a):
            return ('T', tuple(a.shape), a.dtype)
        if a is None or isinstance(a, (bool, int, float, str)):
            return a
        return ('O', type(a).__name__)

    def take(self):
        calls, self.calls = self.calls, []
        return calls


def assert_same_launches(static, dynamic, f):
    """Same library calls in the same order; the guard is yb_grad_guard in static mode and yb_grad_unscale_guard in dynamic mode; every
    other argument is equal, except float arguments that are exactly f times the static one (the inverse loss scale)."""
    assert len(static) == len(dynamic)
    scaled = 0
    for (ns, as_), (nd, ad) in zip(static, dynamic):
        if ns in GUARDS or nd in GUARDS:
            assert (ns, nd) == GUARDS
            continue
        assert ns == nd and len(as_) == len(ad), (ns, nd)
        for x, y in zip(as_, ad):
            if isinstance(x, float) and x != y:
                assert y == x * f, (ns, x, y)
                scaled += 1
            else:
                assert x == y, (ns, x, y)
    assert (scaled > 0) == (f != 1.0)


# ------------------------------------------------------------------------------------------------------------------------------------
# the kernel
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_factor_update_matches_grad_scaler(ops, seed):
    """Random overflow sequences (inf, -inf or NaN planted in a buffer): found_inf, the factor and the tracker equal GradScaler's update,
    torch._amp_update_scale_ run on the CPU, step for step."""
    g = torch.Generator().manual_seed(seed)
    n, interval = 4099, 3
    clean = torch.randn(n, generator=g)
    f = torch.ones((), device=DEV)
    tracker = torch.zeros((), dtype=torch.int32, device=DEV)
    found = torch.zeros((), device=DEV)
    ref_f, ref_t = torch.ones(()), torch.zeros((), dtype=torch.int32)
    seen = set()
    for step in range(80):
        buf = clean.clone()
        bad = bool(torch.rand((), generator=g).item() < 0.35)
        if bad:
            buf[int(torch.randint(n, (), generator=g))] = (float('inf'), float('-inf'), float('nan'))[step % 3]
        dbuf = buf.to(DEV)
        ops.call('yb_grad_unscale_guard', dbuf, n, found, f, tracker, interval)
        torch._amp_update_scale_(ref_f, ref_t, torch.full((), float(bad)), 2.0, 0.5, interval)
        ref_f.clamp_(2.0 ** -24, 2.0 ** 24)
        assert found.item() == float(bad), step
        assert f.item() == ref_f.item() and tracker.item() == ref_t.item(), (step, f.item(), ref_f.item(), tracker.item(), ref_t.item())
        seen.add(f.item())
    assert len(seen) >= 3          # the sequence moved the factor both ways


def test_factor_clamped_at_both_bounds(ops):
    n = 64
    found = torch.zeros((), device=DEV)
    tracker = torch.zeros((), dtype=torch.int32, device=DEV)
    for f0, bad, interval, expect in ((2.0 ** -24, True, 5, 2.0 ** -24), (2.0 ** -23, True, 5, 2.0 ** -24), (2.0 ** 24, False, 1, 2.0 ** 24),
                                      (2.0 ** 23, False, 1, 2.0 ** 24)):
        f = torch.full((), f0, device=DEV)
        for _ in range(3):
            buf = torch.randn(n, device=DEV)
            if bad:
                buf[7] = float('inf')
            ops.call('yb_grad_unscale_guard', buf, n, found, f, tracker, interval)
            assert found.item() == float(bad)
            assert f.item() == expect and tracker.item() == 0, (f0, f.item())


@pytest.mark.parametrize('n', [3, 4096, 4099, 1 << 20 | 1])
@pytest.mark.parametrize('k', [-3, -1, 1, 6])
def test_arena_pass_divides_by_factor_exactly(ops, n, k):
    g = torch.Generator().manual_seed(n + k)
    x = torch.randn(n, generator=g) * torch.exp2(torch.randint(-20, 20, (n,), generator=g).float())
    buf = x.to(DEV)
    found = torch.full((), 7.0, device=DEV)
    f = torch.full((), 2.0 ** k, device=DEV)
    tracker = torch.zeros((), dtype=torch.int32, device=DEV)
    ops.call('yb_grad_unscale_guard', buf, n, found, f, tracker, 100)
    assert found.item() == 0.0 and tracker.item() == 1 and f.item() == 2.0 ** k
    assert torch.equal(buf.cpu().view(torch.int32), (x * 2.0 ** -k).view(torch.int32))


@pytest.mark.parametrize('where', ['first', 'last_body', 'tail'])
@pytest.mark.parametrize('bad', [float('inf'), float('nan')])
def test_arena_pass_zeroes_on_non_finite(ops, where, bad):
    n = 4099                                          # 1024 float4 and a tail of 3
    buf = torch.randn(n, device=DEV)
    buf[{'first': 0, 'last_body': 4095, 'tail': n - 1}[where]] = bad
    found = torch.zeros((), device=DEV)
    f = torch.full((), 4.0, device=DEV)
    tracker = torch.full((), 5, dtype=torch.int32, device=DEV)
    ops.call('yb_grad_unscale_guard', buf, n, found, f, tracker, 100)
    assert found.item() == 1.0 and bool((buf == 0).all())
    assert f.item() == 2.0 and tracker.item() == 0


def test_arena_pass_leaves_bits_at_factor_one(ops):
    n = 4099
    x = torch.randn(n)
    x[:4] = torch.tensor([-0.0, 1e-45, -1e-40, 3.4e38])       # signed zero, subnormals, the largest values keep their bits
    buf = x.to(DEV)
    found = torch.zeros((), device=DEV)
    f = torch.ones((), device=DEV)
    tracker = torch.zeros((), dtype=torch.int32, device=DEV)
    ops.call('yb_grad_unscale_guard', buf, n, found, f, tracker, 100)
    assert found.item() == 0.0 and torch.equal(buf.cpu().view(torch.int32), x.view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------------------------
# every training chain
# ------------------------------------------------------------------------------------------------------------------------------------
def _net(name):
    import model
    import model.densenet
    import model.inception3
    import model.inception4
    import model.mobilenet
    import model.resnet
    import model.vgg
    import model.yolo2
    anchors = O.anchors_yolo_voc()
    torch.manual_seed(0)
    bn = name != 'inception4_nobn'
    cc = model.ConfigChannels(make_config(bn=bn))
    if name == 'darknet':
        net = model.yolo2.Darknet(cc, anchors, 20)
        net.load_state_dict(O.make_state_dict(0), strict=False)
    elif name == 'tiny':
        net = model.yolo2.Tiny(cc, anchors, 20)
    elif name == 'mobilenet':
        net = model.mobilenet.MobileNet(cc, anchors, 20)
    elif name == 'resnet18':
        net = model.resnet.resnet18(cc, anchors, 20)
    elif name in ('vgg11', 'vgg11_bn'):
        import vgg_oracle as V
        net = getattr(model.vgg, name)(cc, anchors, 20)
        net.load_state_dict(V.make_state_dict(name, seed=4), strict=False)
    elif name == 'inception3':
        net = model.inception3.Inception3(cc, anchors, 20)
    elif name.startswith('inception4'):
        import inception4_oracle as I
        net = model.inception4.Inception4(cc, anchors, 20)
        net.load_state_dict(I.make_state_dict(5, bn=bn), strict=False)
    elif name == 'densenet121':
        net = model.densenet.densenet121(cc, anchors, 20)
    return net.to(DEV).train(), anchors


CHAINS = ['darknet', 'tiny', 'mobilenet', 'resnet18', 'vgg11', 'vgg11_bn', 'inception3', 'inception4_bn', 'inception4_nobn', 'densenet121']


@pytest.mark.parametrize('name', CHAINS)
def test_dynamic_step_equals_static_step_at_the_same_scale(ops, name, monkeypatch):
    """On the same parameters and batch (fused SGD at lr 0 keeps the parameters), a dynamic step at f in {0.5, 1, 2} against a static step at
    base * f: found_inf 0, the same launches (assert_same_launches) and the same gradients.  base is the chain's tuned scale halved until a
    static step at 2 * base does not overflow on this batch (on these small grids BatchNorm over a few values per channel can push some
    chains' gradients past their tuned scale)."""
    import model
    import train as yb_train
    net, anchors = _net(name)
    bn = name != 'inception4_nobn'
    inference = model.Inference(make_config(bn=bn), net, anchors).train()
    opt = torch.optim.SGD(net.parameters(), lr=0.0, fused=True)
    size = 128 if name.startswith('inception') else 64
    batch = make_batch(2, size, 60)
    trainer = net.trainer
    static_cfg, dynamic_cfg = make_config(bn=bn), make_config('dynamic', 1000, bn=bn)
    tuned = trainer.grad_scale
    base = tuned / 2
    for _ in range(30):
        trainer.grad_scale = base * 2
        yb_train.iterate(inference, opt, anchors, static_cfg, batch)
        if trainer.found_inf.item() == 0.0:
            break
        base /= 2
    print('%s: base = tuned scale %g / %g' % (name, tuned, tuned / base))
    rec = Recorder(ops)
    monkeypatch.setattr(ops, 'call', rec)

    def step(f, dynamic):
        if dynamic:
            trainer.grad_scale = base
            trainer.set_loss_scale('dynamic', 1000)
            trainer.loss_scale_state(torch.device(DEV, torch.cuda.current_device()))[0].fill_(f)
        else:
            trainer.grad_scale = base * f
        out = yb_train.iterate(inference, opt, anchors, dynamic_cfg if dynamic else static_cfg, batch)
        torch.cuda.synchronize()
        assert trainer.found_inf.item() == 0.0, (name, f, dynamic)
        if dynamic:
            assert trainer.loss_factor.item() == f and out['loss_scale'].item() == base * f
        else:
            assert 'loss_scale' not in out
        return trainer.arena.flat.clone(), rec.take()

    s1, calls_s1 = step(1.0, False)
    s2, _ = step(1.0, False)
    assert 'yb_grad_guard' in [c[0] for c in calls_s1] and 'yb_grad_unscale_guard' not in [c[0] for c in calls_s1]
    spread = rel_l2(s2, s1)
    for f in (0.5, 1.0, 2.0):
        s, calls_s = (s1, calls_s1) if f == 1.0 else step(f, False)
        d, calls_d = step(f, True)
        assert 'yb_grad_unscale_guard' in [c[0] for c in calls_d] and 'yb_grad_guard' not in [c[0] for c in calls_d]
        assert_same_launches(calls_s, calls_d, f)
        assert_agree(d, s, spread, '%s f=%g' % (name, f))


# ------------------------------------------------------------------------------------------------------------------------------------
# recovery, growth and the graphed step on Darknet-19
# ------------------------------------------------------------------------------------------------------------------------------------
HPARAM_MULT = 2.0 ** 16        # loss weights that overflow the tuned scale by several powers of two


@pytest.fixture(scope='module')
def overflow_case():
    """Darknet-19 with HPARAM_MULT times the default loss weights, one batch, and j: the smallest j >= 1 for which a static step at
    grad_scale * 2^-j does not overflow (a static step at grad_scale does).  Also that step's gradients, twice."""
    import model
    import train as yb_train
    net, anchors = _net('darknet')
    cfg = make_config(hparam_mult=HPARAM_MULT)
    inference = model.Inference(cfg, net, anchors).train()
    sd0 = copy.deepcopy(net.state_dict())
    batch = make_batch(2, 64, 70)
    opt = torch.optim.SGD(net.parameters(), lr=0.0, fused=True)
    gs = net.trainer.grad_scale
    found = []
    for j in range(0, 25):
        net.trainer.grad_scale = gs * 2.0 ** -j
        yb_train.iterate(inference, opt, anchors, cfg, batch)
        found.append(net.trainer.found_inf.item())
        if found[-1] == 0.0:
            break
    assert found[0] == 1.0 and found[-1] == 0.0, found
    j = len(found) - 1
    s1 = net.trainer.arena.flat.clone()
    yb_train.iterate(inference, opt, anchors, cfg, batch)
    assert net.trainer.found_inf.item() == 0.0
    s2 = net.trainer.arena.flat.clone()
    net.trainer.grad_scale = gs
    print('overflow case: j = %d' % j)
    return dict(net=net, anchors=anchors, inference=inference, sd0=sd0, batch=batch, j=j, gs=gs, s1=s1, s2=s2)


def _reset(case):
    net = case['net']
    net.load_state_dict(case['sd0'])
    net.trainer.grad_scale = case['gs']
    net.trainer.loss_factor = net.trainer.growth_tracker = None


def test_recovery_from_overflow(overflow_case):
    """Dynamic mode with fused Adam: exactly j skipped steps (found_inf 1, parameters unchanged, factor halved each time) down to 2^-j, then a
    step on the gradients of the static step at grad_scale * 2^-j."""
    import train as yb_train
    case = overflow_case
    _reset(case)
    net, j = case['net'], case['j']
    cfg = make_config('dynamic', 1000, hparam_mult=HPARAM_MULT)
    opt = torch.optim.Adam(net.parameters(), 1e-4, fused=True)
    before = {n: p.detach().clone() for n, p in net.named_parameters()}
    for i in range(j):
        out = yb_train.iterate(case['inference'], opt, case['anchors'], cfg, case['batch'])
        assert net.trainer.found_inf.item() == 1.0, i
        assert net.trainer.loss_factor.item() == 2.0 ** -(i + 1) and net.trainer.growth_tracker.item() == 0
        assert out['loss_scale'].item() == case['gs'] * 2.0 ** -(i + 1)
        assert all(torch.equal(p.detach(), before[n]) for n, p in net.named_parameters()), i
    yb_train.iterate(case['inference'], opt, case['anchors'], cfg, case['batch'])
    assert net.trainer.found_inf.item() == 0.0 and net.trainer.loss_factor.item() == 2.0 ** -j and net.trainer.growth_tracker.item() == 1
    assert_agree(net.trainer.arena.flat.clone(), case['s1'], rel_l2(case['s2'], case['s1']), 'recovered step at 2^-%d' % j)
    assert any(not torch.equal(p.detach(), before[n]) for n, p in net.named_parameters())


def test_growth_after_clean_steps(ops):
    """growth_interval = 2 from a base of a sixteenth of the tuned scale: the factor doubles after every second clean step; the gradients at
    the grown factor 4 agree with a static step at base * 4."""
    import model
    import train as yb_train
    net, anchors = _net('darknet')
    inference = model.Inference(make_config(), net, anchors).train()
    opt = torch.optim.SGD(net.parameters(), lr=0.0, fused=True)
    batch = make_batch(2, 64, 80)
    base = net.trainer.grad_scale / 16
    net.trainer.grad_scale = base
    cfg = make_config('dynamic', 2)
    factors, scales = [], []
    for _ in range(5):
        out = yb_train.iterate(inference, opt, anchors, cfg, batch)
        assert net.trainer.found_inf.item() == 0.0
        factors.append(net.trainer.loss_factor.item())
        scales.append(out['loss_scale'].item())
    assert factors == [1.0, 2.0, 2.0, 4.0, 4.0] and scales == [base * f for f in factors]
    yb_train.iterate(inference, opt, anchors, cfg, batch)              # at factor 4
    assert net.trainer.found_inf.item() == 0.0 and net.trainer.loss_factor.item() == 8.0
    d = net.trainer.arena.flat.clone()
    net.trainer.grad_scale = base * 4
    statics = []
    for _ in range(2):
        yb_train.iterate(inference, opt, anchors, make_config(), batch)
        assert net.trainer.found_inf.item() == 0.0
        statics.append(net.trainer.arena.flat.clone())
    assert_agree(d, statics[0], rel_l2(statics[1], statics[0]), 'grown factor 4')


def test_graphed_step_matches_eager(overflow_case):
    """GraphedStep in dynamic mode (growth_interval 1, fused capturable Adam) over j + 1 steps -- j overflows, then the clean step, which
    doubles the factor -- against eager iterate from the same state: the same found_inf, factor, tracker and loss scale after every step, and
    parameter updates that agree.  Every step runs on the starting parameters (the overflowed ones are skipped), so the sequence is the
    calibration's; later steps would run on parameters that the float-atomic reductions make differ slightly between the two runs, and a
    step near the overflow threshold could then go either way.  A capture that did not restore the factor after its warm-up steps would
    start the replays lower."""
    import train as yb_train
    case = overflow_case
    j = case['j']
    cfg = make_config('dynamic', 1, hparam_mult=HPARAM_MULT)
    net = case['net']

    def run(graphed):
        _reset(case)
        opt = torch.optim.Adam(net.parameters(), 1e-4, fused=True, capturable=True)
        if graphed:
            step = yb_train.GraphedStep(case['inference'], opt, case['anchors'], cfg)
        else:
            def step(d):
                return yb_train.iterate(case['inference'], opt, case['anchors'], cfg, d)
        traj = []
        for i in range(j + 1):
            out = step(case['batch'])
            traj.append((net.trainer.found_inf.item(), net.trainer.loss_factor.item(), int(net.trainer.growth_tracker.item()),
                         out['loss_scale'].item()))
        if graphed:
            assert len(step.graphs) == 1
            step.close()
        return traj, {n: p.detach().clone() for n, p in net.named_parameters()}

    _reset(case)
    t_e, p_e = run(False)
    t_g, p_g = run(True)
    print('eager %s\ngraph %s' % (t_e, t_g))
    assert t_e == t_g
    gs = case['gs']
    assert t_e == [(1.0, 2.0 ** -(i + 1), 0, gs * 2.0 ** -(i + 1)) for i in range(j)] + [(0.0, 2.0 ** -(j - 1), 0, gs * 2.0 ** -(j - 1))]
    sd0 = case['sd0']
    de = torch.cat([(p_e[n] - sd0[n]).flatten() for n in p_e])
    dg = torch.cat([(p_g[n] - sd0[n]).flatten() for n in p_e])
    cos = (torch.dot(de.double(), dg.double()) / (de.double().norm() * dg.double().norm())).item()
    assert de.norm().item() > 0 and cos >= 0.8, cos
    assert 0.8 <= (dg.norm() / de.norm()).item() <= 1.25


def test_capture_restores_factor(overflow_case):
    """The warm-up steps of the capture overflow (the factor halves twice) and are undone: after capture, before the first replay, the factor
    is 1 and the tracker 0."""
    import train as yb_train
    case = overflow_case
    _reset(case)
    net = case['net']
    opt = torch.optim.Adam(net.parameters(), 1e-4, fused=True, capturable=True)
    step = yb_train.GraphedStep(case['inference'], opt, case['anchors'], make_config('dynamic', 2, hparam_mult=HPARAM_MULT))
    dev = torch.device(DEV, torch.cuda.current_device())
    key = tuple(tuple(case['batch'][k].shape) for k in step.keys)
    step._capture(key, case['batch'], dev)
    torch.cuda.synchronize()
    assert net.trainer.loss_factor.item() == 1.0 and net.trainer.growth_tracker.item() == 0
    step.close()


# ------------------------------------------------------------------------------------------------------------------------------------
# the default path
# ------------------------------------------------------------------------------------------------------------------------------------
def test_default_path_launches(ops, monkeypatch):
    """Without the key, a step calls yb_grad_guard and never yb_grad_unscale_guard, creates no factor and returns no loss_scale; with
    `loss_scale = dynamic` it is the other way round, and the rest of the launches are the same."""
    import model
    import train as yb_train
    net, anchors = _net('darknet')
    inference = model.Inference(make_config(), net, anchors).train()
    opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9)
    batch = make_batch(2, 64, 90)
    rec = Recorder(ops)
    monkeypatch.setattr(ops, 'call', rec)
    out = yb_train.iterate(inference, opt, anchors, make_config(), batch)
    static = rec.take()
    names = [c[0] for c in static]
    assert names.count('yb_grad_guard') == 1 and 'yb_grad_unscale_guard' not in names
    assert 'loss_scale' not in out and net.trainer.loss_factor is None and net.trainer.loss_scale == 'static'
    with pytest.warns(RuntimeWarning, match='found_inf'):
        out = yb_train.iterate(inference, opt, anchors, make_config('dynamic'), batch)
    dynamic = rec.take()
    names = [c[0] for c in dynamic]
    assert names.count('yb_grad_unscale_guard') == 1 and 'yb_grad_guard' not in names
    assert 'loss_scale' in out and net.trainer.growth_interval == 2000
    assert_same_launches(static, dynamic, 1.0)


# ------------------------------------------------------------------------------------------------------------------------------------
# two ranks
# ------------------------------------------------------------------------------------------------------------------------------------
WORLD = 2


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(WORLD), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', device_id=torch.device('cuda', rank))
    import model
    import train as yb_train
    from b200 import ddp
    net, anchors = _net('darknet')
    inference = yb_train.ensure_model(model.Inference(make_config(), net, anchors)).train()
    opt = torch.optim.Adam(net.parameters(), 1e-4, fused=True)
    cfg = make_config('dynamic', 1000)
    batch = make_batch(2, 64, 100 + rank)
    gs = net.trainer.grad_scale
    states = []
    for i in range(2):
        # step 0: only rank 1 runs at a scale its fp16 gradients cannot hold; the all-reduced inf reaches rank 0
        net.trainer.grad_scale = gs * 2.0 ** 40 if (i == 0 and rank == 1) else gs
        yb_train.iterate(inference, opt, anchors, cfg, batch)
        torch.cuda.synchronize()
        states.append((net.trainer.found_inf.item(), net.trainer.loss_factor.item(), int(net.trainer.growth_tracker.item())))
    torch.save(states, os.path.join(out, 'rank%d.pt' % rank))
    ddp.shutdown()
    dist.destroy_process_group()


def test_two_ranks_move_the_factor_in_lockstep():
    if torch.cuda.device_count() < WORLD:
        pytest.skip('needs %d GPUs' % WORLD)
    import shutil
    import tempfile
    import torch.multiprocessing as mp
    out = tempfile.mkdtemp(prefix='yb_ls_')
    ctx = mp.start_processes(_worker, args=(_free_port(), out), nprocs=WORLD, join=False, start_method='spawn')
    deadline = time.time() + 300
    while not ctx.join(timeout=5):
        if time.time() > deadline:
            for p in ctx.processes:
                p.kill()
            pytest.fail('workers did not finish within 300 s')
    res = [torch.load(os.path.join(out, 'rank%d.pt' % r)) for r in range(WORLD)]
    shutil.rmtree(out, ignore_errors=True)
    assert res[0] == res[1]
    assert res[0] == [(1.0, 0.5, 0), (0.0, 0.5, 1)]
