"""Channel-pruned Darknet-19 and Tiny YOLOv2 on the GPU: the channel-tail conv entry (yb_conv_bn_act_tail_fwd) against the plain entry
on a zero-padded operand and against float64, its refusals, the pruned plugins against the executed reference (tests/golden/pruned.npz)
and the oracle, and the launches of full-width models, which must not reach the new entry."""
import configparser
import os

import numpy as np
import pytest
import torch

import pruned_oracle as PO
import test_conv_contract as CC
from oracle import yolo2_oracle as O

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TOL_DARKNET = 2.5e-3    # the full-width golden tests' bounds: Darknet-19 'fast' end to end (test_gpu_parity.TOL_FAST_E2E), Tiny 3e-3
TOL_TINY = 3e-3
TAIL_CINS = (8, 24, 40, 72, 104, 200, 464, 1000, 1288)


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    return config


@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'pruned.npz'))


def bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.float16 else t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------------------------------------------
# the kernel contract
# ------------------------------------------------------------------------------------------------------------------------------------
def tail_operands(ops, b, h, w, cin, cout, k, seed):
    """x fp16 NHWC [b,h,w,cin + 8] whose channels [cin, cin + 8) hold NaN and +-Inf, the same x materialised with zeros up to cin_pad,
    the fp32 weight zero-padded to cin_pad and packed, scale (some negative) and shift."""
    cin_pad = ops.round_up(cin, 32)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=g).half()
    wt = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5
    scale[1::3] *= -1
    shift = torch.randn(cout, generator=g) * 0.1
    x_nhwc = x.permute(0, 2, 3, 1)
    junk = torch.tensor([float('nan'), float('inf'), -float('inf'), float('nan')] * 2, dtype=torch.float16).expand(b, h, w, 8)
    x_tail = torch.cat([x_nhwc, junk], -1).contiguous().to(DEV)
    x_pad = torch.cat([x_nhwc, torch.zeros(b, h, w, cin_pad - cin, dtype=torch.float16)], -1).contiguous().to(DEV)
    wp = torch.zeros(cout, cin_pad, k, k)
    wp[:, :cin] = wt
    w16 = ops.pack_weight_f16(wp.to(DEV).contiguous(), 0)
    return x, wt, x_tail, x_pad, w16, scale.to(DEV), shift.to(DEV)


TILES = [(0, 0), (64, 1), (128, 1), (64, 2), (128, 2)]     # (0, 0): the library's own choice


@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('cin', TAIL_CINS)
def test_tail_conv_equals_plain_conv_on_padded_operand(ops, cin, k):
    """Every tile and both output modes: bit-identical to yb_conv_bn_act_fwd_ws on x materialised with zeros up to cin_pad (same forced
    tile, no stream-K), although the tail call's x holds NaN and Inf in channels [cin, x_ld); and inside the float64 bound of
    test_conv_contract (K counted over cin_pad).  M = 2 * 9 * 13 = 234 leaves partial 128- and 256-row tiles, Cout 136 a partial N tile."""
    b, h, w = 2, 9, 13
    slope = 0.1
    ws = ops.conv_workspace(DEV)
    for out_mode, cout in ((ops.OUT_F16_NHWC, 136), (ops.OUT_F32_NCHW, 125)):
        x, wt, x_tail, x_pad, w16, scale, shift = tail_operands(ops, b, h, w, cin, cout, k, seed=cin * 10 + k)
        acc, S = CC.conv64(x.to(DEV), wt.half().to(DEV), k)
        ref, E = CC.epilogue(CC.np64(acc), CC.np64(S), k * k * ops.round_up(cin, 32), 0, scale, shift, slope)
        for bn, mt in TILES:
            if out_mode == ops.OUT_F32_NCHW and bn * mt > 128:
                continue            # the two-consumer tile stores fp16 NHWC only
            flags = (ops.conv_force_bn(bn) | ops.conv_force_mt(mt)) if bn else 0
            if out_mode == ops.OUT_F16_NHWC:
                y_ld, off = cout + 24, 16
                y_t = torch.full((b, h, w, y_ld), float('nan'), dtype=torch.float16, device=DEV)
                y_t.view(torch.int16).fill_(CC.SENTINEL)
                y_p = y_t.clone()
            else:
                off = 0
                y_t = torch.full((b, cout, h, w), float('nan'), device=DEV)
                y_p = y_t.clone()
            ops.conv_bn_act_tail(x_tail, w16, scale, shift, slope, cin, out=y_t, out_mode=out_mode, y_ch_off=off, flags=flags)
            ops.conv_bn_act(x_pad, w16, scale, shift, slope, out=y_p, out_mode=out_mode, y_ch_off=off, workspace=ws,
                            flags=flags | ops.CONV_NO_STREAMK | ops.CONV_NO_SMALLK)
            torch.cuda.synchronize()
            tag = 'cin%d k%d mode%d tile %dx%d' % (cin, k, out_mode, bn, mt)
            assert torch.equal(bits(y_t), bits(y_p)), tag
            if out_mode == ops.OUT_F16_NHWC:
                guard = torch.cat([y_t[..., :off], y_t[..., off + cout:]], -1)
                assert bool((guard.view(torch.int16) == CC.SENTINEL).all()), tag + ': guard channels written'
                CC.check_f16(tag, y_t[..., off:off + cout].permute(0, 3, 1, 2), ref, E, group='tail')
            else:
                CC.check_f32(tag, y_t, ref, E, group='tail')


def test_tail_conv_ignores_channels_past_cin(ops):
    """Channels [cin, x_ld) of x never enter the result: zeros there and NaN / Inf there give the same bits, on a wide x_ld."""
    b, h, w, cin, cout, k = 2, 16, 16, 40, 64, 3
    x, wt, x_tail, x_pad, w16, scale, shift = tail_operands(ops, b, h, w, cin, cout, k, seed=7)
    x_zero = torch.zeros(b, h, w, 80, dtype=torch.float16, device=DEV)
    x_bad = torch.full((b, h, w, 80), float('inf'), dtype=torch.float16, device=DEV)
    x_bad[..., 60:] = float('nan')
    x_zero[..., :cin] = x_tail[..., :cin]
    x_bad[..., :cin] = x_tail[..., :cin]
    y0 = ops.conv_bn_act_tail(x_zero, w16, scale, shift, 0.1, cin)
    y1 = ops.conv_bn_act_tail(x_bad, w16, scale, shift, 0.1, cin)
    assert torch.equal(bits(y0), bits(y1)) and bool(torch.isfinite(y0.float()).all())


def test_tail_conv_refusals_leave_the_output_untouched(ops):
    from b200 import lib
    b, h, w, cin, cout, k = 1, 8, 8, 40, 64, 3
    x, wt, x_tail, x_pad, w16, scale, shift = tail_operands(ops, b, h, w, cin, cout, k, seed=3)
    y = torch.empty(b, h, w, cout, dtype=torch.float16, device=DEV)
    y.view(torch.int16).fill_(CC.SENTINEL)
    flat = torch.zeros(x_tail.numel() + 8, dtype=torch.float16, device=DEV)
    x_mis = flat[1:1 + x_tail.numel()].view(x_tail.shape)           # 2-byte aligned
    s = torch.cuda.current_stream().cuda_stream
    L = lib.load()

    def call(xx, cin_, cin_pad, x_ld, flags=0, ww=w16):
        return L.yb_conv_bn_act_tail_fwd(xx.data_ptr(), ww.data_ptr(), scale.data_ptr(), shift.data_ptr(), 0.1, y.data_ptr(), b, h, w,
                                         cin_, cin_pad, cout, k, x_ld, cout, 0, 0, flags, s)
    x_ld = x_tail.shape[-1]
    cases = {
        'cin % 8': (call(x_tail, 36, 64, x_ld), -1),
        'x_ld < cin': (call(x_tail, cin, 64, 32), -1),
        'x_ld % 8': (call(x_tail, cin, 64, 44), -1),
        'cin_pad': (call(x_tail, cin, 96, x_ld), -1),
        'misaligned x': (call(x_mis, cin, 64, x_ld), -1),
        'pool': (call(x_tail, cin, 64, x_ld, ops.CONV_POOL2X2), -2),
        'chain': (call(x_tail, cin, 64, x_ld, ops.CONV_CHAIN1X1), -2),
        'stream-K': (call(x_tail, cin, 64, x_ld, ops.CONV_FORCE_STREAMK), -2),
    }
    torch.cuda.synchronize()
    for name, (rc, want) in cases.items():
        assert rc == want, '%s: rc %d (%s)' % (name, rc, lib.last_error())
    assert bool((y.view(torch.int16) == CC.SENTINEL).all())


# ------------------------------------------------------------------------------------------------------------------------------------
# the plugins
# ------------------------------------------------------------------------------------------------------------------------------------
def build_darknet(sd, ratio=1):
    import model
    import model.yolo2
    cfg = make_config()
    dnn = model.yolo2.Darknet(model.ConfigChannels(cfg, sd if ratio == 1 else None), O.anchors_yolo_voc(), 20, ratio=ratio)
    res = dnn.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys)
    return dnn.to(DEV).eval()


def build_tiny(sd):
    import model
    import model.yolo2
    net = model.yolo2.Tiny(model.ConfigChannels(make_config(), sd), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def pruned_sd(golden):
    sd = PO.darknet_pruned_state_dict(PO.keep_from_npz(golden, 'darknet_'))
    return sd


@pytest.fixture(scope='module')
def pruned(pruned_sd):
    return build_darknet(pruned_sd)


def count_tail_launches(fn):
    from b200 import ops
    n = [0]
    orig = ops.conv_bn_act_tail

    def rec(*a, **kw):
        n[0] += 1
        return orig(*a, **kw)
    ops.conv_bn_act_tail = rec
    try:
        fn()
    finally:
        ops.conv_bn_act_tail = orig
    return n[0]


@pytest.mark.parametrize('size', [64, 416])
def test_pruned_darknet_vs_executed_reference(pruned, golden, size):
    x = O.synth_images(1, size, size, seed=10 if size == 64 else 0).to(DEV)
    n = count_tail_launches(lambda: pruned(x))
    f = pruned(x)
    ref = torch.from_numpy(golden['darknet_feature%d' % size])
    assert f.shape == ref.shape
    e = rel_err(f, ref)
    print('pruned darknet %d: rel err %.3e, %d tail launches' % (size, e, n))
    assert e <= TOL_DARKNET and n > 0


@pytest.mark.parametrize('size', [64, 416])
def test_darknet_ratio_075_vs_executed_reference(golden, size):
    dnn = build_darknet(O.make_state_dict(0, ratio=0.75), ratio=0.75)
    x = O.synth_images(1, size, size, seed=10 if size == 64 else 0).to(DEV)
    f = dnn(x)
    e = rel_err(f, torch.from_numpy(golden['ratio075_feature%d' % size]))
    assert e <= TOL_DARKNET, e


@pytest.mark.parametrize('size', [64, 416])
def test_pruned_tiny_vs_executed_reference(golden, size):
    net = build_tiny(PO.tiny_pruned_state_dict(PO.keep_from_npz(golden, 'tiny_')))
    x = O.synth_images(1, size, size, seed=10 if size == 64 else 0).to(DEV)
    n = count_tail_launches(lambda: net(x))
    f = net(x)
    ref = torch.from_numpy(golden['tiny_feature%d' % size])
    e = rel_err(f, ref)
    print('pruned tiny %d: rel err %.3e, %d tail launches' % (size, e, n))
    assert f.shape == ref.shape and e <= TOL_TINY and n > 0


def oracle_on_gpu(forward, sd, x):
    """The oracle's fp32 restatement on the GPU (TF32 off), for batch sizes the CPU would take minutes over."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            return forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV))
    finally:
        torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize('shape', [(32, 416, 416), (3, 96, 224), (2, 320, 160)])
def test_pruned_darknet_batch_and_non_square_vs_oracle(pruned, pruned_sd, shape):
    b, h, w = shape
    x = O.synth_images(b, h, w, seed=b + h)
    f = pruned(x.to(DEV))
    ref = oracle_on_gpu(O.darknet_forward, pruned_sd, x)
    assert f.shape == (b, 125, h // 32, w // 32)
    e = rel_err(f, ref)
    assert e <= TOL_DARKNET, e


def test_pruned_tiny_non_square_vs_oracle(golden):
    sd = PO.tiny_pruned_state_dict(PO.keep_from_npz(golden, 'tiny_'))
    net = build_tiny(sd)
    x = O.synth_images(4, 96, 160, seed=4)
    e = rel_err(net(x.to(DEV)), oracle_on_gpu(O.tiny_forward, sd, x))
    assert e <= TOL_TINY, e


def test_pruned_darknet_uint8_equals_fp32(pruned):
    frames = torch.randint(0, 256, (3, 96, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(9)).to(DEV)
    f_u8 = pruned(frames)
    f_f32 = pruned((frames.float() / 255.0).permute(0, 3, 1, 2).contiguous())
    assert rel_err(f_u8, f_f32) <= 2e-3


def test_pruned_darknet_detect_pipeline_graph_equals_eager(pruned):
    import detect
    import model
    from b200.pipeline import DetectPipeline
    cfg = make_config()
    inference = model.Inference(cfg, pruned, O.anchors_yolo_voc()).eval()
    x = O.synth_images(4, 416, 416, seed=7).to(DEV)
    eager = DetectPipeline(inference, cfg, 4, 416, 416, slots=1, use_graph=False).prepare()
    graph = DetectPipeline(inference, cfg, 4, 416, 416, slots=1, use_graph=True).prepare()
    outs = []
    for pipe in (eager, graph):             # the two share the engine's activation plan: each result is copied before the next run
        pipe.x[0].copy_(x)
        torch.cuda.synchronize()
        out = pipe.run(0)
        pipe.wait_all()
        outs.append({k: v.clone() for k, v in out.items()})
        torch.cuda.synchronize()
    for k in ('feature', 'iou', 'yx_min', 'yx_max', 'n_keep', 'keep_box'):
        assert torch.equal(outs[0][k], outs[1][k]), k
    pred = model._inference(inference, x)
    assert torch.equal(pred['feature'], outs[0]['feature'])
    results = detect.postprocess_batch(cfg, pred)
    assert len(results) == 4


# ------------------------------------------------------------------------------------------------------------------------------------
# full-width launches stay as they are
# ------------------------------------------------------------------------------------------------------------------------------------
def record_convs(fn):
    """(x channels, weight shape, flags) of every ops.conv_bn_act call made by fn()."""
    from b200 import ops
    calls = []
    orig = ops.conv_bn_act

    def rec(x, w, *a, **kw):
        calls.append((x.shape[-1], tuple(w.shape), kw.get('flags', 0)))
        return orig(x, w, *a, **kw)
    ops.conv_bn_act = rec
    try:
        fn()
    finally:
        ops.conv_bn_act = orig
    return calls


def test_full_width_and_ratio_half_never_reach_the_tail_entry():
    """Full-width Darknet-19 (416 and 608, fp32 and uint8 input) and Tiny, and Darknet(ratio=0.5) whose 16-filter layers1.0 is padded to
    32: no launch goes to the channel-tail entry, and every full-width conv reads the unit's own weight on an input of the same width."""
    dnn = build_darknet(O.make_state_dict(0))
    for size in (416, 608):
        x = O.synth_images(2, size, size, seed=1).to(DEV)
        assert count_tail_launches(lambda: dnn(x)) == 0
        calls = record_convs(lambda: dnn(x))
        assert len(calls) >= 19
        for c, wshape, _ in calls:
            assert c % 32 == 0 and wshape[-1] == c, (c, wshape)
    u8 = torch.randint(0, 256, (2, 416, 416, 3), dtype=torch.uint8).to(DEV)
    assert count_tail_launches(lambda: dnn(u8)) == 0
    net = build_tiny(O.make_tiny_state_dict(0))
    assert count_tail_launches(lambda: net(O.synth_images(2, 416, 416, seed=1).to(DEV))) == 0
    half = build_darknet(O.make_state_dict(0, ratio=0.5), ratio=0.5)
    x = O.synth_images(2, 128, 128, seed=3)
    assert count_tail_launches(lambda: half(x.to(DEV))) == 0
    assert half.engine.padded_unit() == 'layers1.0'
    assert rel_err(half(x.to(DEV)), oracle_on_gpu(O.darknet_forward, O.make_state_dict(0, ratio=0.5), x)) <= TOL_DARKNET
