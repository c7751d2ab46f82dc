"""Inception-v4 plugin (model.inception4) and the count-exclusive average pool it adds.

CPU: the restatement in inception4_oracle.py against the executed reference (inception4.npz) for every variant (BatchNorm on / off, ratio
0.5, a pruned checkpoint); the state_dict keys and shapes; the initialisation; the input errors; the new C entry point in the header and the
ctypes table; and the padded channel layout, without a GPU: the oracle's activations placed in the plugin's layouts and run through the
plugin's scattered fp32 weights with F.conv2d give the oracle's outputs at the mapped channels and zeros everywhere else.

GPU: the pool bit for bit against an fp32 restatement of its rule; the plugin against the golden and the oracle (heads, blocks, each block
fed the oracle's input, the worst image of a batch of 32); CUDA-graph replay, cache invalidation, decode + NMS on its head; exact zeros in the
padded channels."""
import configparser
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception4_oracle as I
from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu
MEASURED = {}


def record(name, value):
    """Measured figures of this run -> $YB_PARITY_OUT/inception4_measured.json when that directory is given."""
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'inception4_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_config(bn=True, **extra):
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': str(int(bn))}, 'model': {'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    config.read_dict(extra)
    return config


# variant -> (BatchNorm, ratio, pruned widths, state_dict seed); the golden's heads at 107 x 139 on image seed VARIANT_SEED
VARIANTS = {'nobn': (False, 1, None, 1), 'ratio05': (True, 0.5, None, 2), 'pruned': (True, 1, I.pruned_widths(), 3)}
VARIANT_SEED = 7


def variant_sd(tag):
    bn, ratio, pruned, seed = VARIANTS[tag]
    return I.make_state_dict(seed, ratio=ratio, bn=bn, pruned=pruned)


def build(seed=0, tag=None):
    """The plugin with the oracle's synthetic weights: ratio 1 with BatchNorm, or one of VARIANTS (the pruned one built from its checkpoint as
    ConfigChannels(config, state_dict))."""
    import model
    import model.inception4
    bn, ratio, pruned, _ = VARIANTS[tag] if tag else (True, 1, None, seed)
    sd = variant_sd(tag) if tag else I.make_state_dict(seed)
    cc = model.ConfigChannels(make_config(bn), sd if pruned else None)
    net = model.inception4.Inception4(cc, O.anchors_yolo_voc(), 20, ratio=ratio)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net.eval(), sd


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'inception4.npz'))


SIZES = ((75, 75, 1), (107, 139, 2), (416, 416, 0), (320, 608, 3))
GRIDS = {(75, 75): (1, 1), (107, 139): (2, 3), (416, 416): (11, 11), (320, 608): (8, 17)}
BLOCKS = (3, 4, 5, 6, 10, 11, 18, 21)          # one block of each kind, as stored in the golden


def sampled(golden, name, t):
    """(got, ref) restricted to the golden's stored elements of activation `name`."""
    idx, ref, _ = O.load_sampled(golden, name)
    got = t.detach().double().cpu().reshape(-1)
    return (got if idx is None else got[torch.from_numpy(idx)]), torch.from_numpy(np.asarray(ref)).double().reshape(-1)


def key_of(net):
    """unit module -> its key prefix in the state_dict."""
    return {m: n for n, m in net.named_modules()}


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_restatement_vs_reference_golden(golden):
    sd = I.make_state_dict(0)
    for h, w, seed in SIZES:
        got = {}
        with torch.no_grad():
            f = I.inception4_forward(sd, O.synth_images(1, h, w, seed=seed), collect=got)
        ref = torch.from_numpy(golden['feature_%dx%d' % (h, w)])
        assert tuple(ref.shape[-2:]) == GRIDS[(h, w)]
        assert ((f - ref).norm() / ref.norm()).item() < 1e-5, (h, w)
        if (h, w) == (107, 139):
            for k in BLOCKS:
                a, r = sampled(golden, 'act_%d' % k, got[k])
                assert ((a - r).norm() / r.norm()).item() < 1e-5, k
    x = O.synth_images(1, 107, 139, seed=VARIANT_SEED)
    for tag in VARIANTS:
        with torch.no_grad():
            f = I.inception4_forward(variant_sd(tag), x)
        ref = torch.from_numpy(golden['feature_' + tag])
        assert ((f - ref).norm() / ref.norm()).item() < 1e-5, tag


def test_state_dict_keys_and_shapes(golden):
    for bn, tag in ((True, ''), (False, '_nobn')):
        import model
        import model.inception4
        net = model.inception4.Inception4(model.ConfigChannels(make_config(bn)), O.anchors_yolo_voc(), 20)
        sd = net.state_dict()
        assert list(sd.keys()) == list(golden['keys' + tag])
        assert [','.join(str(d) for d in v.shape) for v in sd.values()] == list(golden['shapes' + tag])
        assert list(sd.keys())[-2:] == ['features.22.weight', 'features.22.bias']
        assert ('features.6.branch3.1.conv.weight' in sd) and (('features.19.branch2_3a.bn.running_var' in sd) == bn)
        assert ('features.6.branch0.conv.bias' in sd) == (not bn)
    for tag in VARIANTS:
        net, _ = build(tag=tag)
        shapes = [','.join(str(d) for d in v.shape) for k, v in net.state_dict().items() if not k.endswith('num_batches_tracked')]
        assert shapes == list(golden['shapes_' + tag]), tag
    bns = [m for m in build()[0].modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert bns and all(m.eps == 1e-3 for m in bns)


def test_initialisation_follows_the_reference():
    """kaiming_normal (fan_in, gain sqrt 2) on every conv, BatchNorm weight 1 and bias 0, trainable as `[batch_norm] gamma / beta`."""
    import model
    import model.inception4
    torch.manual_seed(0)
    net = model.inception4.Inception4(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    for key in ('features.21.branch2_2', 'features.11.branch2.4', 'features.4.branch1.1'):
        w = net.get_submodule(key).conv.weight.detach()
        fan_in = w[0].numel()
        assert abs(float(w.std()) / (2.0 / fan_in) ** 0.5 - 1) < 0.03, key
    w = net.features[22].weight.detach()
    assert abs(float(w.std()) / (2.0 / w.shape[1]) ** 0.5 - 1) < 0.05
    bn = net.features[6].branch0.bn
    assert bool((bn.weight == 1).all() and (bn.bias == 0).all()) and bn.weight.requires_grad and bn.bias.requires_grad
    frozen = model.inception4.Inception4(model.ConfigChannels(make_config(batch_norm={'gamma': '0', 'beta': '0'})), O.anchors_yolo_voc(), 20)
    assert all(not (m.weight.requires_grad or m.bias.requires_grad) for m in frozen.modules() if isinstance(m, torch.nn.BatchNorm2d))
    assert 'pretrainedmodels' not in sys.modules
    assert net.scope('features.19.branch2_3a.conv.weight') == 'features.19.branch2_3a'


def test_input_errors():
    import model
    import model.inception4
    net, _ = build()
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 74, 128))              # Reduction_B's output would be empty
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 128, 74))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 4, 75, 75))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 75, 75))               # CPU tensor: no CPU fallback
    net.train()
    with pytest.raises(NotImplementedError):
        net(torch.zeros(1, 3, 75, 75))
    sd = {'features.0.conv.weight': torch.zeros(40, 3, 3, 3), 'features.1.conv.weight': torch.zeros(32, 40, 3, 3),
          'features.2.conv.weight': torch.zeros(64, 32, 3, 3)}
    with pytest.raises(ValueError, match='features.0 has 40 filters'):
        model.inception4.Inception4(model.ConfigChannels(make_config(), sd), O.anchors_yolo_voc(), 20)


def test_new_entry_point_is_declared():
    from b200 import lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'yolo2_b200.h')).read()
    assert 'yb_avgpool3x3_s1_excl_f16' in lib.SIGNATURES and 'int yb_avgpool3x3_s1_excl_f16(' in header


def test_selectable_from_config():
    import utils
    import model.inception4
    assert utils.parse_attr('model.inception4.Inception4') is model.inception4.Inception4


def place(t, lay):
    """fp32 NCHW t (the reference's channels) -> a buffer of lay.width channels with channel j at lay.pos[j], zero elsewhere."""
    buf = torch.zeros(t.shape[0], lay.width, *t.shape[2:], dtype=t.dtype)
    buf[:, lay.pos] = t
    return buf


def sim_unit(net, sd, keys, unit, buf):
    """One conv unit of the plugin in fp32: the scattered weight on a padded input buffer, then the reference's BatchNorm + ReLU (or bias + ReLU)
    on its real channels.  Asserts that the padded filters give exact zeros."""
    key = keys[unit]
    y = F.conv2d(buf, net.scattered(unit), None, unit.conv.stride, unit.conv.padding)
    cout = unit.conv.out_channels
    assert bool((y[:, cout:] == 0).all()), key
    real = y[:, :cout]
    if unit.bn is None:
        real = real + sd[key + '.conv.bias'].view(1, -1, 1, 1)
    else:
        real = F.batch_norm(real, sd[key + '.bn.running_mean'], sd[key + '.bn.running_var'], sd[key + '.bn.weight'], sd[key + '.bn.bias'], False,
                            0.0, I.BN_EPS)
    return torch.cat([F.relu(real), y[:, cout:]], 1)


def close(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item() < 1e-5


@pytest.mark.parametrize('tag', ['ratio05', 'pruned'])
def test_padded_layout_on_the_cpu(tag):
    """Every conv unit fed the oracle's own input in its padded input layout, and every block assembled from its segments as the plugin writes
    them (convs at their channel offsets, max-pools of the padded input), in fp32 on the CPU: equal to the oracle at the mapped channels, zero
    at every other channel; the head likewise."""
    net, sd = build(tag=tag)
    keys = key_of(net)
    units, acts = {}, {}
    x = O.synth_images(1, 107, 139, seed=VARIANT_SEED)
    with torch.no_grad():
        I.inception4_forward(sd, x, collect=acts, units=units)
        for unit, lay in net.layouts.items():
            key = keys[unit]
            if lay is None:                          # the stem conv: 3 input channels, its own kernel
                continue
            t_in, t_out = units[key]
            if key == I.HEAD:
                y = F.conv2d(place(t_in, lay), net.scattered_head(), sd[I.HEAD + '.bias'])
                assert close(y, t_out), key
                continue
            y = sim_unit(net, sd, keys, unit, place(t_in, lay))
            cout = unit.conv.out_channels
            assert close(y[:, :cout], t_out) and y.shape[1] == (cout + 31) // 32 * 32, key
        prev = acts['stem']
        for i, (m, segs, lay) in enumerate(net.blocks):
            lin = net.layouts[next(us[0] for kind, us, _ in segs if kind != 'max')]
            xin = place(prev, lin)
            ref = acts[i + 3]
            out = torch.full((1, lay.width) + ref.shape[2:], float('nan'))
            memo = {}
            for kind, us, off in segs:
                if kind == 'max':
                    y = F.max_pool2d(xin, 3, 2)
                else:
                    y = I.avg_pool(xin) if kind == 'avg' else xin
                    for j, u in enumerate(us):
                        if us[:j + 1] not in memo:
                            memo[us[:j + 1]] = sim_unit(net, sd, keys, u, y)
                        y = memo[us[:j + 1]]
                out[:, off:off + y.shape[1]] = y
            assert not bool(out.isnan().any()), 'features.%d: channels no segment writes' % (i + 3)
            mapped = torch.zeros(lay.width, dtype=torch.bool)
            mapped[lay.pos] = True
            assert close(out[:, lay.pos], ref), 'features.%d' % (i + 3)
            assert bool((out[:, ~mapped] == 0).all()), 'features.%d' % (i + 3)
            prev = ref
    assert any(lay is not None and lay.width != lay.pos.numel() for lay in net.layouts.values())     # the layouts are not the identity


def test_layout_is_the_identity_at_ratio_1():
    net, _ = build()
    for lay in list(net.layouts.values()) + [b[2] for b in net.blocks]:
        assert lay is None or (lay.width == lay.pos.numel() and torch.equal(lay.pos, torch.arange(lay.width)))


# ------------------------------------------------------------------------------------------------
# GPU: the count-exclusive average pool
# ------------------------------------------------------------------------------------------------
def pool_rule(x16, exclude):
    """fp32 restatement of the pools' rule on fp16 NHWC x: the in-range taps of the 3 x 3 window added in row-major order starting from 0,
    divided once by the count (or by 9), rounded to fp16."""
    x = x16.float().permute(0, 3, 1, 2)
    b, c, h, w = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    ones = F.pad(torch.ones(1, 1, h, w), (1, 1, 1, 1))
    acc = torch.zeros_like(x)
    n = torch.zeros(1, 1, h, w)
    for r in range(3):
        for s in range(3):
            inside = ones[:, :, r:r + h, s:s + w]
            acc = torch.where(inside > 0, acc + xp[:, :, r:r + h, s:s + w], acc)
            n = n + inside
    return (acc / (n if exclude else torch.full_like(n, 9.0))).half().permute(0, 2, 3, 1).contiguous()


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int16)


@gpu
def test_count_exclusive_pool_bit_exact():
    from b200 import ops
    g = torch.Generator().manual_seed(41)
    for b, h, w, c in ((2, 7, 9, 16), (2, 8, 6, 24), (1, 1, 9, 8), (1, 9, 1, 8), (3, 1, 1, 8), (1, 2, 2, 32), (2, 49, 49, 384), (2, 24, 24, 1024),
                       (2, 11, 11, 1536)):
        x = (torch.randn(b, h, w, c, generator=g) * 3).half()
        y = ops.avgpool3x3_s1_excl(x.to(DEV))
        assert torch.equal(bits(y), bits(pool_rule(x, True))), (b, h, w, c)
        y9 = ops.avgpool3x3_s1(x.to(DEV))
        assert torch.equal(bits(y9), bits(pool_rule(x, False))), (b, h, w, c)          # the v3 pool keeps its rule
        if h > 2 and w > 2:
            assert torch.equal(bits(y[:, 1:-1, 1:-1]), bits(y9[:, 1:-1, 1:-1])), (b, h, w, c)
    # a border that tells the two divisors apart: a constant image averages to itself only when the count excludes the padding
    x = torch.full((1, 5, 6, 8), 2.0, dtype=torch.float16, device=DEV)
    assert bool((ops.avgpool3x3_s1_excl(x) == 2.0).all()) and float(ops.avgpool3x3_s1(x)[0, 0, 0, 0]) == float(torch.tensor(8.0 / 9).half())


# ------------------------------------------------------------------------------------------------
# GPU: plugin
# ------------------------------------------------------------------------------------------------
# measured on an H100 80GB HBM3 (700 W): heads and activations vs the golden <= 2.1e-3 (head at 416 x 416), the worst image of a batch of
# 32 2.4e-3 (416 x 416), every block fed the oracle's input <= 9.9e-4; the bounds are twice the worst of each
TOL_E2E = 4e-3
TOL_BLOCK = 1.9e-3


@gpu
def test_plugin_vs_reference_golden(golden):
    net, _ = build()
    net = net.to(DEV)
    rec = {}
    with torch.no_grad():
        for h, w, seed in SIZES:
            f = net(O.synth_images(1, h, w, seed=seed).to(DEV))
            assert tuple(f.shape) == (1, 125) + GRIDS[(h, w)]
            rec['feature_%dx%d' % (h, w)] = rel_err(f, torch.from_numpy(golden['feature_%dx%d' % (h, w)]))
        acts = {}
        net.run(O.synth_images(1, 107, 139, seed=2).to(DEV), collect=acts)
        for k in BLOCKS:
            got, ref = sampled(golden, 'act_%d' % k, acts[k].permute(0, 3, 1, 2))
            rec['act_%d' % k] = rel_err(got, ref)
        x = O.synth_images(1, 107, 139, seed=VARIANT_SEED).to(DEV)
        for tag in VARIANTS:
            net_v = build(tag=tag)[0].to(DEV)
            rec['feature_' + tag] = rel_err(net_v(x), torch.from_numpy(golden['feature_' + tag]))
    record('golden', rec)
    assert all(v <= TOL_E2E for v in rec.values()), rec


@gpu
@pytest.mark.parametrize('tag', [None, 'pruned'])
def test_each_block_fed_oracle_input(tag):
    """Every block at 107 x 139, fed the oracle's own (fp16-rounded) input in its padded layout: its output at the mapped channels vs the
    oracle's block."""
    net, sd = build(tag=tag)
    net = net.to(DEV)
    acts = {}
    with torch.no_grad():
        I.inception4_forward(sd, O.synth_images(1, 107, 139, seed=2), collect=acts)
    rec = {}
    with torch.no_grad():
        prev = acts['stem']
        for i, (m, segs, lay) in enumerate(net.blocks):
            lin = net.layouts[next(us[0] for kind, us, _ in segs if kind != 'max')]
            x = place(prev.half().float(), lin).permute(0, 2, 3, 1).contiguous().half().to(DEV)
            ref = I.block_forward(sd, prev.half().float(), i + 3)
            got = net.block(i + 3, x).permute(0, 3, 1, 2).float().cpu()
            rec['features.%d' % (i + 3)] = rel_err(got[:, lay.pos], ref)
            prev = acts[i + 3]
    record('blocks_%s' % (tag or 'ratio1'), rec)
    assert all(v <= TOL_BLOCK for v in rec.values()), rec


def _oracle_on_gpu(sd, x):
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return I.inception4_forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@gpu
def test_batch32_vs_oracle():
    net, sd = build()
    net = net.to(DEV)
    rec = {}
    for h, w, seed in ((416, 416, 4), (320, 608, 5)):
        x = O.synth_images(32, h, w, seed=seed)
        with torch.no_grad():
            y = net(x.to(DEV))
        assert tuple(y.shape) == (32, 125) + GRIDS[(h, w)]
        ref = _oracle_on_gpu(sd, x)
        per = [rel_err(y[i], ref[i]) for i in range(32)]
        rec['batch32_%dx%d' % (h, w)] = [max(per), int(np.argmax(per))]
    record('batch32_worst_image', rec)
    assert all(v[0] <= TOL_E2E for v in rec.values()), rec


@gpu
def test_padded_channels_hold_exact_zeros():
    """Pruned widths: every block buffer is zero, bit for bit, at every channel its layout does not map (padded filters, padded inputs carried
    through the max-pools)."""
    net, _ = build(tag='pruned')
    net = net.to(DEV)
    acts = {}
    with torch.no_grad():
        net.run(O.synth_images(2, 107, 139, seed=8).to(DEV), collect=acts)
    torch.cuda.synchronize()
    padded = 0
    for i, (m, segs, lay) in enumerate(net.blocks):
        mapped = torch.zeros(lay.width, dtype=torch.bool)
        mapped[lay.pos] = True
        a = bits(acts[i + 3])
        assert bool((a[..., ~mapped] == 0).all()), 'features.%d' % (i + 3)
        padded += int((~mapped).sum())
    assert padded > 0
    f = net.features
    assert bool((bits(acts['stem'])[..., f[2].conv.out_channels:] == 0).all())       # features.2: 61 filters of 64
    from b200 import ops
    with torch.no_grad():
        a0 = ops.stem3x3_s2(O.synth_images(2, 107, 139, seed=8).to(DEV), *net._operands(f[0]), pad=0)
    assert f[0].conv.out_channels == 29 and a0.shape[-1] == 32 and bool((bits(a0)[..., 29:] == 0).all())   # features.0: 3 zero filters


@gpu
def test_inference_reload_graph_and_postprocess():
    import detect
    import model
    net, _ = build()
    net = net.to(DEV)
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    inference = model.Inference(cfg, net, anchors).eval()
    pred = model._inference(inference, O.synth_images(2, 416, 416, seed=2).to(DEV))
    assert tuple(pred['feature'].shape) == (2, 125, 11, 11)
    results = detect.postprocess_batch(cfg, pred)
    torch.cuda.synchronize()
    # decode + NMS on the GPU's own 11 x 11 feature match the oracle's
    dec = O.decode(pred['feature'].cpu(), anchors)
    for k in ('iou', 'yx_min', 'yx_max'):
        assert rel_err(pred[k], dec[k]) <= 1e-5, k
    for bi, res in enumerate(results):
        exp = O.postprocess(pred['iou'][bi].reshape(-1).cpu(), pred['yx_min'][bi].reshape(-1, 2).cpu(), pred['yx_max'][bi].reshape(-1, 2).cpu(),
                            pred['prob'][bi].reshape(-1, 20).cpu(), True, 0.3, 0.005, 0.45)
        assert (res is None) == (exp is None)
        if res is not None:
            assert res[3].cpu().tolist() == exp[3].tolist()
    # cached operands follow load_state_dict
    x = O.synth_images(2, 107, 139, seed=3).to(DEV)
    with torch.no_grad():
        y0 = net(x)
        net.load_state_dict(I.make_state_dict(1), strict=False)
        y1 = net(x)
        y_fresh = build(1)[0].to(DEV)(x)
    assert torch.equal(y1, y_fresh) and not torch.equal(y0, y1)
    # train() / eval() drops the cache
    assert net._cache
    net.train()
    assert not net._cache
    net.eval()
    with torch.no_grad():
        assert torch.equal(net(x), y1)
    # CUDA-graph replay is bit-identical to eager
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(s):
        net(static_x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        static_y = net(static_x)
    static_x.copy_(O.synth_images(2, 107, 139, seed=6).to(DEV))
    graph.replay()
    with torch.no_grad():
        eager = net(static_x)
    torch.cuda.synchronize()
    assert torch.equal(static_y, eager)
