"""VGG plugin (model.vgg: vgg11 / 13 / 16 / 19 and their _bn forms, inference) and its 64-filter first-layer kernel.

CPU: the restatement in vgg_oracle.py against the executed reference (vgg.npz: heads, every pool, a pruned checkpoint); the state_dict keys
and shapes of all eight constructors; the initialisation; the input errors; the new C entry point in the header and the ctypes table.

GPU: the first-layer kernel element by element against fp64 on its own fp16-rounded operands (activated, activated + pooled), the pooled
form against the unpooled one followed by yb_maxpool2x2_f16, exact zeros in padded filters; the plugin against the golden and the oracle
(every constructor at 416 x 416 and 320 x 608, the worst image of a batch of 32, the pruned model); decode + NMS on its head inside
model.Inference; cache invalidation and CUDA-graph replay."""
import configparser
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgg_oracle as V
from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu
MEASURED = {}


def record(name, value):
    """Measured figures of this run -> $YB_PARITY_OUT/vgg_measured.json when that directory is given."""
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'vgg_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def bits(t):
    return t.detach().contiguous().view(torch.int16).cpu()


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    return config


def build(name, seed=0, pruned=None):
    """The plugin with the oracle's synthetic weights (a pruned one built from its checkpoint as ConfigChannels(config, state_dict))."""
    import model
    import model.vgg
    sd = V.make_state_dict(name, seed, pruned=pruned)
    net = getattr(model.vgg, name)(model.ConfigChannels(make_config(), sd if pruned else None), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net.eval(), sd


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'vgg.npz'))


HEADS = ('vgg11', 'vgg11_bn', 'vgg16', 'vgg19_bn')
SIZES = ((64, 64, 1), (96, 160, 2), (416, 416, 0))
POOLS = ('vgg16_bn', 96, 160, 2)
PRUNED = ('vgg11_bn', 96, 160, 5)


def sampled(golden, name, t):
    """(got, ref) restricted to the golden's stored elements of activation `name`."""
    idx, ref, _ = O.load_sampled(golden, name)
    got = t.detach().double().cpu().reshape(-1)
    return (got if idx is None else got[torch.from_numpy(idx)]), torch.from_numpy(np.asarray(ref)).double().reshape(-1)


def pool_indices(name):
    return [i for kind, i, _ in V.layers(name) if kind == 'pool']


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_restatement_vs_reference_golden(golden):
    with torch.no_grad():
        for name in HEADS:
            sd = V.make_state_dict(name)
            for h, w, seed in SIZES:
                f = V.vgg_forward(sd, O.synth_images(1, h, w, seed=seed), name)
                ref = torch.from_numpy(golden['feature_%s_%dx%d' % (name, h, w)])
                assert tuple(ref.shape) == (1, 125, h // 32, w // 32)
                assert ((f - ref).norm() / ref.norm()).item() < 1e-5, (name, h, w)
        name, h, w, seed = POOLS
        got = {}
        V.vgg_forward(V.make_state_dict(name), O.synth_images(1, h, w, seed=seed), name, collect=got)
        assert sorted(got) == pool_indices(name)
        for i in got:
            a, r = sampled(golden, 'pool_%d' % i, got[i])
            assert ((a - r).norm() / r.norm()).item() < 1e-5, i
        name, h, w, seed = PRUNED
        pruned = V.pruned_widths()
        f = V.vgg_forward(V.make_state_dict(name, 3, pruned=pruned), O.synth_images(1, h, w, seed=seed), name, pruned=pruned)
        ref = torch.from_numpy(golden['feature_pruned'])
        assert ((f - ref).norm() / ref.norm()).item() < 1e-5


def test_state_dict_keys_and_shapes(golden):
    import model
    import model.vgg
    for name in V.NAMES:
        net = getattr(model.vgg, name)(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
        sd = net.state_dict()
        assert list(sd.keys()) == list(golden['keys_' + name]), name
        assert [','.join(str(d) for d in v.shape) for v in sd.values()] == list(golden['shapes_' + name]), name
        assert list(sd.keys())[-2:] == ['conv.weight', 'conv.bias']
        bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        assert bool(bns) == name.endswith('_bn') and all(m.eps == 1e-5 and m.momentum == 0.1 for m in bns)
    net, _ = build(*PRUNED[:1], seed=3, pruned=V.pruned_widths())
    shapes = [','.join(str(d) for d in v.shape) for k, v in net.state_dict().items() if not k.endswith('num_batches_tracked')]
    assert shapes == list(golden['shapes_pruned'])


def test_batch_norm_follows_the_name_not_the_config():
    import model
    import model.vgg
    config = make_config()
    config.set('batch_norm', 'enable', '0')
    net = model.vgg.vgg11_bn(model.ConfigChannels(config), O.anchors_yolo_voc(), 20)
    assert any(isinstance(m, torch.nn.BatchNorm2d) for m in net.modules())
    config.set('batch_norm', 'enable', '1')
    net = model.vgg.vgg11(model.ConfigChannels(config), O.anchors_yolo_voc(), 20)
    assert not any(isinstance(m, torch.nn.BatchNorm2d) for m in net.modules())


def test_initialisation_follows_the_reference():
    """torchvision 0.2's VGG._initialize_weights: conv weights N(0, 2 / (kh * kw * out_channels)), conv biases 0, BatchNorm weight 1, bias 0."""
    import model
    import model.vgg
    torch.manual_seed(0)
    net = model.vgg.vgg16_bn(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    for key in ('features.0', 'features.7', 'features.24', 'features.40'):
        w = net.get_submodule(key).weight.detach()
        assert abs(float(w.std()) / (2.0 / (9 * w.shape[0])) ** 0.5 - 1) < 0.03, key
        assert abs(float(w.mean())) < 0.1 * (2.0 / (9 * w.shape[0])) ** 0.5, key
        assert bool((net.get_submodule(key).bias == 0).all())
    w = net.conv.weight.detach()
    assert abs(float(w.std()) / (2.0 / w.shape[0]) ** 0.5 - 1) < 0.1 and bool((net.conv.bias == 0).all())
    bn = net.features[1]
    assert bool((bn.weight == 1).all() and (bn.bias == 0).all())


def test_input_errors():
    import model
    import model.vgg
    net, _ = build('vgg11')
    for shape in ((1, 3, 48, 64), (1, 3, 64, 80), (1, 4, 64, 64), (3, 64, 64)):
        with pytest.raises(ValueError):
            net(torch.zeros(*shape))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))               # CPU tensor: no CPU fallback
    net.train()
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))               # training: no CPU path either
    with pytest.raises(ValueError, match='features.0 has 80 filters'):
        model.vgg.vgg11(model.ConfigChannels(make_config(), V.make_state_dict('vgg11', pruned={'features.0.weight': 80})), O.anchors_yolo_voc(), 20)


def test_new_entry_point_is_declared():
    from b200 import lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'yolo2_b200.h')).read()
    assert 'yb_conv0_c64_bn_act_fwd' in lib.SIGNATURES and 'int yb_conv0_c64_bn_act_fwd(' in header


def test_selectable_from_config():
    import utils
    import model.vgg
    for name in V.NAMES:
        assert utils.parse_attr('model.vgg.' + name) is getattr(model.vgg, name)


# ------------------------------------------------------------------------------------------------
# GPU: first-layer kernel
# ------------------------------------------------------------------------------------------------
def first_layer_ref(x, w, scale, shift, slope, pool):
    """fp64 conv on the kernel's fp16-rounded operands, then the fp32 epilogue's rule."""
    z = F.conv2d(x.half().double(), w.half().double(), padding=1)
    t = z * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    t = torch.where(t > 0, t, t * slope)
    if pool:
        t = F.max_pool2d(t, 2, 2)
    return t.permute(0, 2, 3, 1)


@gpu
def test_first_layer_kernel_vs_fp64():
    from b200 import ops
    g = torch.Generator().manual_seed(11)
    rec = {}
    for b, h, w, slope in ((2, 32, 16, 0.0), (1, 64, 96, 0.0), (3, 96, 160, 0.1), (1, 416, 416, 0.0)):
        x = torch.rand(b, 3, h, w, generator=g) * 2 - 0.5
        wt = torch.randn(64, 3, 3, 3, generator=g) * 0.3
        scale = 0.5 + torch.rand(64, generator=g)
        shift = torch.randn(64, generator=g) * 0.2
        args = [t.to(DEV) for t in (x, wt, scale, shift)]
        for pool in (False, True):
            y = ops.conv0_c64_bn_act(*args, slope, pool=pool)
            ref = first_layer_ref(x, wt, scale, shift, slope, pool)
            assert tuple(y.shape) == tuple(ref.shape)
            err = (y.double().cpu() - ref).abs()
            # fp16 output rounding (2^-11 relative) plus fp32 accumulation
            assert bool((err <= ref.abs() * 2 ** -10 + 1e-4).all()), (b, h, w, pool, float(err.max()))
            rec['%dx%dx%d_pool%d' % (b, h, w, pool)] = float((err / (ref.abs() + 1e-3)).max())
    record('first_layer_rel', rec)


@gpu
def test_first_layer_pooled_equals_unpooled_then_pool():
    from b200 import ops
    g = torch.Generator().manual_seed(12)
    for b, h, w in ((2, 32, 32), (1, 96, 160), (4, 416, 416)):
        args = [t.to(DEV) for t in (torch.rand(b, 3, h, w, generator=g), torch.randn(64, 3, 3, 3, generator=g) * 0.3,
                                    0.5 + torch.rand(64, generator=g), torch.randn(64, generator=g) * 0.2)]
        full = ops.conv0_c64_bn_act(*args, 0.0)
        pooled = ops.conv0_c64_bn_act(*args, 0.0, pool=True)
        # equal values: fp16 rounding is monotonic, so the max of the rounded values is the rounded max
        assert torch.equal(pooled, ops.maxpool2x2(full)), (b, h, w)


@gpu
def test_first_layer_padded_filters_are_exact_zeros():
    from b200 import ops
    g = torch.Generator().manual_seed(13)
    x = torch.rand(2, 3, 64, 96, generator=g).to(DEV)
    wt = torch.zeros(64, 3, 3, 3)
    wt[:48] = torch.randn(48, 3, 3, 3, generator=g)
    scale, shift = torch.ones(64), torch.zeros(64)
    scale[:48], shift[:48] = 0.5 + torch.rand(48, generator=g), torch.randn(48, generator=g)
    for pool in (False, True):
        y = ops.conv0_c64_bn_act(x, wt.to(DEV), scale.to(DEV), shift.to(DEV), 0.0, pool=pool)
        assert bool((bits(y)[..., 48:] == 0).all()) and bool((y[..., :48] != 0).any())


@gpu
def test_first_layer_errors():
    from b200 import ops
    one = torch.ones(64, device=DEV)
    with pytest.raises(RuntimeError):
        ops.conv0_c64_bn_act(torch.zeros(1, 3, 48, 32, device=DEV), torch.zeros(64, 3, 3, 3, device=DEV), one, one, 0.0)   # H % 32
    with pytest.raises(RuntimeError):
        ops.conv0_c64_bn_act(torch.zeros(1, 3, 32, 40, device=DEV), torch.zeros(64, 3, 3, 3, device=DEV), one, one, 0.0)   # W % 16
    with pytest.raises(ValueError):
        ops.conv0_c64_bn_act(torch.zeros(1, 3, 32, 32, device=DEV), torch.zeros(32, 3, 3, 3, device=DEV), one, one, 0.0)
    with pytest.raises(RuntimeError):
        ops.conv0_c64_bn_act(torch.zeros(1, 3, 32, 32), torch.zeros(64, 3, 3, 3), one.cpu(), one.cpu(), 0.0)


# ------------------------------------------------------------------------------------------------
# GPU: plugin
# ------------------------------------------------------------------------------------------------
# measured on an H100 80GB HBM3 (700 W): heads and pools vs the golden <= 1.75e-3 (vgg19_bn at 416 x 416), every constructor vs the oracle
# <= 2.15e-3 (one image) and 2.46e-3 (the worst image of a batch of 32, vgg19_bn), the pruned vgg11_bn 1.85e-3; the bound is twice the worst
TOL_E2E = 5e-3


@gpu
def test_plugin_vs_reference_golden(golden):
    rec = {}
    with torch.no_grad():
        for name in HEADS:
            net = build(name)[0].to(DEV)
            for h, w, seed in SIZES:
                f = net(O.synth_images(1, h, w, seed=seed).to(DEV))
                assert tuple(f.shape) == (1, 125, h // 32, w // 32)
                rec['%s_%dx%d' % (name, h, w)] = rel_err(f, torch.from_numpy(golden['feature_%s_%dx%d' % (name, h, w)]))
        name, h, w, seed = POOLS
        net = build(name)[0].to(DEV)
        acts = {}
        net.run(O.synth_images(1, h, w, seed=seed).to(DEV), collect=acts)
        assert sorted(acts) == pool_indices(name)
        for i in acts:
            got, ref = sampled(golden, 'pool_%d' % i, acts[i].permute(0, 3, 1, 2))
            rec['pool_%d' % i] = rel_err(got, ref)
        name, h, w, seed = PRUNED
        net = build(name, 3, pruned=V.pruned_widths())[0].to(DEV)
        rec['pruned'] = rel_err(net(O.synth_images(1, h, w, seed=seed).to(DEV)), torch.from_numpy(golden['feature_pruned']))
    record('golden', rec)
    assert all(v <= TOL_E2E for v in rec.values()), rec


def _oracle_on_gpu(sd, x, name, pruned=None):
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return V.vgg_forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV), name, pruned=pruned)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@gpu
@pytest.mark.parametrize('name', V.NAMES)
def test_every_constructor_vs_oracle(name):
    """416 x 416 and 320 x 608 (one image each) and the worst image of a batch of 32 at 416 x 416."""
    net, sd = build(name, seed=1)
    net = net.to(DEV)
    rec = {}
    for b, h, w, seed in ((1, 416, 416, 3), (1, 320, 608, 4), (32, 416, 416, 5)):
        x = O.synth_images(b, h, w, seed=seed)
        with torch.no_grad():
            y = net(x.to(DEV))
        assert tuple(y.shape) == (b, 125, h // 32, w // 32)
        ref = _oracle_on_gpu(sd, x, name)
        rec['%dx%dx%d' % (b, h, w)] = max(rel_err(y[i], ref[i]) for i in range(b))
    record('oracle_' + name, rec)
    assert all(v <= TOL_E2E for v in rec.values()), rec


@gpu
def test_pruned_model_vs_oracle_and_padded_zeros():
    pruned = V.pruned_widths()
    net, sd = build('vgg11_bn', seed=2, pruned=pruned)
    net = net.to(DEV)
    x = O.synth_images(4, 320, 608, seed=6)
    acts = {}
    with torch.no_grad():
        y = net.run(x.to(DEV), collect=acts)
    ref = _oracle_on_gpu(sd, x, 'vgg11_bn', pruned)
    err = max(rel_err(y[i], ref[i]) for i in range(4))
    record('oracle_pruned', err)
    assert err <= TOL_E2E
    # every pooled buffer is zero, bit for bit, past its producer's real filters (features.0: 48 of 64)
    for u in net.units:
        if u.pool:
            a = acts[u.pool_index]
            c = u.conv.out_channels
            assert a.shape[-1] > c and bool((bits(a)[..., c:] == 0).all()), u.pool_index


@gpu
def test_inference_reload_graph_and_postprocess():
    import detect
    import model
    net, _ = build('vgg16')
    net = net.to(DEV)
    cfg = make_config()
    anchors = O.anchors_yolo_voc()
    inference = model.Inference(cfg, net, anchors).eval()
    pred = model._inference(inference, O.synth_images(2, 416, 416, seed=2).to(DEV))
    assert tuple(pred['feature'].shape) == (2, 125, 13, 13)
    results = detect.postprocess_batch(cfg, pred)
    torch.cuda.synchronize()
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
    x = O.synth_images(2, 96, 160, seed=3).to(DEV)
    with torch.no_grad():
        y0 = net(x)
        net.load_state_dict(V.make_state_dict('vgg16', 1), strict=False)
        y1 = net(x)
        y_fresh = build('vgg16', 1)[0].to(DEV)(x)
    assert torch.equal(y1, y_fresh) and not torch.equal(y0, y1)
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
    static_x.copy_(O.synth_images(2, 96, 160, seed=6).to(DEV))
    graph.replay()
    with torch.no_grad():
        eager = net(static_x)
    torch.cuda.synchronize()
    assert torch.equal(static_y, eager)
