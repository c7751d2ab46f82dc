"""DenseNet plugin (model.densenet): the restatement in densenet_oracle.py against the executed reference (densenet.npz), the module tree and
state_dict keys, the torchvision-0.2 key remap and the input errors on CPU; on the GPU the pre-activation 1x1 conv (bit-identity with the plain
conv on a materialised operand, accuracy against fp64), the two pool kernels (bit-exact) and the plugin against the reference."""
import configparser
import json
import os

import numpy as np
import pytest
import torch

import densenet_oracle as D
from oracle import yolo2_oracle as O

DEV = 'cuda'
NAMES = ('densenet121', 'densenet169', 'densenet201', 'densenet161')


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    return config


def build(name, seed=0):
    import model
    import model.densenet
    net = getattr(model.densenet, name)(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(D.make_densenet_state_dict(name, seed), strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net.eval()


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'densenet.npz'))


MEASURED = {}


def record(name, value):
    """Measured figures of this run -> $YB_PARITY_OUT/densenet_measured.json when that directory is given."""
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'densenet_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_restatement_vs_reference_golden(golden):
    for name, size, seed in (('densenet121', 64, 10), ('densenet121', 416, 0), ('densenet169', 64, 10), ('densenet201', 64, 10)):
        sd = D.make_densenet_state_dict(name, 0)
        got = {}
        with torch.no_grad():
            f = D.densenet_forward(sd, O.synth_images(1, size, size, seed=seed), name, collect=got)
        ref = torch.from_numpy(golden['%s_feature%d' % (name, size)])
        assert ((f - ref).norm() / ref.norm()).item() < 1e-5, (name, size)
        if (name, size) == ('densenet121', 64):
            for k in ('denseblock1', 'transition1', 'denseblock2', 'transition2', 'denseblock3', 'transition3', 'denseblock4'):
                r = torch.from_numpy(golden['densenet121_act_' + k])
                assert ((got[k] - r).norm() / r.norm()).item() < 1e-5, k


def test_state_dict_keys_and_shapes(golden):
    for name in NAMES:
        net = build(name) if name != 'densenet161' else None
        if net is None:
            import model
            import model.densenet
            net = model.densenet.densenet161(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
        sd = net.state_dict()
        assert list(sd.keys()) == list(golden['%s_keys' % name]), name
        assert [','.join(str(d) for d in v.shape) for v in sd.values()] == list(golden['%s_shapes' % name]), name


def test_legacy_key_remap():
    """torchvision-0.2 checkpoints (the reference's Saver files, ImageNet weights of that era) name dense-layer parameters `norm.1`, `conv.2`."""
    import re
    sd = D.make_densenet_state_dict('densenet121', 3)
    old = {re.sub(r'(denselayer\d+\.(?:norm|conv))([12])\.', r'\1.\2.', k): v for k, v in sd.items()}
    assert any('.norm.1.' in k for k in old) and not any('norm1' in k for k in old)
    net = build('densenet121', 0)
    res = net.load_state_dict(old, strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    got = net.state_dict()
    for k, v in sd.items():
        assert torch.equal(got[k], v), k


def test_input_errors():
    net = build('densenet121')
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 48, 64))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))                    # CPU tensor: no CPU fallback
    net.train()
    with pytest.raises(NotImplementedError):
        net(torch.zeros(1, 3, 64, 64))
    import model
    import model.densenet
    n161 = model.densenet.densenet161(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20).eval()
    with pytest.raises(NotImplementedError, match='96-channel stem.*growth rate 48'):
        n161(torch.zeros(1, 3, 64, 64))
    # the reference's constructors forward **kwargs such as drop_rate to DenseNet.__init__ (dropout acts in training only)
    assert model.densenet.densenet121(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20, drop_rate=0).drop_rate == 0


# ------------------------------------------------------------------------------------------------
# GPU: kernels
# ------------------------------------------------------------------------------------------------
def _f16_affine(c, g):
    """fp16-representable scale / shift: fmaf and a separate multiply and add agree, and the fp64 host arithmetic is exact."""
    return (torch.rand(c, generator=g) + 0.5).half().float(), (torch.randn(c, generator=g) * 0.5).half().float()


@pytest.mark.gpu
def test_preact_conv_bit_identical_to_materialised_k1():
    from b200 import ops
    g = torch.Generator().manual_seed(7)
    for cin in (64, 96, 512, 1024, 1920):
        b, h, w = 3, 13, 13
        x_ld = cin + 32
        x = (torch.randn(b, h, w, x_ld, generator=g)).half()
        ps, pb = _f16_affine(cin, g)
        wt = torch.randn(128, cin, 1, 1, generator=g) * (2.0 / cin) ** 0.5
        w125 = torch.randn(125, cin, 1, 1, generator=g) * (1.0 / cin) ** 0.5
        scale, shift = torch.rand(128, generator=g) + 0.5, torch.randn(128, generator=g) * 0.1
        wp, wp125 = ops.pack_weight_f16(wt.to(DEV)), ops.pack_weight_f16(w125.to(DEV))
        xd = x.to(DEV)
        for relu in (0, 1):
            a = x[..., :cin].double() * ps.double() + pb.double()
            if relu:
                a = a.clamp_min(0)
            a = a.float().half().to(DEV).contiguous()
            for bn, mt in ((64, 1), (128, 1), (64, 2)):
                flags = ops.conv_force_bn(bn) | ops.conv_force_mt(mt) | ops.CONV_NO_STREAMK
                # fp16 NHWC into channels [64, 192) of a 256-wide buffer, neighbours held by a sentinel
                y = torch.full((b, h, w, 256), 7.0, dtype=torch.float16, device=DEV)
                ops.conv1x1_preact(xd, wp, ps.to(DEV), pb.to(DEV), relu, scale.to(DEV), shift.to(DEV), 0.1, out=y, y_ch_off=64, cin=cin, flags=flags)
                yr = torch.full_like(y, 7.0)
                ops.conv_bn_act(a, wp, scale.to(DEV), shift.to(DEV), 0.1, out=yr, y_ch_off=64, flags=flags)
                assert torch.equal(y, yr), (cin, relu, bn, mt)
                assert bool((y[..., :64] == 7).all() and (y[..., 192:] == 7).all())
                # fp32 NCHW head form, Cout = 125
                one, bias = torch.ones(125, device=DEV), (torch.randn(125, generator=g) * 0.1).to(DEV)
                yf = ops.conv1x1_preact(xd, wp125, ps.to(DEV), pb.to(DEV), relu, one, bias, 1.0, out_mode=ops.OUT_F32_NCHW, cin=cin, flags=flags)
                yfr = ops.conv_bn_act(a, wp125, one, bias, 1.0, out_mode=ops.OUT_F32_NCHW, flags=flags)
                assert torch.equal(yf, yfr), (cin, relu, bn, mt, 'f32')


# shapes whose tiles x K-blocks give every SM >= 4 K-blocks, so forced stream-K is taken (the selection otherwise keeps whole tiles):
# BK = 32 (Cin 96, 3 K-blocks per tile, segments cross tile boundaries) and BK = 64 (Cin 1024 / 1920, 16 / 30 K-blocks)
STREAMK_SHAPES = ((96, 32, 26), (1024, 8, 26), (1920, 4, 26))


def _streamk_flags(ops, b, hw, cin, out_mode=0):
    flags = ops.conv_force_bn(128) | ops.conv_force_mt(1) | ops.CONV_FORCE_STREAMK
    ch = ops.conv_choice(b, hw, hw, cin, 128 if out_mode == 0 else 125, 1, out_mode=out_mode, flags=flags, workspace=True)
    assert ch['streamk'] and ch['kernel'] == 'conv_igemm_kernel', ch
    return flags


@pytest.mark.gpu
def test_preact_conv_accuracy_vs_fp64():
    from b200 import ops
    g = torch.Generator().manual_seed(8)
    ws = ops.conv_workspace()
    worst = {}
    for cin, b, hw in ((96, 2, 26), (512, 4, 26)) + STREAMK_SHAPES:
        x = torch.randn(b, hw, hw, cin, generator=g).half()
        ps, pb = torch.rand(cin, generator=g) * 1.5 + 0.1, torch.randn(cin, generator=g) * 0.3
        wt = (torch.randn(128, cin, 1, 1, generator=g) * (2.0 / cin) ** 0.5).half().float()
        a = torch.relu(x.double() * ps.double() + pb.double())
        ref = torch.einsum('bhwc,oc->bhwo', a, wt[:, :, 0, 0].double())
        one, zero = torch.ones(128, device=DEV), torch.zeros(128, device=DEV)
        runs = [('whole_tiles', dict())]
        if (cin, b, hw) in STREAMK_SHAPES:
            runs.append(('streamk', dict(workspace=ws, flags=_streamk_flags(ops, b, hw, cin))))
        for kind, kw in runs:
            y = ops.conv1x1_preact(x.to(DEV), ops.pack_weight_f16(wt.to(DEV)), ps.to(DEV), pb.to(DEV), 1, one, zero, 1.0, **kw)
            e = rel_err(y, ref)
            worst[kind] = max(worst.get(kind, 0.0), e)
            assert e <= 1e-3, (cin, b, hw, kind, e)
    record('preact_accuracy_worst', worst)


@pytest.mark.gpu
def test_preact_conv_streamk_bit_identical_to_materialised_k1():
    """Stream-K segments (partial dump and collect through the workspace) of the pre-activation kernel against K1 on the materialised operand
    with the same tile, the same forced split and the same workspace: identical summation order, so identical bits."""
    from b200 import ops
    g = torch.Generator().manual_seed(10)
    ws = ops.conv_workspace()
    for cin, b, hw in STREAMK_SHAPES:
        x = torch.randn(b, hw, hw, cin + 32, generator=g).half()
        ps, pb = _f16_affine(cin, g)
        wt = torch.randn(128, cin, 1, 1, generator=g) * (2.0 / cin) ** 0.5
        scale, shift = (torch.rand(128, generator=g) + 0.5).to(DEV), (torch.randn(128, generator=g) * 0.1).to(DEV)
        wp = ops.pack_weight_f16(wt.to(DEV))
        a = (x[..., :cin].double() * ps.double() + pb.double()).clamp_min(0).float().half().to(DEV).contiguous()
        flags = _streamk_flags(ops, b, hw, cin)
        y = ops.conv1x1_preact(x.to(DEV), wp, ps.to(DEV), pb.to(DEV), 1, scale, shift, 0.0, cin=cin, flags=flags, workspace=ws)
        yr = ops.conv_bn_act(a, wp, scale, shift, 0.0, flags=flags, workspace=ws)
        assert torch.equal(y, yr), (cin, b, hw)


@pytest.mark.gpu
def test_densenet_pool_kernels():
    from b200 import ops
    g = torch.Generator().manual_seed(9)
    for b, h, w, c, x_ld in ((2, 26, 26, 256, 256), (3, 14, 10, 96, 128)):
        x = torch.randn(b, h, w, x_ld, generator=g).half()
        s, t = _f16_affine(c, g)
        y = torch.empty(b, h // 2, w // 2, c, dtype=torch.float16, device=DEV)
        ops.call('yb_bn_relu_avgpool2x2_f16', x.to(DEV), x_ld, s.to(DEV), t.to(DEV), y, b, h, w, c)
        r = (x[..., :c].double() * s.double() + t.double()).float().clamp_min(0)      # exact: fp16-representable affine
        ref = ((r[:, 0::2, 0::2] + r[:, 0::2, 1::2]) + (r[:, 1::2, 0::2] + r[:, 1::2, 1::2])) * 0.25
        assert torch.equal(y.cpu(), ref.half())
    for b, h, w, c, ld, off in ((2, 32, 48, 64, 256, 0), (1, 13, 27, 16, 64, 24)):
        x = torch.randn(b, h, w, c, generator=g).half().to(DEV)
        oh, ow = (h + 1) // 2, (w + 1) // 2
        y = torch.full((b, oh, ow, ld), 5.0, dtype=torch.float16, device=DEV)
        ops.call('yb_maxpool3x3_s2_ld_f16', x, y, ld, off, b, h, w, c)
        ref = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1)
        assert torch.equal(y[..., off:off + c].float(), ref)
        assert bool((y[..., :off] == 5).all() and (y[..., off + c:] == 5).all())
        y2 = torch.empty(b, oh, ow, c, dtype=torch.float16, device=DEV)
        ops.call('yb_maxpool3x3_s2_f16', x, y2, b, h, w, c)
        assert torch.equal(y2, y[..., off:off + c])


# ------------------------------------------------------------------------------------------------
# GPU: plugin
# ------------------------------------------------------------------------------------------------
TOL_E2E = 3e-3
TOL_LAYER = 2e-3


@pytest.mark.gpu
def test_plugin_vs_reference_golden(golden):
    rec = {}
    for name in ('densenet121', 'densenet169', 'densenet201'):
        net = build(name).to(DEV)
        with torch.no_grad():
            rec[name + '_feature64'] = rel_err(net(O.synth_images(1, 64, 64, seed=10).to(DEV)), torch.from_numpy(golden[name + '_feature64']))
            if name == 'densenet121':
                f416 = net(O.synth_images(1, 416, 416, seed=0).to(DEV))
                assert f416.shape == (1, 125, 13, 13)
                rec[name + '_feature416'] = rel_err(f416, torch.from_numpy(golden['densenet121_feature416']))
                acts = {}
                net.run(O.synth_images(1, 64, 64, seed=10).to(DEV), collect=acts)
                for k, v in acts.items():
                    rec['densenet121_act_' + k] = rel_err(v.permute(0, 3, 1, 2), torch.from_numpy(golden['densenet121_act_' + k]))
    record('golden', rec)
    assert all(v <= TOL_E2E for v in rec.values()), rec


@pytest.mark.gpu
def test_each_dense_layer_fed_oracle_input():
    """Every dense layer of densenet121 at 64x64, fed the oracle's own (fp16-rounded) block buffer: its 32 new channels vs the oracle."""
    name = 'densenet121'
    net = build(name).to(DEV)
    sd = D.make_densenet_state_dict(name, 0)
    acts = {}
    with torch.no_grad():
        D.densenet_forward(sd, O.synth_images(1, 64, 64, seed=10), name, collect=acts)
    worst = (0.0, '')
    bl, _ = D.blocks(name)
    with torch.no_grad():
        for bi, n, cin0 in bl:
            x = acts['pool0'] if bi == 1 else acts['transition%d' % (bi - 1)]
            feats = [x]
            _, _, h, w = x.shape
            cend = cin0 + n * 32
            buf = torch.zeros(1, h, w, cend, dtype=torch.float16, device=DEV)
            tmp = torch.empty(1, h, w, 128, dtype=torch.float16, device=DEV)
            block = getattr(net.features, 'denseblock%d' % bi)
            for j in range(n):
                cat = torch.cat(feats, 1)
                key = 'features.denseblock%d.denselayer%d' % (bi, j + 1)
                ref = D.dense_layer(sd, cat, key)
                c = cat.shape[1]
                buf[..., :c] = cat.permute(0, 2, 3, 1).half().to(DEV)
                net.dense_layer(key[len('features.'):], getattr(block, 'denselayer%d' % (j + 1)), buf, c, tmp)
                worst = max(worst, (rel_err(buf[..., c:c + 32].permute(0, 3, 1, 2), ref), key))
                feats.append(ref)
    record('worst_dense_layer', list(worst))
    assert worst[0] <= TOL_LAYER, worst


def _oracle_on_gpu(sd, x, name):
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return D.densenet_forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV), name)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.gpu
def test_batch32_and_non_square_vs_oracle():
    name = 'densenet121'
    net = build(name).to(DEV)
    sd = D.make_densenet_state_dict(name, 0)
    x = O.synth_images(32, 416, 416, seed=4)
    with torch.no_grad():
        y = net(x.to(DEV))
    ref = _oracle_on_gpu(sd, x, name)
    per = [rel_err(y[i], ref[i]) for i in range(32)]
    xr = O.synth_images(2, 320, 416, seed=5)
    with torch.no_grad():
        yr = net(xr.to(DEV))
    assert yr.shape == (2, 125, 10, 13)
    e_rect = rel_err(yr, _oracle_on_gpu(sd, xr, name))
    record('batch32_worst_image', [max(per), int(np.argmax(per))])
    record('non_square_320x416', e_rect)
    assert max(per) <= TOL_E2E and e_rect <= TOL_E2E, (max(per), e_rect)


@pytest.mark.gpu
def test_inference_reload_and_graph():
    import detect
    import model
    net = build('densenet121').to(DEV)
    cfg = make_config()
    inference = model.Inference(cfg, net, O.anchors_yolo_voc()).eval()
    pred = model._inference(inference, O.synth_images(3, 416, 416, seed=2).to(DEV))
    assert all(bool(torch.isfinite(v).all()) for v in pred.values() if isinstance(v, torch.Tensor))
    assert len(detect.postprocess_batch(cfg, pred)) == 3
    # cached operands follow load_state_dict
    x = O.synth_images(2, 128, 128, seed=3).to(DEV)
    with torch.no_grad():
        net(x)
        net.load_state_dict(D.make_densenet_state_dict('densenet121', 1), strict=False)
        y1 = net(x)
        y_fresh = build('densenet121', 1).to(DEV)(x)
    assert torch.equal(y1, y_fresh)
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
    static_x.copy_(O.synth_images(2, 128, 128, seed=6).to(DEV))
    graph.replay()
    with torch.no_grad():
        eager = net(static_x)
    torch.cuda.synchronize()
    assert torch.equal(static_y, eager)
