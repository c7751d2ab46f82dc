"""The configured tensor transform on the GPU (transform.TensorTransform, Backbone.set_input_transform):

  - yb_totensor_lut_u8 against torchvision's chain, bit for bit;
  - every first-layer `_lut` entry against its fp32 entry on the transformed image, bit for bit (both pad modes, pooled and not, fast and
    split, both conv0 kernel forms, batch 3, non-square);
  - every backbone's eval forward on uint8 frames against its forward on torchvision's fp32 image;
  - Darknet without a transform: the uint8 first layer is still yb_conv0_u8_bn_leaky_pool_fwd's 1/255 scaling;
  - DetectPipeline(uint8_input=True) with a transform: graph replay = eager = the fp32 pipeline on the transformed image;
  - train.iterate / GraphedStep on a Collate uint8 batch: the trainer gets torchvision's image bits and the launches of the fp32 step plus
    the one table launch."""
import configparser

import numpy as np
import pytest
import torch
import torchvision.transforms as T

from oracle import yolo2_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda'

IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
TRANSFORMS = {'to_tensor': [], 'reference': [((0.5, 0.5, 0.5), (1.0, 1.0, 1.0))], 'imagenet': [IMAGENET]}


def tensor_transform(name):
    import transform
    return transform.TensorTransform([T.ToTensor()] + [T.Normalize(m, s) for m, s in TRANSFORMS[name]])


def frames(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (b, h, w, 3), generator=g, dtype=torch.uint8).to(DEV)


def torchvision_image(t, x):
    """torchvision's chain, frame by frame on the CPU, as the reference applies it -> fp32 CUDA [B,3,H,W]."""
    chain = T.Compose(t.transforms)
    return torch.stack([chain(f.numpy()) for f in x.cpu()]).to(DEV)


def make_config(bn=True, **extra):
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': str(int(bn))}, 'model': {'pretrained': '0', 'threshold': '0.6'},
                   'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                   'hparam': {k: repr(float(v)) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    cfg.read_dict(extra)
    return cfg


def randomise_bn(net, seed):
    g = torch.Generator().manual_seed(seed)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            n = m.num_features
            m.weight.data.copy_(0.5 + torch.rand(n, generator=g))
            m.bias.data.copy_(torch.randn(n, generator=g) * 0.2)
            m.running_mean.copy_(torch.randn(n, generator=g) * 0.2)
            m.running_var.copy_(0.5 + torch.rand(n, generator=g))
    return net


def build(name):
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
    cc = model.ConfigChannels(make_config(bn=name != 'inception4_nobn'))
    if name.startswith('darknet'):
        net = model.yolo2.Darknet(cc, anchors, 20)
        net.load_state_dict(O.make_state_dict(0), strict=False)
    elif name == 'tiny':
        net = model.yolo2.Tiny(cc, anchors, 20)
    elif name.startswith('mobilenet'):
        net = model.mobilenet.MobileNet(cc, anchors, 20)
    elif name in ('resnet18', 'resnet50'):
        net = getattr(model.resnet, name)(cc, anchors, 20)
    elif name == 'densenet121':
        net = model.densenet.densenet121(cc, anchors, 20)
    elif name == 'inception3':
        import inception_oracle
        net = model.inception3.Inception3(cc, anchors, 20)
        net.load_state_dict(inception_oracle.make_inception_state_dict(4), strict=False)
    elif name.startswith('inception4'):
        import inception4_oracle
        net = model.inception4.Inception4(cc, anchors, 20)
        net.load_state_dict(inception4_oracle.make_state_dict(5, bn=name == 'inception4_bn'), strict=False)
    else:
        import vgg_oracle
        net = getattr(model.vgg, name)(cc, anchors, 20)
        net.load_state_dict(vgg_oracle.make_state_dict(name, seed=4), strict=False)
    if name in ('tiny', 'mobilenet', 'mobilenet_strict', 'resnet18', 'resnet50', 'densenet121'):
        randomise_bn(net, 3)
    net = net.to(DEV).eval()
    if name.endswith('_strict'):
        if name.startswith('darknet'):
            net.engine.set_precision('strict')
        else:
            net.set_precision('strict')
    return net, anchors


# ------------------------------------------------------------------------------------------------------------------------------------
# the table launch
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('shape', [(3, 96, 160), (2, 7, 13)])
def test_totensor_lut_equals_torchvision(name, shape):
    t = tensor_transform(name)
    x = frames(*shape, seed=1)
    got = t(x)
    assert got.shape == (shape[0], 3, shape[1], shape[2]) and got.dtype == torch.float32
    assert torch.equal(got, torchvision_image(t, x))
    assert t.lut(x.device) is t.lut(x.device)           # cached per device


# ------------------------------------------------------------------------------------------------------------------------------------
# every `_lut` entry against its fp32 entry
# ------------------------------------------------------------------------------------------------------------------------------------
def weights(cout, k, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(cout, 3, k, k, generator=g) * 0.3).to(DEV)
    scale = (0.5 + torch.rand(cout, generator=g)).to(DEV)
    shift = (torch.randn(cout, generator=g) * 0.1).to(DEV)
    return w, scale, shift


@pytest.mark.parametrize('name', ['reference', 'imagenet'])
@pytest.mark.parametrize('hw', [(96, 160), (48, 64)])     # 96 x 160: the operands-in-place form; 48 x 64 (H % 32 != 0): the first form
def test_conv0_lut(name, hw):
    from b200 import ops
    t = tensor_transform(name)
    x = frames(3, *hw, seed=2)
    w, s, b = weights(32, 3, 5)
    ref = ops.conv0_bn_leaky_pool(t(x), w, s, b, 0.1)
    got = ops.conv0_bn_leaky_pool(x, w, s, b, 0.1, lut=t.lut(x.device))
    assert torch.equal(got, ref)


@pytest.mark.parametrize('name', ['reference', 'imagenet'])
@pytest.mark.parametrize('pool', [False, True])
def test_conv0_c64_lut(name, pool):
    from b200 import ops
    t = tensor_transform(name)
    x = frames(3, 96, 160, seed=3)
    w, s, b = weights(64, 3, 6)
    ref = ops.conv0_c64_bn_act(t(x), w, s, b, 0.0, pool=pool)
    got = ops.conv0_c64_bn_act(x, w, s, b, 0.0, pool=pool, lut=t.lut(x.device))
    assert torch.equal(got, ref)


@pytest.mark.parametrize('name', ['reference', 'imagenet'])
@pytest.mark.parametrize('split', [False, True])
def test_mb_conv0_lut(name, split):
    from b200 import ops
    t = tensor_transform(name)
    x = frames(3, 96, 160, seed=4)
    w, s, b = weights(32, 3, 7)
    outs = []
    for args in ((t(x),), (x, t.lut(x.device))):
        y = torch.full((3, 48, 80, 64 if split else 32), float('nan'), dtype=torch.float16, device=DEV)
        entry = 'yb_mb_conv0_%s%s_fwd' % ('split' if split else 'bn_relu', '' if len(args) == 1 else '_lut')
        ops.call(entry, *args, w, s, b, y, 3, 96, 160)
        outs.append(y)
    assert torch.equal(outs[1], outs[0])


@pytest.mark.parametrize('name', ['reference', 'imagenet'])
@pytest.mark.parametrize('pad, hw', [(0, (107, 139)), (0, (96, 160)), (1, (96, 160)), (1, (107, 139))])
def test_stem3x3_s2_lut(name, pad, hw):
    from b200 import ops
    t = tensor_transform(name)
    x = frames(3, *hw, seed=5)
    w, s, b = weights(32, 3, 8)
    assert torch.equal(ops.stem3x3_s2(x, w, s, b, pad=pad, lut=t.lut(x.device)), ops.stem3x3_s2(t(x), w, s, b, pad=pad))


@pytest.mark.parametrize('name', ['reference', 'imagenet'])
def test_stem7x7_lut(name):
    from b200 import ops
    t = tensor_transform(name)
    x = frames(3, 96, 160, seed=6)
    w, s, b = weights(64, 7, 9)
    outs = []
    for args in ((t(x),), (x, t.lut(x.device))):
        y = torch.full((3, 48, 80, 64), float('nan'), dtype=torch.float16, device=DEV)
        ops.call('yb_stem7x7_bn_relu_fwd' if len(args) == 1 else 'yb_stem7x7_bn_relu_lut_fwd', *args, w, s, b, y, 3, 96, 160)
        outs.append(y)
    assert torch.equal(outs[1], outs[0])


def test_lut_entries_refuse_a_null_table():
    from b200 import ops
    x = frames(1, 32, 32, seed=0)
    w, s, b = weights(64, 7, 1)
    y = torch.zeros(1, 16, 16, 64, dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError, match='null table'):
        ops.call('yb_stem7x7_bn_relu_lut_fwd', x, None, w, s, b, y, 1, 32, 32)
    assert float(y.float().abs().sum()) == 0.0


# ------------------------------------------------------------------------------------------------------------------------------------
# every backbone
# ------------------------------------------------------------------------------------------------------------------------------------
BACKBONES = ['darknet', 'darknet_strict', 'tiny', 'mobilenet', 'mobilenet_strict', 'resnet18', 'resnet50', 'densenet121', 'inception3',
             'inception4_bn', 'inception4_nobn', 'vgg11', 'vgg11_bn']


@pytest.mark.parametrize('tname', sorted(TRANSFORMS))
@pytest.mark.parametrize('name', BACKBONES)
def test_backbone_uint8_equals_fp32_on_transformed_image(name, tname):
    """net.set_input_transform(t)(frames) against net(torchvision's image).  Should a backbone's eval forward not repeat its own fp32 result
    bit for bit, the uint8 result is held to twice that run-to-run spread instead (its first layer is held bit for bit above)."""
    net, _ = build(name)
    t = tensor_transform(tname)
    hw = (107, 139) if name.startswith('inception') else (96, 160)
    x = frames(3, *hw, seed=11)
    xf = torchvision_image(t, x)
    with torch.no_grad():
        ref = net(xf).clone()
        again = net(xf).clone()
        got = net.set_input_transform(t)(x).clone()
        f32_with_transform = net(xf).clone()          # an fp32 input is taken as already transformed
    assert got.shape == ref.shape and got.dtype == torch.float32 and bool(torch.isfinite(ref).all())
    if torch.equal(ref, again):
        assert torch.equal(got, ref)
        assert torch.equal(f32_with_transform, ref)
    else:
        spread = (ref - again).abs().max().item()
        err = (got - ref).abs().max().item()
        print('%s / %s: fp32 run-to-run spread %.3e, uint8 against fp32 %.3e' % (name, tname, spread, err))
        assert err <= 2 * spread


@pytest.mark.parametrize('name', ['tiny', 'resnet18', 'vgg11_bn'])
def test_backbone_uint8_without_transform_is_to_tensor(name):
    net, _ = build(name)
    x = frames(3, 96, 160, seed=12)
    import transform
    with torch.no_grad():
        assert net.input_transform is None
        assert torch.equal(net(x), net(transform.to_tensor(x)))


def test_darknet_without_transform_keeps_the_scaled_uint8_kernel():
    """No transform: Darknet's uint8 first layer is yb_conv0_u8_bn_leaky_pool_fwd (v * (1/255), the parent's kernel), not a table."""
    from b200 import ops
    net, _ = build('darknet')
    x = frames(3, 96, 160, seed=13)
    eng = net.engine
    acts = {}
    with torch.no_grad():
        feat = eng.forward(x, collect=acts).clone()
        u0 = eng.units1[0]
        ref0 = ops.conv0_u8_bn_leaky_pool(x, u0.w16, u0.scale, u0.shift, u0.slope)
        assert torch.equal(acts['layers1.0(pooled)'], ref0)
        assert torch.equal(net(x), feat)


# ------------------------------------------------------------------------------------------------------------------------------------
# the detection pipeline
# ------------------------------------------------------------------------------------------------------------------------------------
def test_detect_pipeline_with_transform():
    import model
    from b200.pipeline import DetectPipeline
    net, anchors = build('darknet')
    t = tensor_transform('reference')
    net.set_input_transform(t)
    cfg = make_config()
    inference = model.Inference(cfg, net, anchors).eval()
    x = frames(4, 416, 416, seed=14)
    outs = []
    for uint8, graph in ((True, False), (True, True), (False, True)):
        pipe = DetectPipeline(inference, cfg, 4, 416, 416, slots=1, use_graph=graph, uint8_input=uint8).prepare()
        pipe.x[0].copy_(x if uint8 else t(x))
        torch.cuda.synchronize()
        out = pipe.run(0)
        pipe.wait_all()
        outs.append({k: v.clone() for k, v in out.items()})
        torch.cuda.synchronize()
    for k in ('feature', 'iou', 'yx_min', 'yx_max', 'n_keep', 'keep_box', 'n_det'):
        assert torch.equal(outs[0][k], outs[1][k]), k
        assert torch.equal(outs[1][k], outs[2][k]), k
    for k in ('det_keep', 'det_cls', 'det_score'):            # each image's first n_det entries are written
        for i, n in enumerate(outs[0]['n_det'].tolist()):
            assert torch.equal(outs[0][k][i, :n], outs[1][k][i, :n]), k
            assert torch.equal(outs[1][k][i, :n], outs[2][k][i, :n]), k


# ------------------------------------------------------------------------------------------------------------------------------------
# training on a uint8 batch
# ------------------------------------------------------------------------------------------------------------------------------------
class Recorder(object):
    """Wraps b200.ops.call: the name and the arguments (tensors as shape and dtype) of every library call."""

    def __init__(self, ops):
        self.real = ops.call
        self.calls = []

    def __call__(self, name, *args):
        self.calls.append((name, tuple(('T', tuple(a.shape), a.dtype) if torch.is_tensor(a) else a for a in args)))
        return self.real(name, *args)


def collate_batch():
    import utils.data as ud
    samples = []
    for i, (h, w, n) in enumerate(((90, 120, 2), (75, 100, 1), (64, 64, 3))):
        g = np.random.RandomState(70 + i)
        lo = (g.rand(n, 2) * [h * 0.5, w * 0.5]).astype(np.float32)
        samples.append(dict(image=O.synth_frame(40 + i, h, w), yx_min=lo, yx_max=lo + (g.rand(n, 2) * [h * 0.4, w * 0.4] + 4).astype(np.float32),
                            cls=g.randint(0, 20, n)))
    return ud.Collate([(64, 96)], maintain=3, seed=2)(samples)


def train_net(name):
    import model
    net, anchors = build(name)
    net = net.train()
    inference = model.Inference(make_config(), net, anchors).train()
    opt = torch.optim.SGD(net.parameters(), lr=0.0, momentum=0.0)
    return net, inference, opt, anchors


@pytest.mark.parametrize('name', ['darknet', 'resnet18'])
def test_iterate_uint8_with_transform(name, monkeypatch):
    import train as yb_train
    from b200 import ops
    batch = collate_batch()
    assert batch['tensor'].dtype == torch.uint8
    net, inference, opt, anchors = train_net(name)
    t = tensor_transform('reference')
    net.set_input_transform(t)
    seen = []
    real_forward = net.trainer.forward
    monkeypatch.setattr(net.trainer, 'forward', lambda x: (seen.append(x.clone()), real_forward(x))[1])
    rec = Recorder(ops)
    monkeypatch.setattr(ops, 'call', rec)
    fp32 = dict(batch, tensor=torchvision_image(t, batch['tensor']))
    yb_train.iterate(inference, opt, anchors, make_config(), fp32)
    ref_calls, rec.calls = rec.calls, []
    yb_train.iterate(inference, opt, anchors, make_config(), batch)
    got_calls = rec.calls
    assert torch.equal(seen[0], fp32['tensor']) and torch.equal(seen[1], fp32['tensor'])
    assert got_calls[0][0] == 'yb_totensor_lut_u8' and got_calls[1:] == ref_calls


@pytest.mark.parametrize('name', ['darknet', 'resnet18'])
def test_graphed_step_uint8_with_transform(name, monkeypatch):
    import train as yb_train
    batch = collate_batch()
    t = tensor_transform('reference')
    launches, images = [], []
    for uint8 in (False, True):
        net, inference, opt, anchors = train_net(name)
        net.set_input_transform(t)
        seen = []
        real_forward = net.trainer.forward
        monkeypatch.setattr(net.trainer, 'forward', lambda x, seen=seen, real=real_forward: (seen.append(x), real(x))[1])
        data = batch if uint8 else dict(batch, tensor=torchvision_image(t, batch['tensor']))
        step = yb_train.GraphedStep(inference, opt, anchors, make_config())
        step(data)
        torch.cuda.synchronize()
        launches.append(step.launches)
        images.append(seen[-1].clone())              # the captured step's input buffer, as the replay left it
        step.finish()
    assert torch.equal(images[1], images[0]) and torch.equal(images[0], torchvision_image(t, batch['tensor']))
    assert launches[1] == launches[0] + 1
