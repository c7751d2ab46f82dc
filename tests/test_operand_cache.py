"""The backbone plugins' kernel-operand cache (b200.engine.OperandCache) and the shared plugin base (model.Backbone).

CPU: OperandCache hits return the stored object and rebuild on an in-place update, a replaced tensor or a changed `extra`; every plugin drops
its cached operands on a train() / eval() switch (and only then), also through train.GraphedStep.finish; every plugin names its trainer.

GPU: every plugin at a small size, launches counted with b200.ops.launch_count: a second eval forward issues no pack or fold launch and
nothing else changes; after an in-place parameter update the forward re-packs everything and equals a freshly built model bit for bit;
.train().eval() re-packs and gives the same output."""
import configparser

import pytest
import torch

import model
import model.densenet
import model.inception3
import model.inception4
import model.mobilenet
import model.resnet
import model.vgg
import model.yolo2
from b200 import engine
from b200 import ops
from b200 import train_engine
from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu

# plugin -> (constructor, the b200.train_engine class that trains it, input height and width)
PLUGINS = {
    'darknet': (model.yolo2.Darknet, 'DarknetTrainer', (64, 96)),
    'tiny': (model.yolo2.Tiny, 'TinyTrainer', (64, 96)),
    'resnet18': (model.resnet.resnet18, 'ResNetTrainer', (64, 96)),
    'mobilenet': (model.mobilenet.MobileNet, 'MobileNetTrainer', (64, 96)),
    'vgg11_bn': (model.vgg.vgg11_bn, 'VGGTrainer', (64, 96)),
    'inception3': (model.inception3.Inception3, 'InceptionTrainer', (107, 139)),
    'inception4': (model.inception4.Inception4, 'Inception4Trainer', (107, 139)),
    'densenet121': (model.densenet.densenet121, 'DenseNetTrainer', (64, 96)),
}
PREP = ('pack_weight_f16', 'pack_weight_split_f16', 'pack_weight_khw_f16', 'bn_fold')     # the operand builds of the eval forwards


def build(name):
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}})
    return PLUGINS[name][0](model.ConfigChannels(config), O.anchors_yolo_voc(), 20)


# ---- CPU ---------------------------------------------------------------------------------------------
def test_hit_returns_the_stored_object():
    cache, p = engine.OperandCache(), torch.nn.Parameter(torch.ones(4))
    built = []

    def make():
        built.append(p.detach().clone())
        return built[-1]
    first = cache.fetch('k', (p,), make)
    assert cache.fetch('k', (p,), make) is first and len(built) == 1
    assert cache.fetch('c', (), lambda: torch.zeros(1)) is cache.fetch('c', (), lambda: torch.ones(1))      # tensors=(): built once
    assert len(cache) == 2


def test_updates_rebuild():
    p, q = torch.nn.Parameter(torch.ones(4)), torch.nn.Parameter(torch.ones(4))
    cache, built = engine.OperandCache(), []

    def fetch(tensors, extra=()):
        return cache.fetch('k', tensors, lambda: built.append(None) or len(built), extra)
    assert fetch((p, q)) == 1 and fetch((p, q)) == 1
    with torch.no_grad():
        p.add_(1)                    # advances p._version (p.data.add_ would not)
    assert fetch((p, q)) == 2 and fetch((p, q)) == 2
    q.data = torch.zeros(4)          # replaced storage: same version counter, new data_ptr
    assert fetch((p, q)) == 3 and fetch((p, q)) == 3
    assert fetch((p, q), extra=(32,)) == 4 and fetch((p, q), extra=(32,)) == 4 and fetch((p, q), extra=(64,)) == 5
    assert list(cache) == ['k']      # one entry per key
    cache.clear()
    assert cache == {}
    assert fetch((p, q), extra=(64,)) == 6


@pytest.mark.parametrize('name', sorted(PLUGINS))
def test_train_eval_switch_drops_the_operands(name):
    import train as yb_train
    net = build(name).eval()
    assert isinstance(net, model.Backbone) and type(net).TRAINER is getattr(train_engine, PLUGINS[name][1])
    units = []
    if name == 'darknet':
        units = net.engine.all_units()
    elif name == 'tiny':
        units = [u for u, _ in net._plan()]

    def fill():
        net._cache['x'] = 1
        for u in units:
            u._wver = u._bver = ('x',)

    def dropped():
        if name == 'darknet':            # Darknet's operands live in its engine's units
            return all(u._wver is None and u._bver is None for u in units)
        return net._cache == {} and all(u._wver is None and u._bver is None for u in units)

    fill()
    net.eval()                           # no mode change: the operands stay
    assert net._cache and not dropped()
    for switch in (net.train, net.eval):
        fill()
        switch()
        assert dropped()
    fill()
    yb_train.GraphedStep(model.Inference(None, net, O.anchors_yolo_voc()), None, None, None).finish()
    assert dropped()


# ---- GPU ---------------------------------------------------------------------------------------------
@pytest.fixture
def prep_launches(monkeypatch):
    """Counts the kernel launches issued inside the operand builds (b200.ops.launch_count)."""
    count = [0]
    for fn in PREP:
        def counted(*args, _fn=getattr(ops, fn), **kwargs):
            n0 = ops.launch_count
            try:
                return _fn(*args, **kwargs)
            finally:
                count[0] += ops.launch_count - n0
        monkeypatch.setattr(ops, fn, counted)
    return count


@gpu
@pytest.mark.parametrize('name', sorted(PLUGINS))
def test_eval_operands_follow_parameter_versions(name, prep_launches):
    h, w = PLUGINS[name][2]
    torch.manual_seed(0)
    net = build(name)
    for m in net.modules():              # variance-preserving weights, so that every layer's fp16 activations stay finite and non-zero
        if isinstance(m, torch.nn.Conv2d):
            torch.nn.init.kaiming_normal_(m.weight)
    net = net.to(DEV).eval()
    x = O.synth_images(2, h, w, seed=1).to(DEV)

    def forward():
        p0, n0 = prep_launches[0], ops.launch_count
        with torch.no_grad():
            y = net(x)
        torch.cuda.synchronize()
        return y, ops.launch_count - n0, prep_launches[0] - p0

    y1, n1, p1 = forward()
    y2, n2, p2 = forward()
    assert torch.isfinite(y1).all() and y1.abs().max() > 0
    assert p1 > 0 and p2 == 0 and n2 == n1 - p1 and torch.equal(y1, y2)
    with torch.no_grad():
        for p in net.parameters():
            p.add_(torch.randn_like(p), alpha=0.01)
    y3, n3, p3 = forward()
    assert (n3, p3) == (n1, p1) and not torch.equal(y3, y1)
    fresh = build(name)
    fresh.load_state_dict(net.state_dict())
    with torch.no_grad():
        assert torch.equal(fresh.to(DEV).eval()(x), y3)
    net.train().eval()
    y4, n4, p4 = forward()
    assert (n4, p4) == (n1, p1) and torch.equal(y4, y3)
