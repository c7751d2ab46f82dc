"""The two-consumer conv tile with the 2x2 max-pool fused into its epilogue (conv_wide_pool_kernel, YB_CONV_POOL2X2).

A pooled tile is 64 pool windows x their 4 positions; every output is the fp32 sum of the plain tile and goes through the same scale /
shift, leaky and fp16 rounding before an fp16 max in maxpool2x2_kernel's order.  So the fused launch must equal the plain two-consumer
launch followed by yb_maxpool2x2_f16 bit for bit, including which of +0 and -0 a tie keeps.  Every case writes a channel slice
(y_ch_off) of a wider buffer filled with a sentinel, and covers Darknet's two pooled 3x3 layers (104x104 64->128 and 52x52 128->256),
pooled grids that end inside a tile, one and two N tiles and both BK instantiations."""
import configparser

import pytest
import torch
import torch.nn.functional as F

from oracle import yolo2_oracle as O

pytestmark = pytest.mark.gpu

DEV = 'cuda'
SENTINEL = -7.5
PAD_LO, PAD_HI = 16, 24          # sentinel channels below and above the slice


@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


def bits(t):
    return t.contiguous().view(torch.int16)


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_unit(ops, b, h, w, cin, cout, seed, negative=False, tiny=False):
    """A 3x3 conv + BN + leaky unit.  negative: BN shifts push most outputs below zero (the leaky branch); tiny: scales of ~1e-9 round
    most outputs to +0 or -0 in fp16, so the max meets many signed-zero ties."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=gen)
    wt = torch.randn(cout, cin, 3, 3, generator=gen) * (2.0 / (cin * 9)) ** 0.5
    sd = {'u.conv.weight': wt, 'u.bn.weight': torch.rand(cout, generator=gen) + 0.5, 'u.bn.bias': torch.randn(cout, generator=gen) * 0.1,
          'u.bn.running_mean': torch.randn(cout, generator=gen) * 0.1, 'u.bn.running_var': torch.rand(cout, generator=gen) + 0.5}
    if negative:
        sd['u.bn.bias'] = sd['u.bn.bias'] - 1.5
    if tiny:
        sd['u.bn.weight'] = sd['u.bn.weight'] * 1e-9
        sd['u.bn.bias'] = torch.zeros(cout)
    scale, shift = ops.bn_fold(*(sd['u.bn.' + n].to(DEV) for n in ('weight', 'bias', 'running_mean', 'running_var')))
    return x, sd, x.to(DEV).permute(0, 2, 3, 1).contiguous().half(), ops.pack_weight_f16(wt.to(DEV)), scale, shift


def forced(ops, extra=0):
    return ops.conv_force_bn(128) | ops.conv_force_mt(2) | ops.CONV_NO_STREAMK | extra


def pooled_sliced(ops, x16, w16, scale, shift, flags):
    b, h, w, _ = x16.shape
    cout = w16.shape[0]
    buf = torch.full((b, h // 2, w // 2, PAD_LO + cout + PAD_HI), SENTINEL, dtype=torch.float16, device=DEV)
    ops.conv_bn_act(x16, w16, scale, shift, 0.1, out=buf, y_ch_off=PAD_LO, flags=flags)
    assert bool((buf[..., :PAD_LO] == SENTINEL).all()), 'channels below the slice were written'
    assert bool((buf[..., PAD_LO + cout:] == SENTINEL).all()), 'channels above the slice were written'
    return buf[..., PAD_LO:PAD_LO + cout]


CASES = [
    # b, H, W (conv input = output), cin, cout, input kind, what the case covers
    (2, 104, 104, 64, 128, '', 'layers1.6 at batch 2: BK = 64, one N tile, 169 pooled tiles'),
    (2, 52, 52, 128, 256, '', 'layers1.10 at batch 2: two N tiles'),
    (1, 20, 28, 64, 128, 'negative', 'pooled 1x10x14 = 140 windows: the last tile ends at row 12'),
    (3, 12, 44, 32, 256, 'negative', 'pooled 3x6x22 = 396 windows, BK = 32, two N tiles'),
    (2, 4, 4, 64, 128, '', 'pooled 2x2x2 = 8 windows: one tile, mostly past the end'),
    (2, 20, 20, 32, 128, 'tiny', 'outputs rounded to +0 / -0: signed-zero ties, BK = 32'),
    (1, 36, 36, 64, 256, 'tiny', 'signed-zero ties, two N tiles'),
]


@pytest.mark.parametrize('case', CASES, ids=[c[-1] for c in CASES])
def test_fused_pool_equals_conv_then_pool(ops, case):
    b, h, w, cin, cout, kind, _ = case
    x, sd, x16, w16, scale, shift = make_unit(ops, b, h, w, cin, cout, 11 * cin + cout + h + w, kind == 'negative', kind == 'tiny')
    ch = ops.conv_choice(b, h, w, cin, cout, 3, flags=forced(ops, ops.CONV_POOL2X2))
    assert ch['kernel'] == 'conv_wide_kernel' and ch['pooled'] and not ch['streamk'] and ch['bk'] == (64 if cin % 64 == 0 else 32), ch
    got = pooled_sliced(ops, x16, w16, scale, shift, forced(ops, ops.CONV_POOL2X2))
    full = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=forced(ops))
    want = ops.maxpool2x2(full)
    assert torch.equal(bits(got), bits(want)), 'fused max-pool differs from conv + maxpool2x2'
    if kind == 'negative':
        assert (full < 0).float().mean().item() > 0.5
    if kind == 'tiny':
        zeros = full == 0
        assert zeros.float().mean().item() > 0.5 and bool((zeros & torch.signbit(full)).any()) and bool((zeros & ~torch.signbit(full)).any())
    if b * h * w <= 4096 and kind != 'tiny':     # the fp64 oracle on the CPU: small cases only
        ref = F.max_pool2d(O.conv_unit(x.double(), {k: v.double() for k, v in sd.items()}, 'u', 3, True, True), 2)
        assert rel_err(got.permute(0, 3, 1, 2), ref) <= 1e-3


@pytest.mark.parametrize('shape', [(32, 104, 104, 64, 128), (32, 52, 52, 128, 256)], ids=['layers1.6', 'layers1.10'])
def test_darknet_layers_choose_the_pooled_form(ops, shape):
    """At batch 32, 416x416 the library's own selection takes the fused form for both layers, without forcing a tile."""
    b, h, w, cin, cout = shape
    ch = ops.conv_choice(b, h, w, cin, cout, 3, flags=ops.CONV_POOL2X2)
    assert ch['kernel'] == 'conv_wide_kernel' and ch['pooled'] and not ch['streamk'] and ch['rows'] == 256, ch
    assert ch == dict(ops.conv_choice(b, h, w, cin, cout, 3), pooled=True)


def test_pooled_form_refusals(ops):
    """Stream-K, odd sizes and shapes whose selection is not the two-consumer tile are refused, and a refused launch writes nothing."""
    x, sd, x16, w16, scale, shift = make_unit(ops, 2, 12, 12, 64, 128, 5)
    with pytest.raises(RuntimeError):
        ops.conv_choice(2, 12, 12, 64, 128, 3, flags=ops.conv_force_bn(128) | ops.conv_force_mt(2) | ops.CONV_FORCE_STREAMK | ops.CONV_POOL2X2)
    buf = torch.full((2, 6, 6, 128), SENTINEL, dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError):
        ops.conv_bn_act(x16, w16, scale, shift, 0.1, out=buf, workspace=ops.conv_workspace(DEV),
                        flags=ops.conv_force_bn(128) | ops.conv_force_mt(2) | ops.CONV_FORCE_STREAMK | ops.CONV_POOL2X2)
    with pytest.raises(RuntimeError):        # 128 x 128 tiles: no pooled form
        ops.conv_bn_act(x16, w16, scale, shift, 0.1, out=buf, flags=ops.conv_force_bn(128) | ops.conv_force_mt(1) | ops.CONV_POOL2X2)
    torch.cuda.synchronize()
    assert bool((buf == SENTINEL).all()), 'a refused launch wrote its output'
    with pytest.raises(RuntimeError):        # odd H
        ops.conv_choice(2, 13, 12, 64, 128, 3, flags=forced(ops, ops.CONV_POOL2X2))
    with pytest.raises(RuntimeError):        # 1x1
        ops.conv_choice(2, 12, 12, 64, 128, 1, flags=forced(ops, ops.CONV_POOL2X2))


def test_c2_forward_fused_pools_equal_unfused():
    """The C2 forward (batch 32, 416x416) with the pools of layers1.6 and layers1.10 fused and unfused gives the same head feature bit
    for bit, eager and graphed."""
    import model
    import model.yolo2
    from b200 import ops
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}})
    dnn = model.yolo2.Darknet(model.ConfigChannels(cfg), O.anchors_yolo_voc(), 20)
    dnn.load_state_dict(O.make_state_dict(0), strict=False)
    dnn = dnn.to(DEV).eval()
    x = torch.rand(32, 3, 416, 416, generator=torch.Generator().manual_seed(9)).to(DEV)
    eng = dnn.engine
    calls = []
    orig = ops.conv_bn_act

    def spy(*a, **kw):
        calls.append(kw.get('flags', 0))
        return orig(*a, **kw)
    ops.conv_bn_act = spy
    try:
        eng.fuse_wide_pool = False
        off = eng.forward(x).clone()
        pools_off = sum(1 for f in calls if f & ops.CONV_POOL2X2)
        del calls[:]
        eng.fuse_wide_pool = True
        on = eng.forward(x).clone()
        pools_on = sum(1 for f in calls if f & ops.CONV_POOL2X2)
    finally:
        ops.conv_bn_act = orig
    assert (pools_off, pools_on) == (1, 3), (pools_off, pools_on)
    assert torch.equal(on, off), 'fusing the pools changed the head feature'
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.forward(x, plan_id=1)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = eng.forward(x, plan_id=1)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, off)
