"""The two-consumer conv tile with the following 1x1 unit run in its epilogue (conv_wide_chain_kernel, yb_conv_bn_act_chain_fwd).

After a 64-row half of the tile is converted to fp16, its 128 channels are the register A operand of a second GEMM against the 1x1 weight,
with the same k16 steps in the same channel order as the 1x1 unit's own launch, and the same scale / shift / leaky / fp16 epilogue.  So the
fused launch must equal the plain producer launch followed by the plain 1x1 launch bit for bit.  Every case writes a channel slice
(y_ch_off) of a wider buffer filled with a sentinel; it covers Darknet's layers1.4 -> layers1.5 pair (104x104, 64 -> 128 -> 64), grids
whose pixel count ends inside a tile, Cout2 below 64, and negative and signed-zero second-unit outputs."""
import configparser

import pytest
import torch

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


def bn_params(gen, c, prefix, negative=False, tiny=False):
    sd = {prefix + '.bn.weight': torch.rand(c, generator=gen) + 0.5, prefix + '.bn.bias': torch.randn(c, generator=gen) * 0.1,
          prefix + '.bn.running_mean': torch.randn(c, generator=gen) * 0.1, prefix + '.bn.running_var': torch.rand(c, generator=gen) + 0.5}
    if negative:
        sd[prefix + '.bn.bias'] = sd[prefix + '.bn.bias'] - 1.5
    if tiny:
        sd[prefix + '.bn.weight'] = sd[prefix + '.bn.weight'] * 1e-9
        sd[prefix + '.bn.bias'] = torch.zeros(c)
    return sd


def make_pair(ops, b, h, w, cin, k, cout2, seed, kind=''):
    """Unit a: k x k conv Cin -> 128 + BN + leaky; unit c: 1x1 conv 128 -> Cout2 + BN + leaky.  kind 'negative': c's BN shifts push
    most of its outputs below zero (the leaky branch); 'tiny': c's scales of ~1e-9 round most of its outputs to +0 or -0 in fp16."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=gen)
    wa = torch.randn(128, cin, k, k, generator=gen) * (2.0 / (cin * k * k)) ** 0.5
    wc = torch.randn(cout2, 128, 1, 1, generator=gen) * (2.0 / 128) ** 0.5
    sd = {'a.conv.weight': wa, 'c.conv.weight': wc}
    sd.update(bn_params(gen, 128, 'a'))
    sd.update(bn_params(gen, cout2, 'c', kind == 'negative', kind == 'tiny'))

    def fold(p):
        return ops.bn_fold(*(sd[p + '.bn.' + n].to(DEV) for n in ('weight', 'bias', 'running_mean', 'running_var')))
    ua = (ops.pack_weight_f16(wa.to(DEV)),) + fold('a')
    uc = (ops.pack_weight_f16(wc.to(DEV)),) + fold('c')
    return x, sd, x.to(DEV).permute(0, 2, 3, 1).contiguous().half(), ua, uc


def fused_sliced(ops, x16, ua, uc, flags=0, workspace=None):
    b, h, w, _ = x16.shape
    cout2 = uc[0].shape[0]
    buf = torch.full((b, h, w, PAD_LO + cout2 + PAD_HI), SENTINEL, dtype=torch.float16, device=DEV)
    ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, out=buf, y_ch_off=PAD_LO, flags=flags, workspace=workspace,
                    chain=(uc[0], uc[1], uc[2], 0.1))
    assert bool((buf[..., :PAD_LO] == SENTINEL).all()), 'channels below the slice were written'
    assert bool((buf[..., PAD_LO + cout2:] == SENTINEL).all()), 'channels above the slice were written'
    return buf[..., PAD_LO:PAD_LO + cout2]


def separate(ops, x16, ua, uc, workspace=None):
    mid = ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, workspace=workspace)
    return mid, ops.conv_bn_act(mid, uc[0], uc[1], uc[2], 0.1, workspace=workspace)


CASES = [
    # b, H, W, cin, k, cout2, kind, what the case covers
    (32, 104, 104, 64, 3, 64, '', 'layers1.4 -> layers1.5 at batch 32, 416x416'),
    (1, 20, 28, 64, 3, 64, 'negative', '560 pixels: the last tile ends at row 48 of its 256'),
    (3, 12, 44, 128, 3, 64, '', '1584 pixels, Cin = 128: the last tile ends inside consumer 0'),
    (2, 9, 7, 64, 1, 32, 'negative', '1x1 producer, 126 pixels, Cout2 = 32'),
    (2, 20, 20, 64, 3, 40, 'tiny', 'second-unit outputs rounded to +0 / -0, Cout2 = 40'),
]


@pytest.mark.parametrize('case', CASES, ids=[c[-1] for c in CASES])
def test_fused_chain_equals_two_launches(ops, case):
    b, h, w, cin, k, cout2, kind, _ = case
    x, sd, x16, ua, uc = make_pair(ops, b, h, w, cin, k, cout2, 7 * cin + cout2 + h + w + k, kind)
    ws = ops.conv_workspace(DEV)
    # the small grids force the two-consumer tile, which their own selection may not take; the 1x1 launch keeps its own selection
    flags = 0 if b * h * w >= 100000 else ops.conv_force_bn(128) | ops.conv_force_mt(2)
    ch = ops.conv_choice(b, h, w, cin, 128, k, flags=flags | ops.CONV_CHAIN1X1)
    assert ch['kernel'] == 'conv_wide_kernel' and ch['chained'] and not ch['streamk'] and ch['bk'] == 64 and ch['bn'] == 128, ch
    got = fused_sliced(ops, x16, ua, uc, flags=flags, workspace=ws)
    mid, want = separate(ops, x16, ua, uc, workspace=ws)
    assert torch.equal(bits(got), bits(want)), 'fused 1x1 differs from the two launches'
    if kind == 'negative':
        assert (want < 0).float().mean().item() > 0.5
    if kind == 'tiny':
        zeros = want == 0
        assert zeros.float().mean().item() > 0.5 and bool((zeros & torch.signbit(want)).any()) and bool((zeros & ~torch.signbit(want)).any())
    if b * h * w <= 4096 and kind != 'tiny':     # the fp64 oracle on the CPU: small cases only
        sd64 = {n: v.double() for n, v in sd.items()}
        ref = O.conv_unit(O.conv_unit(x.double(), sd64, 'a', k, True, True), sd64, 'c', 1, True, True)
        assert rel_err(got.permute(0, 3, 1, 2), ref) <= 2e-3


def test_darknet_pairs_choose_the_chained_form(ops):
    """At batch 32, 416x416 layers1.4 (104x104, 64 -> 128) takes the chained form with the library's own selection, which is its plain
    selection; layers1.8 (52x52, 128 -> 256) has two N tiles and is refused."""
    ch = ops.conv_choice(32, 104, 104, 64, 128, 3, flags=ops.CONV_CHAIN1X1)
    assert ch == dict(ops.conv_choice(32, 104, 104, 64, 128, 3), chained=True) and ch['kernel'] == 'conv_wide_kernel', ch
    with pytest.raises(RuntimeError):
        ops.conv_choice(32, 52, 52, 128, 256, 3, flags=ops.CONV_CHAIN1X1)


def test_chained_form_refusals(ops):
    """Producers other than a 128-channel two-consumer tile, stream-K, a fused pool and a second unit wider than 64 channels are
    refused, and a refused launch writes nothing."""
    x, sd, x16, ua, uc = make_pair(ops, 2, 12, 12, 64, 3, 64, 5)
    ws = ops.conv_workspace(DEV)
    flags_wide = ops.conv_force_bn(128) | ops.conv_force_mt(2)
    for flags in (ops.conv_force_bn(128) | ops.conv_force_mt(1) | ops.CONV_CHAIN1X1,      # 128 x 128 tiles
                  flags_wide | ops.CONV_FORCE_STREAMK | ops.CONV_CHAIN1X1,                # stream-K
                  flags_wide | ops.CONV_POOL2X2 | ops.CONV_CHAIN1X1):                     # fused pool as well
        with pytest.raises(RuntimeError):
            ops.conv_choice(2, 12, 12, 64, 128, 3, flags=flags)
    with pytest.raises(RuntimeError):        # Cout = 256: two N tiles
        ops.conv_choice(2, 12, 12, 64, 256, 3, flags=ops.CONV_CHAIN1X1)
    with pytest.raises(RuntimeError):        # Cin = 32: BK = 32 producers
        ops.conv_choice(2, 12, 12, 32, 128, 3, flags=ops.CONV_CHAIN1X1)
    buf = torch.full((2, 12, 12, 128), SENTINEL, dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError):
        ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, out=buf, workspace=ws, flags=flags_wide | ops.CONV_FORCE_STREAMK,
                        chain=(uc[0], uc[1], uc[2], 0.1))
    with pytest.raises(RuntimeError):        # forced 128 x 128 tiles
        ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, out=buf, flags=ops.conv_force_bn(128) | ops.conv_force_mt(1),
                        chain=(uc[0], uc[1], uc[2], 0.1))
    wc96 = ops.pack_weight_f16(torch.randn(96, 128, 1, 1, device=DEV) * 0.1)
    with pytest.raises(RuntimeError):        # Cout2 = 96 > 64
        ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, out=buf, chain=(wc96, torch.ones(96, device=DEV), torch.zeros(96, device=DEV), 0.1))
    with pytest.raises(RuntimeError):        # the flag without a second unit
        ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, out=buf, flags=ops.CONV_CHAIN1X1)
    torch.cuda.synchronize()
    assert bool((buf == SENTINEL).all()), 'a refused launch wrote its output'
    with pytest.raises(ValueError):          # w2 whose Cin is not the producer's Cout
        ops.conv_bn_act(x16, ua[0], ua[1], ua[2], 0.1, chain=(uc[0][:, :, :, :64].contiguous(), uc[1], uc[2], 0.1))


def test_c2_forward_chain_equals_unchained():
    """The C2 forward (batch 32, 416x416) with layers1.5 fused into layers1.4's launch and with the separate launches gives the same head
    feature bit for bit, eager and graphed."""
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
        calls.append(kw.get('chain') is not None)
        return orig(*a, **kw)
    ops.conv_bn_act = spy
    try:
        eng.fuse_chain = False
        off = eng.forward(x).clone()
        n_off, chained_off = len(calls), sum(calls)
        del calls[:]
        eng.fuse_chain = True
        on = eng.forward(x).clone()
        n_on, chained_on = len(calls), sum(calls)
    finally:
        ops.conv_bn_act = orig
    assert (chained_off, chained_on, n_off - n_on) == (0, 1, 1), (chained_off, chained_on, n_off, n_on)
    assert torch.equal(on, off), 'fusing layers1.5 changed the head feature'
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
