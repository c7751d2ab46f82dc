"""The two-consumer 256 x 128 implicit-GEMM conv (conv_wide_kernel): every form, forced by the tile flags, against the oracle
arithmetic; bit equality with the 128 x 128 one-warpgroup kernel on launches without stream-K (same K-block order, only the
partition of M and N differs); the stream-K flags back at zero after repeated launches; the C2 forward under CUDA graphs on two
streams equal to eager."""
import configparser

import pytest
import torch

from oracle import yolo2_oracle as O

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def rel_err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


def wide(ops, sk):
    return ops.conv_force_bn(128) | ops.conv_force_mt(2) | (ops.CONV_FORCE_STREAMK if sk else ops.CONV_NO_STREAMK)


def narrow(ops):
    return ops.conv_force_bn(128) | ops.conv_force_mt(1) | ops.CONV_NO_STREAMK


def make_unit(ops, b, h, w, cin, cout, k, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=gen)
    wt = torch.randn(cout, cin, k, k, generator=gen) * (2.0 / (cin * k * k)) ** 0.5
    sd = {'u.conv.weight': wt, 'u.bn.weight': torch.rand(cout, generator=gen) + 0.5, 'u.bn.bias': torch.randn(cout, generator=gen) * 0.1,
          'u.bn.running_mean': torch.randn(cout, generator=gen) * 0.1, 'u.bn.running_var': torch.rand(cout, generator=gen) + 0.5}
    ref = O.conv_unit(x, sd, 'u', k, True, True)
    scale, shift = ops.bn_fold(*(sd['u.bn.' + n].to(DEV) for n in ('weight', 'bias', 'running_mean', 'running_var')))
    return x.to(DEV).permute(0, 2, 3, 1).contiguous().half(), ops.pack_weight_f16(wt.to(DEV)), scale, shift, ref


CASES = [
    # b, h, w, cin, cout, k
    (3, 13, 13, 512, 1024, 3),      # layers2.x at batch 3: M = 507, not a multiple of 256
    (2, 26, 26, 256, 512, 3),       # layers1.12 / 1.14 / 1.16
    (2, 52, 52, 128, 256, 3),       # layers1.8 / 1.10
    (2, 104, 104, 64, 128, 3),      # layers1.4 / 1.6: 9 K-blocks per tile
    (3, 13, 13, 1024, 512, 1),      # 1x1 (A through the plain 2-D tiled TMA)
    (2, 13, 13, 1280, 1024, 3),     # layers3.0
    (3, 13, 13, 256, 384, 3),       # three column tiles (odd n-tile count)
    (5, 19, 17, 96, 136, 3),        # BK = 32, ragged rows and a ragged column tile
]


@pytest.mark.parametrize('case', CASES)
def test_wide_tile_vs_oracle_and_narrow(ops, case):
    b, h, w, cin, cout, k = case
    x16, w16, scale, shift, ref = make_unit(ops, b, h, w, cin, cout, k, cin * 5 + cout + h)
    assert ops.conv_choice(b, h, w, cin, cout, k, flags=wide(ops, False))['kernel'] == 'conv_wide_kernel'
    y = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=wide(ops, False))
    err = rel_err(y.permute(0, 3, 1, 2), ref)
    assert err <= 1e-3, 'rel err %.3e' % err
    y128 = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=narrow(ops))
    assert torch.equal(y, y128), 'two-consumer tile differs from the 128 x 128 tile'


SK_CASES = [
    # b, h, w, cin, cout, k: sizes with at least 4 K-blocks per CTA, so a forced stream-K launch really splits tiles
    (3, 13, 13, 512, 1024, 3),      # M = 507, not a multiple of 256
    (2, 26, 26, 256, 512, 3),
    (2, 52, 52, 128, 256, 3),
    (2, 104, 104, 64, 128, 3),
    (13, 13, 13, 1024, 512, 1),     # 1x1
    (2, 13, 13, 1280, 1024, 3),
    (3, 13, 13, 1024, 384, 3),      # three column tiles (odd n-tile count)
    (12, 19, 17, 96, 136, 3),       # BK = 32, ragged rows and a ragged column tile
]


@pytest.mark.parametrize('case', SK_CASES)
def test_wide_tile_streamk(ops, case):
    b, h, w, cin, cout, k = case
    x16, w16, scale, shift, ref = make_unit(ops, b, h, w, cin, cout, k, cin * 3 + cout + k)
    ws = ops.conv_workspace(DEV)
    ch = ops.conv_choice(b, h, w, cin, cout, k, flags=wide(ops, True))
    assert ch['kernel'] == 'conv_wide_kernel' and ch['streamk'], ch
    for rep in range(3):      # repeated launches reuse the workspace: the flags must come back to zero every time
        y = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=wide(ops, True), workspace=ws)
        err = rel_err(y.permute(0, 3, 1, 2), ref)
        assert err <= 1e-3, 'launch %d: rel err %.3e' % (rep, err)
        assert int(ws[:4096].view(torch.int32).abs().sum().item()) == 0, 'stream-K flags not reset'
    y0 = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=narrow(ops))
    assert rel_err(y, y0) <= 2e-3


@pytest.mark.parametrize('sk', [False, True])
def test_wide_tile_channel_slice(ops, sk):
    """y_ch_off into a wider buffer (how layers2.6 writes into the concat): the channels outside the slice stay untouched."""
    b, h, w, cin, cout = 2, 13, 13, 1024, 256
    x16, w16, scale, shift, ref = make_unit(ops, b, h, w, cin, cout, 3, 17)
    ch = ops.conv_choice(b, h, w, cin, cout, 3, flags=wide(ops, sk))
    assert ch['kernel'] == 'conv_wide_kernel' and ch['streamk'] == sk, ch
    buf = torch.full((b, h, w, 400), 3.0, dtype=torch.float16, device=DEV)
    ops.conv_bn_act(x16, w16, scale, shift, 0.1, out=buf, y_ch_off=136, flags=wide(ops, sk), workspace=ops.conv_workspace(DEV) if sk else None)
    assert rel_err(buf[..., 136:392].permute(0, 3, 1, 2), ref) <= 1e-3
    assert bool((buf[..., :136] == 3).all()) and bool((buf[..., 392:] == 3).all())
    if not sk:
        y128 = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=narrow(ops))
        assert torch.equal(buf[..., 136:392], y128)


@pytest.mark.parametrize('sk', [False, True])
def test_wide_tile_split_operands(ops, sk):
    """Strict mode's split operands on the two-consumer tile, without a residual output: A = [a_hi | a_lo | a_hi] over an activation
    that holds [hi | lo], so the third segment's channel offsets wrap around (a_wrap)."""
    b, h, w, cin, cout, k = 3, 13, 13, 256, 512, 3
    gen = torch.Generator().manual_seed(23)
    x = torch.randn(b, cin, h, w, generator=gen)
    wt = torch.randn(cout, cin, k, k, generator=gen) * (2.0 / (cin * k * k)) ** 0.5
    sd = {'u.conv.weight': wt, 'u.bn.weight': torch.rand(cout, generator=gen) + 0.5, 'u.bn.bias': torch.randn(cout, generator=gen) * 0.1,
          'u.bn.running_mean': torch.randn(cout, generator=gen) * 0.1, 'u.bn.running_var': torch.rand(cout, generator=gen) + 0.5}
    ref = O.conv_unit(x, sd, 'u', k, True, True)
    scale, shift = ops.bn_fold(*(sd['u.bn.' + n].to(DEV) for n in ('weight', 'bias', 'running_mean', 'running_var')))
    xn = x.permute(0, 2, 3, 1).contiguous()
    hi = xn.half()
    src = torch.cat([hi, (xn - hi.float()).half()], -1).contiguous().to(DEV)
    w16 = ops.pack_weight_split_f16(wt.to(DEV), True, True)
    assert w16.shape[-1] == 3 * cin
    ch = ops.conv_choice(b, h, w, 3 * cin, cout, k, flags=wide(ops, sk))
    assert ch['kernel'] == 'conv_wide_kernel' and ch['streamk'] == sk, ch
    ws = ops.conv_workspace(DEV) if sk else None
    out = torch.empty(b, h, w, cout, dtype=torch.float16, device=DEV)
    ops.conv_bn_act_split(src, w16, scale, shift, 0.1, out, a_channels=2 * cin, flags=wide(ops, sk), workspace=ws)
    assert rel_err(out.permute(0, 3, 1, 2), ref) <= 1e-3
    if not sk:
        out128 = torch.empty_like(out)
        ops.conv_bn_act_split(src, w16, scale, shift, 0.1, out128, a_channels=2 * cin, flags=narrow(ops))
        assert torch.equal(out, out128)


def test_wide_tile_refused_where_unsupported(ops):
    """The head (fp32 NCHW) has no two-consumer form: forcing it is an error, and the library never picks it there."""
    with pytest.raises(RuntimeError):
        ops.conv_choice(32, 13, 13, 1024, 125, 1, out_mode=ops.OUT_F32_NCHW, flags=wide(ops, False))
    assert ops.conv_choice(32, 13, 13, 1024, 125, 1, out_mode=ops.OUT_F32_NCHW)['kernel'] == 'conv_igemm_kernel'


def test_c2_forward_two_lanes_graphed_equals_eager():
    """The C2 forward (batch 32, 416x416) captured in CUDA graphs on two streams, replayed concurrently, equals the eager forward
    bit for bit: the same launches with the same tile and stream-K choices, each lane with its own workspace."""
    import model
    import model.yolo2
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}})
    dnn = model.yolo2.Darknet(model.ConfigChannels(cfg), O.anchors_yolo_voc(), 20)
    dnn.load_state_dict(O.make_state_dict(0), strict=False)
    dnn = dnn.to(DEV).eval()
    gen = torch.Generator().manual_seed(4)
    xs = [torch.rand(32, 3, 416, 416, generator=gen).to(DEV) for _ in range(2)]
    eager = [dnn.engine.forward(x, plan_id=2).clone() for x in xs]
    graphs, outs, streams = [], [], []
    for lane in range(2):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            dnn.engine.forward(xs[lane], plan_id=lane)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                out = dnn.engine.forward(xs[lane], plan_id=lane)
        torch.cuda.current_stream().wait_stream(s)
        graphs.append(g); outs.append(out); streams.append(s)
    torch.cuda.synchronize()
    for _ in range(3):
        for g, s in zip(graphs, streams):
            with torch.cuda.stream(s):
                g.replay()
        torch.cuda.synchronize()
        for lane in range(2):
            assert torch.equal(outs[lane], eager[lane]), 'lane %d' % lane
