"""The two-consumer conv tile's epilogue (conv_wide_kernel): the last K-block's two row halves retire separately, each consumer
converts a 64-row half with its tile's scale / shift from a shared-memory table, stages it in its 16 KB slice, and a producer-group
thread ships it with TMA stores while the consumer goes on.

Every case writes a channel slice (y_ch_off) of a wider buffer filled with a sentinel: the slice equals the 128 x 128 tile bit for bit
(same K-blocks in the same order, only the partition of M and N differs) and every channel outside it keeps the sentinel.  The cases
cover one, two and many tiles per CTA, 1 and 2 K-blocks per tile, a tile with only its first 64-channel half, ragged last N tiles and
ragged last rows; forced stream-K runs a CTA that dumps one tile's partial sums and then collects and stores another."""
import pytest
import torch

from oracle import yolo2_oracle as O

pytestmark = pytest.mark.gpu

DEV = 'cuda'
SENTINEL = -7.5
PAD_LO, PAD_HI = 24, 16          # sentinel channels below and above the slice


@pytest.fixture(scope='module')
def ops():
    from b200 import ops
    return ops


def rel_err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_unit(ops, b, h, w, cin, cout, k, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=gen)
    wt = torch.randn(cout, cin, k, k, generator=gen) * (2.0 / (cin * k * k)) ** 0.5
    sd = {'u.conv.weight': wt, 'u.bn.weight': torch.rand(cout, generator=gen) + 0.5, 'u.bn.bias': torch.randn(cout, generator=gen) * 0.1,
          'u.bn.running_mean': torch.randn(cout, generator=gen) * 0.1, 'u.bn.running_var': torch.rand(cout, generator=gen) + 0.5}
    scale, shift = ops.bn_fold(*(sd['u.bn.' + n].to(DEV) for n in ('weight', 'bias', 'running_mean', 'running_var')))
    return x, sd, x.to(DEV).permute(0, 2, 3, 1).contiguous().half(), ops.pack_weight_f16(wt.to(DEV)), scale, shift


def wide(ops, sk):
    return ops.conv_force_bn(128) | ops.conv_force_mt(2) | (ops.CONV_FORCE_STREAMK if sk else ops.CONV_NO_STREAMK)


def narrow(ops):
    return ops.conv_force_bn(128) | ops.conv_force_mt(1) | ops.CONV_NO_STREAMK


def run_sliced(ops, x16, w16, scale, shift, flags, workspace=None):
    b, h, w, _ = x16.shape
    cout = w16.shape[0]
    buf = torch.full((b, h, w, PAD_LO + cout + PAD_HI), SENTINEL, dtype=torch.float16, device=DEV)
    ops.conv_bn_act(x16, w16, scale, shift, 0.1, out=buf, y_ch_off=PAD_LO, flags=flags, workspace=workspace)
    assert bool((buf[..., :PAD_LO] == SENTINEL).all()), 'channels below the slice were written'
    assert bool((buf[..., PAD_LO + cout:] == SENTINEL).all()), 'channels above the slice were written'
    return buf[..., PAD_LO:PAD_LO + cout]


def tiles_per_cta(b, h, w, cout):
    tiles = -(-b * h * w // 256) * -(-cout // 128)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return tiles, -(-tiles // sms)


CASES = [
    # b, h, w, cin, cout, k, what the case covers (tiles per CTA on a 132-SM H100)
    (2, 26, 26, 256, 128, 3, 'one tile per CTA (6 tiles), 36 K-blocks'),
    (8, 52, 52, 128, 256, 3, 'two tiles per CTA (170 tiles), both halves'),
    (16, 104, 104, 64, 128, 3, 'many tiles per CTA (676 tiles), 9 K-blocks'),
    (32, 26, 26, 64, 128, 1, 'one K-block per tile (1x1, Cin = 64), 85 tiles'),
    (64, 26, 26, 64, 128, 1, 'one K-block per tile, two tiles per CTA'),
    (64, 26, 26, 128, 128, 1, 'two K-blocks per tile (1x1, Cin = 128), two tiles per CTA'),
    (48, 13, 13, 32, 64, 1, 'one K-block of BK = 32, Cout = 64: only the first half of each tile'),
    (6, 26, 26, 256, 136, 3, 'ragged last N tile: 8 channels'),
    (6, 26, 26, 256, 200, 3, 'ragged last N tile: 72 channels, the second half partly'),
    (3, 13, 13, 512, 1024, 3, 'M = 507: ragged last rows, eight N tiles'),
]


@pytest.mark.parametrize('case', CASES, ids=[c[-1] for c in CASES])
def test_wide_epilogue_equals_narrow_tile(ops, case):
    b, h, w, cin, cout, k, _ = case
    x, sd, x16, w16, scale, shift = make_unit(ops, b, h, w, cin, cout, k, cin + 7 * cout + h)
    ch = ops.conv_choice(b, h, w, cin, cout, k, flags=wide(ops, False))
    assert ch['kernel'] == 'conv_wide_kernel' and not ch['streamk'], ch
    y = run_sliced(ops, x16, w16, scale, shift, wide(ops, False))
    y128 = ops.conv_bn_act(x16, w16, scale, shift, 0.1, flags=narrow(ops))
    assert torch.equal(y, y128), 'two-consumer tile differs from the 128 x 128 tile'
    if b * h * w <= 4096:      # the fp32 oracle on the CPU: small cases only
        ref = O.conv_unit(x, sd, 'u', k, True, True)
        assert rel_err(y.permute(0, 3, 1, 2), ref) <= 1e-3


def test_wide_epilogue_cases_cover_tile_counts():
    """The case list really has one, two and more than two tiles per CTA on this GPU."""
    per_cta = {tiles_per_cta(b, h, w, cout)[1] for b, h, w, _, cout, _, _ in CASES}
    assert {1, 2}.issubset(per_cta) and max(per_cta) > 2, per_cta


def sk_dump_then_collect(units, num_kb, sms):
    """CTAs whose stream-K range ends inside one tile (dumped, processed first) and starts inside an earlier one (collected)."""
    base, rem = divmod(units, sms)
    out = []
    for c in range(sms):
        s = c * base + min(c, rem)
        e = (c + 1) * base + min(c + 1, rem)
        if s % num_kb and e % num_kb and s // num_kb != (e - 1) // num_kb:
            out.append(c)
    return out


@pytest.mark.parametrize('case', [(3, 13, 13, 576, 1024, 3), (12, 19, 17, 96, 200, 3)], ids=['bk64', 'bk32_ragged'])
def test_wide_epilogue_streamk_dump_and_collect(ops, case):
    b, h, w, cin, cout, k = case
    x, sd, x16, w16, scale, shift = make_unit(ops, b, h, w, cin, cout, k, cin + 3 * cout)
    ch = ops.conv_choice(b, h, w, cin, cout, k, flags=wide(ops, True))
    assert ch['kernel'] == 'conv_wide_kernel' and ch['streamk'], ch
    tiles, _ = tiles_per_cta(b, h, w, cout)
    num_kb = k * k * cin // ch['bk']
    assert sk_dump_then_collect(tiles * num_kb, num_kb, ch['grid']), 'no CTA both dumps and collects'
    ws = ops.conv_workspace(DEV)
    y = run_sliced(ops, x16, w16, scale, shift, wide(ops, True), workspace=ws)
    assert int(ws[:4096].view(torch.int32).abs().sum().item()) == 0, 'stream-K flags not reset'
    ref = O.conv_unit(x, sd, 'u', k, True, True)
    assert rel_err(y.permute(0, 3, 1, 2), ref) <= 1e-3
    again = run_sliced(ops, x16, w16, scale, shift, wide(ops, True), workspace=ws)
    assert torch.equal(y, again), 'stream-K launch is not deterministic'
    y0 = run_sliced(ops, x16, w16, scale, shift, wide(ops, False))
    assert rel_err(y, y0) <= 2e-3
