"""Inception-v3 plugin (model.inception3) and the kernels it adds.

CPU: the restatement in inception_oracle.py against the executed reference (inception.npz), the state_dict keys and shapes, the input errors
and the new C entry points in the header and the ctypes table.

GPU: the general-geometry implicit-GEMM conv (yb_conv2d_bn_act_fwd: kh x kw filters, stride 1 / 2, any padding below the filter size) element
by element against float64 on its own fp16 operands with the bound of test_conv_contract.py, on every tile shape yb_conv2d_choice reaches, with
and without forced stream-K; exact relations (the square same-padded form equals yb_conv_bn_act_fwd, valid equals same without its border,
stride 2 equals stride 1 at the selected pixels); refusals; the pools, the weight pack and the stem; the plugin against the reference."""
import configparser
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception_oracle as I
import test_conv_contract as C
from oracle import yolo2_oracle as O

DEV = 'cuda'
gpu = pytest.mark.gpu
MEASURED = {}


def record(name, value):
    """Measured figures of this run -> $YB_PARITY_OUT/inception_measured.json when that directory is given."""
    MEASURED[name] = value
    out = os.environ.get('YB_PARITY_OUT')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'inception_measured.json'), 'w') as f:
            json.dump(MEASURED, f, indent=1, sort_keys=True)


def rel_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def make_config():
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'},
                      'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    return config


def build(seed=0):
    import model
    import model.inception3
    net = model.inception3.Inception3(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    res = net.load_state_dict(I.make_inception_state_dict(seed), strict=False)
    assert not res.unexpected_keys and all(k.endswith('num_batches_tracked') for k in res.missing_keys), res
    return net.eval()


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'inception.npz'))


SIZES = ((75, 75, 1), (107, 139, 2), (416, 416, 0), (320, 608, 3))
GRIDS = {(75, 75): (1, 1), (107, 139): (2, 3), (416, 416): (11, 11), (320, 608): (8, 17)}
BLOCKS = [b[0] for b in I.BLOCKS]


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_restatement_vs_reference_golden(golden):
    sd = I.make_inception_state_dict(0)
    for h, w, seed in SIZES:
        got = {}
        with torch.no_grad():
            f = I.inception_forward(sd, O.synth_images(1, h, w, seed=seed), collect=got)
        ref = torch.from_numpy(golden['feature_%dx%d' % (h, w)])
        assert tuple(ref.shape[-2:]) == GRIDS[(h, w)]
        assert ((f - ref).norm() / ref.norm()).item() < 1e-5, (h, w)
        if (h, w) == (107, 139):
            for k in ['pool1', 'pool2'] + BLOCKS:
                r = torch.from_numpy(golden['act_' + k])
                assert ((got[k] - r).norm() / r.norm()).item() < 1e-5, k


def test_state_dict_keys_and_shapes(golden):
    sd = build().state_dict()
    assert len(sd) == 566 and list(sd.keys())[-2:] == ['conv.weight', 'conv.bias']
    assert list(sd.keys()) == list(golden['keys'])
    assert [','.join(str(d) for d in v.shape) for v in sd.values()] == list(golden['shapes'])
    bns = [m for m in build().modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert bns and all(m.eps == 1e-3 for m in bns)


def test_initialisation_follows_the_reference():
    """model/inception3.py:54-62: conv weights truncated normal on [-0.2, 0.2] with sigma 0.1, BatchNorm weight 1 and bias 0."""
    import model
    import model.inception3
    torch.manual_seed(0)
    net = model.inception3.Inception3(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20)
    w = net.Mixed_7c.branch3x3dbl_2.conv.weight.detach()
    assert float(w.abs().max()) <= 0.2 and abs(float(w.std()) - 0.088) < 0.005      # std of N(0, 0.1) truncated at 2 sigma: 0.0880
    assert bool((net.Mixed_5b.branch1x1.bn.weight == 1).all() and (net.Mixed_5b.branch1x1.bn.bias == 0).all())


def test_input_errors():
    import model
    import model.inception3
    net = build()
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 74, 128))              # Mixed_7a's output would be empty
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 128, 74))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 75, 75))               # CPU tensor: no CPU fallback
    net.train()
    with pytest.raises(NotImplementedError):
        net(torch.zeros(1, 3, 75, 75))
    ti = model.inception3.Inception3(model.ConfigChannels(make_config()), O.anchors_yolo_voc(), 20, transform_input=True).eval()
    with pytest.raises(NotImplementedError):
        ti(torch.zeros(1, 3, 75, 75))


def test_new_entry_points_are_declared():
    from b200 import lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'yolo2_b200.h')).read()
    for name in ('yb_conv2d_bn_act_fwd', 'yb_conv2d_choice', 'yb_pack_weight_khw_f16', 'yb_stem3x3_s2_bn_relu_fwd', 'yb_maxpool3x3_s2_valid_f16',
                 'yb_avgpool3x3_s1_f16'):
        assert name in lib.SIGNATURES and ('int %s(' % name) in header, name


def avg_pool_check(got, ref, E):
    """fp16 avg-pool outputs against a float64 reference: RN16(ref) wherever no fp16 rounding boundary lies within E, else within E + 1/2 ulp."""
    got = C.np64(got)
    bound = E + 0.5 * C.ulp16(np.abs(ref) + E) * (1 + 2.0 ** -10)
    assert (np.abs(got - ref) <= bound).all(), 'avg-pool: outside the bound'
    sure = C.rn16(ref - E) == C.rn16(ref + E)
    assert (got.astype(np.float16)[sure] == C.rn16(ref)[sure]).all(), 'avg-pool: differs from RN16 of the float64 mean'
    return int(sure.sum())


def avg_pool_reference(x, include_pad=True):
    """float64 mean over the 3 x 3 window (NHWC), divisor 9 (count_include_pad) or the number of in-range pixels, and the fp32 error bound
    of a 9-term fp32 sum and one division."""
    xt = torch.from_numpy(C.np64(x)).permute(0, 3, 1, 2)
    s = F.avg_pool2d(xt, 3, 1, 1, count_include_pad=True) * 9
    a = F.avg_pool2d(xt.abs(), 3, 1, 1, count_include_pad=True) * 9
    n = 9.0 if include_pad else F.avg_pool2d(torch.ones_like(xt[:, :1]), 3, 1, 1, count_include_pad=True) * 9     # in-range pixels
    ref = (s / n).permute(0, 2, 3, 1).numpy()
    E = ((10 * C.U) * a / 9).permute(0, 2, 3, 1).numpy() + C.U * np.abs(ref)
    return ref, E


def test_avg_pool_rule_rejects_count_exclude_pad():
    """The avg-pool check accepts RN16 of the divisor-9 mean and rejects the count_include_pad=False mean at the borders."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 7, 9, 16, generator=g).half()
    ref, E = avg_pool_reference(x)
    avg_pool_check(C.rn16(ref), ref, E)
    bad, _ = avg_pool_reference(x, include_pad=False)
    with pytest.raises(AssertionError):
        avg_pool_check(C.rn16(bad), ref, E)


# ------------------------------------------------------------------------------------------------
# GPU: the general-geometry conv
# ------------------------------------------------------------------------------------------------
# (name, kh, kw, stride, pad_h, pad_w)
GEOMS = {'1x7': (1, 7, 1, 0, 3), '7x1': (7, 1, 1, 3, 0), '1x3': (1, 3, 1, 0, 1), '3x1': (3, 1, 1, 1, 0), '5x5': (5, 5, 1, 2, 2),
         '3x3v': (3, 3, 1, 0, 0), '3x3v_s2': (3, 3, 2, 0, 0), '3x3_s2': (3, 3, 2, 1, 1), '1x1_s2': (1, 1, 2, 0, 0)}
# (geometry, b, h, w, cin, cout): Inception's own shapes at 416 x 416 (sides 207, 102, 49, 24, 11; Cin 32 / 96 / 64 as the plugin pads them)
# and ragged ones (one pixel high / wide, an image smaller than one tile, odd sides under stride 2)
CASES = [
    ('3x3v', 1, 207, 207, 32, 32),         # Conv2d_2a_3x3
    ('3x3v', 2, 102, 102, 96, 192),        # Conv2d_4a_3x3 (Cin 80 + 16 zero channels)
    ('5x5', 2, 49, 49, 64, 64),            # branch5x5_2 (Cin 48 + 16)
    ('3x3v_s2', 2, 49, 49, 288, 384),      # Mixed_6a.branch3x3
    ('1x7', 2, 24, 24, 128, 160),          # Mixed_6b..e
    ('7x1', 2, 24, 24, 160, 192),
    ('3x3v_s2', 2, 24, 24, 192, 320),      # Mixed_7a.branch3x3_2
    ('1x3', 2, 11, 11, 384, 384),          # Mixed_7b / 7c
    ('3x1', 2, 11, 11, 384, 384),
    ('1x7', 3, 1, 37, 64, 72),
    ('7x1', 3, 37, 1, 64, 72),
    ('5x5', 1, 7, 9, 64, 40),
    ('3x3v_s2', 1, 9, 7, 96, 24),
    ('3x3_s2', 2, 13, 11, 64, 128),
    ('1x1_s2', 2, 13, 11, 128, 64),
]


def case_id(c):
    return '%s_%dx%dx%d_%d-%d' % c


def conv_inputs(case):
    geom, b, h, w, cin, cout = case
    kh, kw, _, _, _ = GEOMS[geom]
    g = torch.Generator().manual_seed(b * 1000003 + h * 1009 + w * 101 + cin * 7 + cout + kh * 13 + kw)
    x = torch.randn(b, cin, h, w, generator=g).half()
    wt = torch.randn(cout, cin, kh, kw, generator=g) * (2.0 / (cin * kh * kw)) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5
    scale[1::3] *= -1
    shift = torch.randn(cout, generator=g) * 0.1
    return x, wt, scale, shift


def conv_reference(case, x, wt):
    kh, kw, stride, ph, pw = GEOMS[case[0]]
    dev = C.ref_device()
    xd, wd = x.double().to(dev), wt.half().double().to(dev)
    return C.np64(F.conv2d(xd, wd, None, stride, (ph, pw))), C.np64(F.conv2d(xd.abs(), wd.abs(), None, stride, (ph, pw)))


@gpu
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_general_conv_vs_float64(case):
    from b200 import ops
    geom, b, h, w, cin, cout = case
    kh, kw, stride, ph, pw = GEOMS[geom]
    x, wt, scale, shift = conv_inputs(case)
    acc, S = conv_reference(case, x, wt)
    oh, ow = acc.shape[2:]
    x16 = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    w16 = ops.pack_weight_khw_f16(wt.to(DEV))
    sc, sh = scale.to(DEV), shift.to(DEV)
    ws = ops.conv_workspace(DEV)
    K, bk = kh * kw * cin, 64 if cin % 64 == 0 else 32
    num_kb = kh * kw * (cin // bk)
    m_total = b * oh * ow
    slope = 0.1
    taken = []
    for name, bn, mt in C.FORMS:
        wide = bn * mt > 128
        for sk in (False, True):
            flags = C.form_flags(ops, bn, mt, sk)
            ch = ops.conv2d_choice(b, h, w, cin, cout, kh, kw, stride, (ph, pw), flags=flags, workspace=sk)
            if sk and not ch['streamk']:
                continue
            want = dict(kernel='conv_wide_kernel' if wide else 'conv_igemm_kernel', bk=bk, bn=bn, rows=128 * mt, streamk=sk)
            assert {q: ch[q] for q in want} == want, (flags, ch, want)
            taken.append(name + ('+sk' if sk else ''))
            P = C.sk_partials(m_total, 128 * mt, cout, bn, num_kb) if sk else 1
            ref, E = C.epilogue(acc, S, K, P, scale, shift, slope)
            group = 'conv2d_%s%s' % (name, '_sk' if sk else '')
            kwargs = dict(stride=stride, pad=(ph, pw), flags=flags, workspace=ws if sk else None)
            buf = C.sentinel((b, oh, ow, cout + 24))
            ops.conv2d_bn_act(x16, w16, sc, sh, slope, out=buf, y_ch_off=8, **kwargs)
            C.check_f16('%s %s' % (group, geom), C.nchw(buf[..., 8:8 + cout]), ref, E, group)
            assert bool((C.bits(buf[..., :8]) == C.SENTINEL).all()) and bool((C.bits(buf[..., 8 + cout:]) == C.SENTINEL).all()), \
                '%s: wrote outside its channel slice' % group
            if sk:
                torch.cuda.synchronize()
                assert int(ws[:4096].view(torch.int32).abs().sum()) == 0, 'stream-K flags not reset'
            if not wide:
                y32 = ops.conv2d_bn_act(x16, w16, sc, sh, slope, out_mode=ops.OUT_F32_NCHW, **kwargs)
                C.check_f32('%s fp32 %s' % (group, geom), y32, ref, E, group + '_f32')
    record('forms_%s' % case_id(case), taken)


def _square_operands(g, b, h, w, cin, cout, k):
    x = torch.randn(b, h, w, cin, generator=g).half().to(DEV)
    wt = (torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5).to(DEV)
    return x, wt, (torch.rand(cout, generator=g) + 0.5).to(DEV), (torch.randn(cout, generator=g) * 0.1).to(DEV)


@gpu
def test_square_same_form_is_yb_conv_bn_act_fwd():
    """(k, k, stride 1, pad (k-1)/2) through the new entry gives the bits of yb_conv_bn_act_fwd(_ws), with the same kernel choice."""
    from b200 import ops
    g = torch.Generator().manual_seed(21)
    ws = ops.conv_workspace(DEV)
    for b, h, w, cin, cout, k in ((3, 11, 13, 96, 136, 3), (2, 13, 13, 512, 1024, 3), (5, 13, 13, 1024, 200, 1), (2, 16, 8, 32, 48, 3),
                                  (32, 13, 13, 1024, 1024, 3)):
        x, wt, sc, sh = _square_operands(g, b, h, w, cin, cout, k)
        w16 = ops.pack_weight_f16(wt)
        assert torch.equal(ops.pack_weight_khw_f16(wt), w16)
        p = (k - 1) // 2
        for flags, wsp in ((0, None), (0, ws), (ops.CONV_FORCE_STREAMK, ws)):
            assert ops.conv2d_choice(b, h, w, cin, cout, k, k, 1, (p, p), flags=flags, workspace=wsp is not None) == \
                ops.conv_choice(b, h, w, cin, cout, k, flags=flags, workspace=wsp is not None)
            y = ops.conv2d_bn_act(x, w16, sc, sh, 0.1, stride=1, pad=(p, p), flags=flags, workspace=wsp)
            yr = ops.conv_bn_act(x, w16, sc, sh, 0.1, flags=flags, workspace=wsp)
            assert torch.equal(C.bits(y), C.bits(yr)), (b, h, w, cin, cout, k, flags)
        y32 = ops.conv2d_bn_act(x, w16, sc, sh, 1.0, stride=1, pad=(p, p), out_mode=ops.OUT_F32_NCHW)
        assert torch.equal(y32, ops.conv_bn_act(x, w16, sc, sh, 1.0, out_mode=ops.OUT_F32_NCHW))


@gpu
def test_valid_and_stride2_are_selections_of_the_same_padded_conv():
    """Same operands, same K order per output: 3x3 valid = same-padded without its one-pixel border; stride 2 = stride 1 at the even pixels
    (pad 1) or at pixels 2i of the valid output (pad 0); for every tile shape without stream-K."""
    from b200 import ops
    g = torch.Generator().manual_seed(22)
    for b, h, w, cin, cout in ((2, 24, 24, 192, 320), (1, 49, 47, 288, 384), (3, 9, 7, 64, 40), (1, 207, 207, 32, 32)):
        x, wt, sc, sh = _square_operands(g, b, h, w, cin, cout, 3)
        w16 = ops.pack_weight_khw_f16(wt)
        for name, bn, mt in C.FORMS:
            flags = C.form_flags(ops, bn, mt, False) | ops.CONV_NO_SMALLK
            same = ops.conv2d_bn_act(x, w16, sc, sh, 0.1, stride=1, pad=(1, 1), flags=flags)
            valid = ops.conv2d_bn_act(x, w16, sc, sh, 0.1, stride=1, pad=(0, 0), flags=flags)
            assert torch.equal(C.bits(valid), C.bits(same[:, 1:-1, 1:-1])), (b, h, w, name, 'valid')
            s2 = ops.conv2d_bn_act(x, w16, sc, sh, 0.1, stride=2, pad=(1, 1), flags=flags)
            assert torch.equal(C.bits(s2), C.bits(same[:, ::2, ::2])), (b, h, w, name, 'stride 2, pad 1')
            s2v = ops.conv2d_bn_act(x, w16, sc, sh, 0.1, stride=2, pad=(0, 0), flags=flags)
            assert torch.equal(C.bits(s2v), C.bits(valid[:, ::2, ::2])), (b, h, w, name, 'stride 2, pad 0')


@gpu
def test_general_conv_refusals_leave_the_output_untouched():
    from b200 import ops
    g = torch.Generator().manual_seed(23)
    x = torch.randn(1, 9, 9, 96, generator=g).half().to(DEV)
    x80 = torch.randn(1, 9, 9, 80, generator=g).half().to(DEV)
    sc, sh = torch.ones(64, device=DEV), torch.zeros(64, device=DEV)
    lib = ops._l.load()
    for kh, kw, stride, ph, pw, h, w, xin in ((0, 3, 1, 0, 0, 9, 9, x), (8, 3, 1, 0, 0, 9, 9, x), (3, 8, 1, 0, 0, 9, 9, x), (3, 3, 3, 0, 0, 9, 9, x),
                                              (3, 3, 1, 3, 0, 9, 9, x), (1, 3, 1, 0, 3, 9, 9, x), (7, 7, 1, 0, 0, 6, 9, x), (3, 3, 1, 1, 1, 9, 9, x80)):
        cin = xin.shape[-1]
        wt = torch.zeros(64, max(kh, 1), max(kw, 1), cin, dtype=torch.float16, device=DEV)
        y = C.sentinel((1, 9, 9, 64))
        rc = lib.yb_conv2d_bn_act_fwd(ops._p(xin), ops._p(wt), ops._p(sc), ops._p(sh), 0.0, ops._p(y), 1, h, w, cin, 64, kh, kw, stride, ph, pw, cin, 64,
                                      0, 0, 0, None, 0, ops._s())
        assert rc == -1, (kh, kw, stride, ph, pw, h, w, cin, rc)
        out = (ctypes.c_int * 6)()
        assert lib.yb_conv2d_choice(1, h, w, cin, 64, kh, kw, stride, ph, pw, 0, 0, 0, ctypes.byref(out)) == -1
        torch.cuda.synchronize()
        assert bool((C.bits(y) == C.SENTINEL).all()), (kh, kw, stride, ph, pw)


# ------------------------------------------------------------------------------------------------
# GPU: pools, pack, stem
# ------------------------------------------------------------------------------------------------
@gpu
def test_maxpool_and_pack_bit_exact():
    from b200 import ops
    g = torch.Generator().manual_seed(24)
    for b, h, w, c, ld, off in ((2, 205, 205, 64, 64, 0), (2, 100, 100, 192, 192, 0), (2, 49, 49, 288, 768, 480), (1, 24, 24, 768, 1280, 512),
                                (3, 3, 4, 8, 24, 8)):
        x = torch.randn(b, h, w, c, generator=g).half().to(DEV)
        oh, ow = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        y = C.sentinel((b, oh, ow, ld))
        ops.maxpool3x3_s2_valid(x, y, off)
        ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
        assert torch.equal(C.bits(y[..., off:off + c]), C.bits(ref)), (b, h, w, c)
        assert bool((C.bits(y[..., :off]) == C.SENTINEL).all() and (C.bits(y[..., off + c:]) == C.SENTINEL).all())
    for cout, cin, kh, kw, cp, cip in ((80, 64, 1, 1, 96, 64), (192, 80, 3, 3, 192, 96), (64, 48, 5, 5, 64, 64), (160, 160, 1, 7, 160, 160),
                                       (192, 160, 7, 1, 192, 160), (125, 2048, 1, 1, 125, 2048), (384, 384, 3, 1, 384, 384)):
        wt = torch.randn(cout, cin, kh, kw, generator=g).to(DEV)
        got = ops.pack_weight_khw_f16(wt, cp, cip)
        ref = torch.zeros(cp, kh, kw, cip, dtype=torch.float16, device=DEV)
        ref[:cout, :, :, :cin] = wt.half().permute(0, 2, 3, 1)
        assert torch.equal(C.bits(got), C.bits(ref)), (cout, cin, kh, kw)


@gpu
def test_avg_pool_vs_float64_mean():
    from b200 import ops
    g = torch.Generator().manual_seed(25)
    exact = 0
    for b, h, w, c in ((2, 49, 49, 192), (2, 24, 24, 768), (2, 11, 11, 1280), (1, 1, 5, 8), (3, 2, 1, 16)):
        x = (torch.randn(b, h, w, c, generator=g) * 3).half()
        y = ops.avgpool3x3_s1(x.to(DEV))
        ref, E = avg_pool_reference(x)
        exact += avg_pool_check(y, ref, E)
        if h > 1 and w > 1:
            bad, _ = avg_pool_reference(x, include_pad=False)
            with pytest.raises(AssertionError):
                avg_pool_check(y, bad, E)
    record('avgpool_exact_elements', exact)


@gpu
def test_stem_vs_float64_and_pad1_is_mobilenet_conv0():
    from b200 import ops
    g = torch.Generator().manual_seed(26)
    for b, h, w in ((2, 416, 416), (1, 107, 139), (3, 75, 75), (1, 3, 4)):
        x = torch.rand(b, 3, h, w, generator=g)
        wt = torch.randn(32, 3, 3, 3, generator=g) * 0.3
        scale, shift = torch.rand(32, generator=g) + 0.5, torch.randn(32, generator=g) * 0.1
        y = ops.stem3x3_s2(x.to(DEV), wt.to(DEV), scale.to(DEV), shift.to(DEV), pad=0)
        acc = C.np64(F.conv2d(x.double(), wt.double(), None, 2))
        S = C.np64(F.conv2d(x.double().abs(), wt.double().abs(), None, 2))
        # a chain of 27 fp32 fmaf: K = 16 * 27 gives acc_bound = (2 * 27 + 3) ulps of S, more than the chain's 27 roundings
        ref, E = C.epilogue(acc, S, 16 * 27, 1, scale, shift, 0.0)
        C.check_f16('stem %dx%d' % (h, w), C.nchw(y), ref, E, 'stem')
        if h % 2 == 0 and w % 2 == 0:
            y1 = ops.stem3x3_s2(x.to(DEV), wt.to(DEV), scale.to(DEV), shift.to(DEV), pad=1)
            ym = torch.empty(b, h // 2, w // 2, 32, dtype=torch.float16, device=DEV)
            ops.call('yb_mb_conv0_bn_relu_fwd', x.to(DEV), wt.to(DEV), scale.to(DEV), shift.to(DEV), ym, b, h, w)
            assert torch.equal(C.bits(y1), C.bits(ym)), (b, h, w)


# ------------------------------------------------------------------------------------------------
# GPU: plugin
# ------------------------------------------------------------------------------------------------
TOL_E2E = 3e-3
TOL_BLOCK = 2e-3


@gpu
def test_plugin_vs_reference_golden(golden):
    net = build().to(DEV)
    rec = {}
    with torch.no_grad():
        for h, w, seed in SIZES[:3]:
            f = net(O.synth_images(1, h, w, seed=seed).to(DEV))
            assert tuple(f.shape) == (1, 125) + GRIDS[(h, w)]
            rec['feature_%dx%d' % (h, w)] = rel_err(f, torch.from_numpy(golden['feature_%dx%d' % (h, w)]))
        acts = {}
        net.run(O.synth_images(1, 107, 139, seed=2).to(DEV), collect=acts)
        for k, v in acts.items():
            rec['act_' + k] = rel_err(v.permute(0, 3, 1, 2), torch.from_numpy(golden['act_' + k]))
    record('golden', rec)
    assert all(v <= TOL_E2E for v in rec.values()), rec


@gpu
def test_each_block_fed_oracle_input():
    """Every Mixed_* block at 107 x 139, fed the oracle's own (fp16-rounded) input: its concatenated output vs the oracle."""
    net = build().to(DEV)
    sd = I.make_inception_state_dict(0)
    acts = {}
    with torch.no_grad():
        I.inception_forward(sd, O.synth_images(1, 107, 139, seed=2), collect=acts)
    rec = {}
    with torch.no_grad():
        prev = 'pool2'
        for name in BLOCKS:
            x = acts[prev].permute(0, 2, 3, 1).contiguous().half().to(DEV)
            ref = I.block_forward(sd, acts[prev].half().float(), name)
            rec[name] = rel_err(net.block(name, x).permute(0, 3, 1, 2), ref)
            prev = name
    record('blocks', rec)
    assert all(v <= TOL_BLOCK for v in rec.values()), rec


def _oracle_on_gpu(sd, x):
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return I.inception_forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@gpu
def test_batch32_vs_oracle():
    net = build().to(DEV)
    sd = I.make_inception_state_dict(0)
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
def test_inference_reload_graph_and_postprocess():
    import detect
    import model
    net = build().to(DEV)
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
        net(x)
        net.load_state_dict(I.make_inception_state_dict(1), strict=False)
        y1 = net(x)
        y_fresh = build(1).to(DEV)(x)
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
    static_x.copy_(O.synth_images(2, 107, 139, seed=6).to(DEV))
    graph.replay()
    with torch.no_grad():
        eager = net(static_x)
    torch.cuda.synchronize()
    assert torch.equal(static_y, eager)


def test_selectable_from_config():
    """`[model] dnn = model.inception3.Inception3` resolves through utils.parse_attr, as the reference's callers do."""
    import utils
    import model.inception3
    assert utils.parse_attr('model.inception3.Inception3') is model.inception3.Inception3
