"""The photometric chain of transform/image.py (RandomBlur, BGR2HSV, RandomHue, RandomSaturation, RandomBrightness, HSV2RGB, RandomGamma)
against tests/golden/photometric.npz, made by executing the reference's classes with cv2 4.13.

CPU: the numpy restatement (tests/photometric_oracle.py) reproduces every stored SHA-256, the full 2^24 colour cube both ways included;
the host draws equal the reference's; the chain compiler's segments; the blur's kernel limit.
GPU: every op alone, both colour conversions over the cube, chains in the reference's order and another one over batches of 8 at 416²,
608², 97x131, 1x53 and 61x1, the per-image mirrors, `Collate` into one training step, and a CUDA-graph replay with new draws."""
import configparser
import hashlib
import os
import random

import numpy as np
import pytest
import torch

import photometric_oracle as P
from oracle import yolo2_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_OP = dict(RandomBlur='blur', BGR2HSV='bgr2hsv', HSV2RGB='hsv2rgb', BGR2RGB='bgr2rgb', RandomHue='hue', RandomSaturation='saturation',
                 RandomBrightness='brightness', RandomGamma='gamma')
N_DRAWS = dict(RandomBlur=2, RandomHue=1, RandomSaturation=1, RandomBrightness=1, RandomGamma=1)
CANONICAL = ['RandomBlur', 'BGR2HSV', 'RandomHue', 'RandomSaturation', 'RandomBrightness', 'HSV2RGB', 'RandomGamma']


@pytest.fixture(scope='module')
def g():
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'photometric.npz'))


def sha(a):
    a = a.cpu().numpy() if torch.is_tensor(a) else a
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def config(g=None):
    c = configparser.ConfigParser()
    aug = dict(s.split('=') for s in g['augmentation']) if g is not None else {}
    c.read_dict({'augmentation': aug})
    return c


def make(cfg, name):
    import transform.image as ti
    cls = getattr(ti, name)
    return cls(cfg) if name.startswith('Random') else cls()


def split_draws(seq, flat):
    """Flat recorded draws of one image -> one draw per op, typed as the host draws them."""
    out, k = [], 0
    for name in seq:
        n = N_DRAWS.get(name, 0)
        if n == 2:
            out.append((int(flat[k]), int(flat[k + 1])))
        elif name == 'RandomHue':
            out.append(int(flat[k]))
        elif n == 1:
            out.append(float(flat[k]))
        else:
            out.append(None)
        k += n
    return out


def flat_draws(draws):
    out = []
    for d in draws:
        if isinstance(d, tuple):
            out += list(d)
        elif d is not None:
            out.append(d)
    return out


def oracle_chain(seq, image, draws):
    for name, d in zip(seq, draws):
        image = P.apply(ORACLE_OP[name], image, d)
    return image


def case(g, name):
    seq = [str(s) for s in g['case_%s_seq' % name]]
    b, h, w, seed = (int(v) for v in g['case_%s_dims' % name])
    frames = [O.synth_frame(1000 * seed + i, h, w) for i in range(b)]
    return seq, seed, frames


# ---------------------------------------------------------------- CPU

def test_oracle_colour_cube_matches_cv2_sha(g):
    cube = P.hsv_cube()
    assert np.array_equal(sha(P.bgr2hsv(cube)), g['cube_bgr2hsv_sha'])
    assert np.array_equal(sha(P.hsv2rgb(cube)), g['cube_hsv2rgb_sha'])
    cube16 = cube.reshape(-1, 16, 3)
    assert np.array_equal(sha(P.bgr2hsv(cube16)), g['cube16_bgr2hsv_sha'])
    assert np.array_equal(sha(P.hsv2rgb(cube16)), g['cube16_hsv2rgb_sha'])


def test_oracle_blur_matches_cv2_sha(g):
    for f, ((h, w), seed) in enumerate(zip(g['blur_frames'], g['blur_seeds'])):
        src = O.synth_frame(int(seed), int(h), int(w))
        for kw in range(1, P.BLUR_MAX + 1):
            for kh in range(1, P.BLUR_MAX + 1):
                assert np.array_equal(sha(P.blur(src, kw, kh)), g['blur_sha'][f, kw - 1, kh - 1]), (h, w, kw, kh)


def test_oracle_ops_and_chains_match_cv2_sha(g):
    for name in g['alone']:
        name = str(name)
        src = O.synth_frame(int(g['alone_%s_seed' % name]), 61, 83)
        for k in range(4):
            d = split_draws([name], g['alone_%s_draws' % name][k])
            assert np.array_equal(sha(oracle_chain([name], src, d)), g['alone_%s_sha' % name][k]), name
    for name in g['cases']:
        seq, _, frames = case(g, name)
        for i, f in enumerate(frames):
            d = split_draws(seq, g['case_%s_draws' % name][i])
            assert np.array_equal(sha(oracle_chain(seq, f, d)), g['case_%s_sha' % name][i]), (name, i)


def test_host_draws_equal_reference_draws(g):
    import transform.image as ti
    cfg = config(g)
    for name in g['alone']:
        name = str(name)
        op = make(cfg, name)
        random.seed(int(g['alone_%s_seed' % name]))
        for k in range(4):
            got = flat_draws([op.draw()]) or [0]
            assert got == g['alone_%s_draws' % name][k].tolist(), name
    for name in g['cases']:
        seq, seed, frames = case(g, name)
        chain = ti.Compose([make(cfg, n) for n in seq])
        random.seed(seed)
        draws = chain.draw(len(frames))
        assert [flat_draws(d) for d in draws] == g['case_%s_draws' % name].tolist(), name


def test_chain_compiler_segments(g):
    import transform
    import transform.image as ti
    import utils.data as ud
    cfg = config(g)
    canon = transform.get_transform(cfg, ['transform.image.' + n for n in CANONICAL])
    assert [[code for code, _ in s] for s in canon.segments] == [[ti.BLUR, ti.HSV, ti.LUT, ti.RGB, ti.LUT]]
    assert canon.segments[0][2][1] == [2, 3, 4] and not canon.swap_only
    other = ti.Compose([make(cfg, str(n)) for n in g['case_other416_seq']])
    assert [[code for code, _ in s] for s in other.segments] == [[ti.LUT, ti.HSV, ti.LUT, ti.RGB], [ti.BLUR, ti.LUT, ti.SWAP]]
    swap = transform.get_transform(cfg, ['transform.image.BGR2RGB'])
    assert swap.swap_only
    collate = ud.Collate([(64, 64)], transform_image=swap)
    assert collate.bgr2rgb and collate.transform_image is None
    # two tables in a row merge; a long chain splits at the per-launch limits
    long = ti.Compose([ti.BGR2HSV(), ti.HSV2RGB()] * 4)
    assert [len(s) for s in long.segments] == [7, 1]
    # composed tables: hue then saturation then brightness on channels 0 / 1 / 2, gamma on all
    draws = [(3, 2), None, 11, 1.3, 0.7, None, 1.2]
    tab = canon.params([draws])[0][0, 16:16 + 768].reshape(3, 256)
    assert np.array_equal(tab[0], P.hue_lut(11)) and np.array_equal(tab[1], P.scale_lut(1.3)) and np.array_equal(tab[2], P.scale_lut(0.7))
    assert canon.params([draws])[0][0, :8].view(np.int32).tolist() == [3, 2]


def test_blur_beyond_the_pinned_kernels_raises():
    import transform.image as ti
    c = configparser.ConfigParser()
    for bad in ('6 5', '5 7', '0 3', '5'):
        c.read_dict({'augmentation': {'random_blur': bad}})
        with pytest.raises(ValueError):
            ti.RandomBlur(c)
    c.read_dict({'augmentation': {'random_blur': '5 5'}})
    assert ti.RandomBlur(c).adjust == (5, 5)
    with pytest.raises(ValueError):
        P.blur(np.zeros((4, 4, 3), np.uint8), 6, 1)


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
def test_each_op_alone_bit_exact(g):
    cfg = config(g)
    for name in g['alone']:
        name = str(name)
        op = make(cfg, name)
        src = O.synth_frame(int(g['alone_%s_seed' % name]), 61, 83)
        random.seed(int(g['alone_%s_seed' % name]))
        for k in range(4):
            out = op(src) if name != 'BGR2RGB' else op(torch.from_numpy(src).cuda()).contiguous()
            assert out.is_cuda and np.array_equal(sha(out), g['alone_%s_sha' % name][k]), (name, k)


def blur_params(kw, kh, batch=1):
    p = np.zeros((batch, 16), np.uint8)
    p[:, :8] = np.frombuffer(np.array([kw, kh], np.int32).tobytes(), np.uint8)
    return torch.from_numpy(p).cuda()


@pytest.mark.gpu
def test_every_blur_kernel_on_device(g):
    """The device blur alone, for every kernel 1..5 x 1..5 on every stored frame (1 x 37, 29 x 1, 1 x 1, 2 x 3, 33 x 45, 17 x 608): the
    1 x 1 copy, the fixed-point divide with its area-2 overflow in the body and the tail of a row, and the exact area-25 divide."""
    import transform.image as ti
    for f, ((h, w), seed) in enumerate(zip(g['blur_frames'], g['blur_seeds'])):
        x = torch.from_numpy(O.synth_frame(int(seed), int(h), int(w))).cuda()[None]
        for kw in range(1, P.BLUR_MAX + 1):
            for kh in range(1, P.BLUR_MAX + 1):
                out = ti.launch(x, torch.empty_like(x), [(ti.BLUR, [0])], blur_params(kw, kh))
                assert np.array_equal(sha(out[0]), g['blur_sha'][f, kw - 1, kh - 1]), (int(h), int(w), kw, kh)


@pytest.mark.gpu
def test_blur_kernel_size_is_clamped_on_device():
    """A parameter block with a kernel size outside 1..5 is clamped into it on the device, not used to index shared memory."""
    import transform.image as ti
    x = torch.from_numpy(O.synth_frame(70, 40, 70)).cuda()[None]
    seg = [(ti.BLUR, [0])]
    for bad, good in (((0, 9), (1, 5)), ((-3, 2), (1, 2)), ((64, 7), (5, 5))):
        assert torch.equal(ti.launch(x, torch.empty_like(x), seg, blur_params(*bad)), ti.launch(x, torch.empty_like(x), seg, blur_params(*good)))


@pytest.mark.gpu
def test_colour_cube_both_ways_on_device(g):
    import transform.image as ti
    cube = torch.from_numpy(P.hsv_cube()).cuda()
    for frame, suffix in ((cube, ''), (cube.reshape(-1, 16, 3), '16')):
        assert np.array_equal(sha(ti.BGR2HSV()(frame)), g['cube%s_bgr2hsv_sha' % suffix])
        assert np.array_equal(sha(ti.HSV2RGB()(frame)), g['cube%s_hsv2rgb_sha' % suffix])


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['canon416', 'canon608', 'canon97', 'canon1xn', 'other416', 'other97', 'other1xn'])
def test_chain_batch_bit_exact_and_equals_per_image(g, name):
    import transform.image as ti
    seq, seed, frames = case(g, name)
    chain = ti.Compose([make(config(g), n) for n in seq])
    x = torch.from_numpy(np.stack(frames)).cuda()
    draws = [split_draws(seq, d) for d in g['case_%s_draws' % name]]
    assert len(frames) >= 8 and len(set(map(str, draws))) == len(frames)
    out = chain.batch(x, draws)
    for i in range(len(frames)):
        assert np.array_equal(sha(out[i]), g['case_%s_sha' % name][i]), (name, i)
    random.seed(seed)
    assert torch.equal(chain.batch(x), out)                       # drawing on the host gives the same batch
    random.seed(seed)
    for i, f in enumerate(frames):                                # the single-image mirror, image after image
        assert torch.equal(chain(f), out[i]), (name, i)


@pytest.mark.gpu
def test_collate_with_image_train_chain_drives_a_training_step(g):
    import model
    import model.yolo2
    import train as yb_train
    import transform
    import utils.data as ud
    cfg = config(g)
    chain = transform.get_transform(cfg, ['transform.image.' + n for n in CANONICAL])
    samples = []
    for i, (h, w, n) in enumerate(((90, 120, 2), (75, 100, 1), (64, 64, 3), (120, 80, 2))):
        r = np.random.RandomState(60 + i)
        lo = (r.rand(n, 2) * [h * 0.5, w * 0.5]).astype(np.float32)
        samples.append(dict(image=O.synth_frame(30 + i, h, w), yx_min=lo, yx_max=lo + (r.rand(n, 2) * [h * 0.4, w * 0.4] + 4).astype(np.float32),
                            cls=r.randint(0, 20, n)))
    collate = ud.Collate([(96, 96)], seed=1, transform_image=chain)
    random.seed(7)
    batch = collate(samples)
    random.seed(7)
    draws = chain.draw(len(samples))
    for i, smp in enumerate(samples):
        ref = oracle_chain(CANONICAL, O.resize_u8(smp['image'], 96, 96), draws[i])
        assert np.array_equal(batch['tensor'][i].cpu().numpy(), ref), i
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'threshold': '0.6'}, 'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()},
                   'train': {'cross_entropy': '1'}})
    anchors = O.anchors_yolo_voc()
    dnn = model.yolo2.Darknet(model.ConfigChannels(cfg), anchors, 20)
    dnn.load_state_dict(O.make_state_dict(0), strict=False)
    dnn = dnn.to('cuda').train()
    inference = model.Inference(cfg, dnn, anchors).train()
    out = yb_train.iterate(inference, torch.optim.SGD(dnn.parameters(), 1e-4), anchors, cfg, batch)
    lt = float(out['loss_total'].item())
    assert lt == lt and 0.0 < lt < 10.0


@pytest.mark.gpu
def test_graph_replay_with_new_draws_equals_eager(g):
    import transform.image as ti
    chain = ti.Compose([make(config(g), n) for n in CANONICAL])
    seq, seed, frames = case(g, 'canon97')
    x = torch.from_numpy(np.stack(frames)).cuda()
    seg = chain.segments[0]
    random.seed(11)
    p_a, p_b = chain.params(chain.draw(len(frames)))[0], chain.params(chain.draw(len(frames)))[0]
    params = torch.from_numpy(p_a).cuda()
    dst = torch.empty_like(x)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        ti.launch(x, dst, seg, params)                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ti.launch(x, dst, seg, params)
    params.copy_(torch.from_numpy(p_b))
    graph.replay()
    torch.cuda.synchronize()
    eager = ti.launch(x, torch.empty_like(x), seg, torch.from_numpy(p_b).cuda())
    assert torch.equal(dst, eager)
    assert not torch.equal(eager, ti.launch(x, torch.empty_like(x), seg, torch.from_numpy(p_a).cuda()))
