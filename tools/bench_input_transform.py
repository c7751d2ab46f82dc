#!/usr/bin/env python
"""The input transform (transform.TensorTransform through the backbones' first-layer `_lut` kernels) on one GPU at batch 32, 416x416.
Prints ONE JSON line with:

  first_layer   per backbone: its first-layer kernel alone on the fp32 NCHW image against uint8 NHWC frames + the (0.5, 1) table, and
                for Darknet also the uint8 1/255 form (yb_conv0_u8_bn_leaky_pool_fwd), in microseconds per launch
  forward       per backbone: the eval forward from the fp32 image ('fp32'), from uint8 frames through the table in the first layer
                ('fused'), and t(frames) followed by the fp32 forward ('separate'), in milliseconds per batch
  pipeline      Darknet's DetectPipeline(uint8_input=True), graph replays, images/s with the (0.5, 1) transform and without one
and the card's name, power limit and SM clocks read in the same run (nvidia-smi query).  Every number is the median over --rounds rounds
in which the variants of one comparison run alternately, each round timed with CUDA events over --iters calls after a warm-up; the min and
max of the rounds are given as the spread.

    python tools/bench_input_transform.py [--iters 20] [--rounds 7]

Writes nothing to the source tree.
"""
import argparse
import configparser
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, 'yolo2-pytorch_b200'), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

B, H, W = 32, 416, 416
BACKBONES = ['darknet', 'tiny', 'mobilenet', 'resnet18', 'resnet50', 'densenet121', 'inception3', 'inception4', 'vgg16_bn']


def gpu_info():
    q = 'name,power.limit,clocks.max.sm,clocks.sm'
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True)
    vals = [v.strip() for v in r.stdout.strip().split(',')] if r.returncode == 0 else []
    return dict(zip(q.split(','), vals)) if len(vals) == 4 else dict(error=r.stderr.strip())


def build(name):
    import torch
    import model
    import model.densenet
    import model.inception3
    import model.inception4
    import model.mobilenet
    import model.resnet
    import model.vgg
    import model.yolo2
    from oracle import yolo2_oracle as O
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'},
                   'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    anchors = O.anchors_yolo_voc()
    torch.manual_seed(0)
    cc = model.ConfigChannels(cfg)
    ctor = {'darknet': model.yolo2.Darknet, 'tiny': model.yolo2.Tiny, 'mobilenet': model.mobilenet.MobileNet,
            'resnet18': model.resnet.resnet18, 'resnet50': model.resnet.resnet50, 'densenet121': model.densenet.densenet121,
            'inception3': model.inception3.Inception3, 'inception4': model.inception4.Inception4, 'vgg16_bn': model.vgg.vgg16_bn}[name]
    net = ctor(cc, anchors, 20)
    if name == 'darknet':
        net.load_state_dict(O.make_state_dict(0), strict=False)
    return net.cuda().eval(), anchors, cfg


def first_layer(name, net, x_u8, x_f32, lut):
    """(fp32 call, table call[, 1/255 call]) of the backbone's first-layer kernel with its own operands."""
    import torch
    from b200 import ops
    b, h, w = x_u8.shape[:3]
    g = torch.Generator().manual_seed(1)

    def rnd(*shape):
        return torch.randn(*shape, generator=g).cuda()
    if name in ('darknet', 'tiny'):
        wt, s, t = rnd(32, 3, 3, 3), rnd(32), rnd(32)
        out = torch.empty(b, h // 2, w // 2, 32, dtype=torch.float16, device='cuda')
        calls = {'fp32': lambda: ops.conv0_bn_leaky_pool(x_f32, wt, s, t, 0.1, out=out),
                 'u8_lut': lambda: ops.conv0_bn_leaky_pool(x_u8, wt, s, t, 0.1, out=out, lut=lut)}
        if name == 'darknet':
            calls['u8_scale'] = lambda: ops.conv0_u8_bn_leaky_pool(x_u8, wt, s, t, 0.1, out=out)
        return calls
    if name == 'vgg16_bn':
        wt, s, t = rnd(64, 3, 3, 3), rnd(64), rnd(64)
        out = torch.empty(b, h, w, 64, dtype=torch.float16, device='cuda')
        return {'fp32': lambda: ops.conv0_c64_bn_act(x_f32, wt, s, t, 0.0, out=out),
                'u8_lut': lambda: ops.conv0_c64_bn_act(x_u8, wt, s, t, 0.0, out=out, lut=lut)}
    if name.startswith('inception'):
        wt, s, t = rnd(32, 3, 3, 3), rnd(32), rnd(32)
        return {'fp32': lambda: ops.stem3x3_s2(x_f32, wt, s, t, pad=0), 'u8_lut': lambda: ops.stem3x3_s2(x_u8, wt, s, t, pad=0, lut=lut)}
    if name == 'mobilenet':
        wt, s, t = rnd(32, 3, 3, 3), rnd(32), rnd(32)
        out = torch.empty(b, h // 2, w // 2, 32, dtype=torch.float16, device='cuda')
        return {'fp32': lambda: ops.call('yb_mb_conv0_bn_relu_fwd', x_f32, wt, s, t, out, b, h, w),
                'u8_lut': lambda: ops.call('yb_mb_conv0_bn_relu_lut_fwd', x_u8, lut, wt, s, t, out, b, h, w)}
    wt, s, t = rnd(64, 3, 7, 7), rnd(64), rnd(64)
    out = torch.empty(b, h // 2, w // 2, 64, dtype=torch.float16, device='cuda')
    return {'fp32': lambda: ops.call('yb_stem7x7_bn_relu_fwd', x_f32, wt, s, t, out, b, h, w),
            'u8_lut': lambda: ops.call('yb_stem7x7_bn_relu_lut_fwd', x_u8, lut, wt, s, t, out, b, h, w)}


def alternate(calls, iters, rounds, scale):
    """{variant: (median, min, max)} of the per-call time (ms * scale), the variants alternated round by round."""
    import torch
    for fn in calls.values():                 # warm-up: module loads, attributes, lazy allocations, operand packing
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(rounds):
        for k, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / iters * scale)
    return {k: dict(median=round(statistics.median(v), 3), min=round(min(v), 3), max=round(max(v), 3)) for k, v in times.items()}


def pipeline(iters, rounds):
    import torch
    import model
    import transform
    import torchvision.transforms as T
    from b200.pipeline import DetectPipeline
    net, anchors, cfg = build('darknet')
    inference = model.Inference(cfg, net, anchors).eval()
    frames = torch.randint(0, 256, (B, H, W, 3), generator=torch.Generator().manual_seed(3), dtype=torch.uint8).cuda()
    pipes = {}
    for key, t in (('no_transform', None), ('normalize_0.5_1', transform.TensorTransform([T.ToTensor(), T.Normalize((0.5,) * 3, (1.0,) * 3)]))):
        net.set_input_transform(t)            # captured into this pipeline's graphs
        p = DetectPipeline(inference, cfg, B, H, W, slots=2, uint8_input=True).prepare()
        for s in range(2):
            p.x[s].copy_(frames)
        pipes[key] = p

    def run(p):
        def fn():                             # both slots in flight on the pipeline's lanes; the timing stream waits for them
            p.run(0)
            p.run(1)
            cur = torch.cuda.current_stream()
            cur.wait_event(p.done[0])
            cur.wait_event(p.done[1])
        return fn
    res = alternate({k: run(p) for k, p in pipes.items()}, iters, rounds, 1.0)
    return {k: dict(images_per_s=round(2 * B * 1e3 / v['median']), ms_per_2_batches=v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=7)
    a = ap.parse_args()
    import torch
    import transform
    import torchvision.transforms as T
    if not torch.cuda.is_available():
        raise SystemExit('bench_input_transform: no CUDA device')
    t = transform.TensorTransform([T.ToTensor(), T.Normalize((0.5,) * 3, (1.0,) * 3)])
    x_u8 = torch.randint(0, 256, (B, H, W, 3), generator=torch.Generator().manual_seed(2), dtype=torch.uint8).cuda()
    x_f32 = t(x_u8)
    lut = t.lut(x_u8.device)
    out = dict(gpu=gpu_info(), batch=B, height=H, width=W, transform='ToTensor + Normalize(0.5, 1)', first_layer_us={}, forward_ms={})
    with torch.no_grad():
        for name in BACKBONES:
            net, _, _ = build(name)
            out['first_layer_us'][name] = alternate(first_layer(name, net, x_u8, x_f32, lut), 4 * a.iters, a.rounds, 1e3)
            net.set_input_transform(t)
            calls = {'fp32': lambda: net(x_f32), 'fused': lambda: net(x_u8), 'separate': lambda: net(t(x_u8))}
            out['forward_ms'][name] = alternate(calls, a.iters, a.rounds, 1.0)
            del net
            torch.cuda.empty_cache()
        out['pipeline'] = pipeline(a.iters, a.rounds)
    out['gpu_after'] = gpu_info()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
