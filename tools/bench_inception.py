#!/usr/bin/env python
"""Inception-v3 inference throughput on one GPU at batch 32, 416x416.  Prints ONE JSON line:

  ms_per_batch / images_per_s  the forward captured in a CUDA graph after one warm-up call, CUDA events over --steps replays
  gflop_per_image              algorithmic conv FLOPs from the shapes (2 Cin Cout kh kw per output pixel, the reference's channel counts),
                               in total and per geometry (kh x kw, stride, padding)
  shares                       kernel-time shares per family from a separate torch.profiler run of eager forwards: general-geometry conv
                               (implicit GEMM on a conv that is not 1x1 stride 1), 1x1 conv, pools, stem
  tflops                       achieved TFLOP/s of the 1x7 / 7x1 convs and of the stride-2 convs, each conv launched alone (same shapes and
                               channel padding as in the forward), CUDA events over --steps launches
and the card's name, power limit and max SM clock read in the same run (nvidia-smi query).  With --cpu it only prints the FLOP table.

    python tools/bench_inception.py --steps 20

Writes nothing to the source tree.
"""
import argparse
import configparser
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, 'yolo2-pytorch_b200'), ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import inception_oracle as I  # noqa: E402  (the architecture table)

B, H, W = 32, 416, 416


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def out_size(n, k, s, p):
    return (n + 2 * p - k) // s + 1


def unit_shapes(h, w):
    """[(key, cin, cout, kh, kw, stride, pad_h, pad_w, in_h, in_w, out_h, out_w)] of every BasicConv2d and the head for one h x w image.
    Every conv of a Mixed_* block reads a tensor of the block input's size (the stride-2 convs come last in their branch)."""
    units = I.units()
    out = []
    for key, _, _, _, _, _, _, _ in I.STEM:
        cin, cout, kh, kw, s, ph, pw = units[key]
        oh, ow = out_size(h, kh, s, ph), out_size(w, kw, s, pw)
        out.append((key, cin, cout, kh, kw, s, ph, pw, h, w, oh, ow))
        h, w = oh, ow
        if key in ('Conv2d_2b_3x3', 'Conv2d_4a_3x3'):
            h, w = out_size(h, 3, 2, 0), out_size(w, 3, 2, 0)
    for name, _, _, _ in I.BLOCKS:
        nh, nw = h, w
        for key, (cin, cout, kh, kw, s, ph, pw) in units.items():
            if key.startswith(name + '.'):
                oh, ow = out_size(h, kh, s, ph), out_size(w, kw, s, pw)
                out.append((key, cin, cout, kh, kw, s, ph, pw, h, w, oh, ow))
                nh, nw = min(nh, oh), min(nw, ow)
        h, w = nh, nw
    out.append(('conv', 2048, 125, 1, 1, 1, 0, 0, h, w, h, w))
    return out


def geometry(u):
    return '%dx%d s%d p%d,%d' % (u[3], u[4], u[5], u[6], u[7])


def flops(u):
    return 2.0 * u[1] * u[2] * u[3] * u[4] * u[10] * u[11]


def flop_table(h, w):
    shapes = unit_shapes(h, w)
    by = {}
    for u in shapes:
        by[geometry(u)] = by.get(geometry(u), 0.0) + flops(u) / 1e9
    return sum(flops(u) for u in shapes) / 1e9, {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--cpu', action='store_true', help='print the FLOP table only')
    args = ap.parse_args()
    total, by = flop_table(H, W)
    line = dict(net='inception3', batch=B, size=[H, W], gflop_per_image=round(total, 3), gflop_by_geometry=by)
    if args.cpu:
        print(json.dumps(line))
        return
    import torch
    import model
    import model.inception3
    from b200 import ops
    from oracle import yolo2_oracle as O
    assert torch.cuda.is_available(), 'bench_inception needs a GPU'
    line['gpu'] = gpu_info()
    cfg = configparser.ConfigParser()
    cfg.read_dict({'model': {'pretrained': '0'}})
    net = model.inception3.Inception3(model.ConfigChannels(cfg), O.anchors_yolo_voc(), 20)
    net.load_state_dict(I.make_inception_state_dict(0), strict=False)
    net = net.cuda().eval()
    x = O.synth_images(B, H, W, seed=0).cuda()
    with torch.no_grad():
        net(x)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            net(x)
        graph.replay()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.steps):
            graph.replay()
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.steps
    line['ms_per_batch'] = round(ms, 3)
    line['images_per_s'] = round(B * 1000.0 / ms, 1)
    line["conv_tflops_end_to_end"] = round(total * B / ms, 1)         # GFLOP / ms = TFLOP/s
    # kernel-time shares, eager forwards under the profiler
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            net(x)
        torch.cuda.synchronize()
    fam = {'conv': 0.0, 'pool': 0.0, 'stem': 0.0, 'other': 0.0}
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        n = e.key
        if 'conv_igemm_kernel' in n or 'conv_wide_kernel' in n or 'conv_c32_kernel' in n:
            fam['conv'] += t
        elif 'pool' in n:
            fam['pool'] += t
        elif 'mb_conv0_kernel' in n:
            fam['stem'] += t
        else:
            fam['other'] += t
    # general-geometry vs 1x1 split of the conv time: every conv launched alone, CUDA events
    shapes = unit_shapes(H, W)
    per = {}
    for u in shapes[1:]:
        key, cin, cout, kh, kw, s, ph, pw, ih, iw, oh, ow = u
        cin_p, cout_p = (cin + 31) // 32 * 32, (cout + 31) // 32 * 32 if key != 'conv' else cout
        xa = torch.randn(B, ih, iw, cin_p, device='cuda').half()
        wt = ops.pack_weight_khw_f16(torch.randn(cout_p, cin_p, kh, kw, device='cuda') * 0.05)
        sc, sh = torch.ones(cout_p, device='cuda'), torch.zeros(cout_p, device='cuda')
        mode = ops.OUT_F32_NCHW if key == 'conv' else ops.OUT_F16_NHWC                   # the head writes the fp32 NCHW feature
        run = lambda: ops.conv2d_bn_act(xa, wt, sc, sh, 0.0, stride=s, pad=(ph, pw), out_mode=mode)    # noqa: E731
        run()
        t0.record()
        for _ in range(args.steps):
            run()
        t1.record()
        torch.cuda.synchronize()
        per[key] = (t0.elapsed_time(t1) / args.steps, flops(u) * B, u)
    general = sum(v[0] for v in per.values() if not (v[2][3] == 1 and v[2][4] == 1 and v[2][5] == 1))
    plain = sum(v[0] for v in per.values() if v[2][3] == 1 and v[2][4] == 1 and v[2][5] == 1)
    tot = sum(fam.values())
    conv_share = fam['conv'] / tot
    line['shares'] = dict(general_conv=round(conv_share * general / (general + plain), 3), conv1x1=round(conv_share * plain / (general + plain), 3),
                          pool=round(fam['pool'] / tot, 3), stem=round(fam['stem'] / tot, 3), other=round(fam['other'] / tot, 3))
    sel = {'1x7_7x1': [v for v in per.values() if (v[2][3], v[2][4]) in ((1, 7), (7, 1))], 'stride2': [v for v in per.values() if v[2][5] == 2]}
    line['tflops'] = {k: round(sum(v[1] for v in vs) / sum(v[0] for v in vs) / 1e9, 1) for k, vs in sel.items()}
    line['ms_convs_alone'] = round(general + plain, 3)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
