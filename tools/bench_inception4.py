#!/usr/bin/env python
"""Inception-v4 inference throughput on one GPU at batch 32, 416x416.  Prints ONE JSON line:

  ms_per_batch / images_per_s  the forward captured in a CUDA graph after one warm-up call, CUDA events over --steps replays
  gflop_per_image              algorithmic conv FLOPs from the shapes (2 Cin Cout kh kw per output pixel, the reference's channel counts),
                               in total and per geometry (kh x kw, stride, padding)
  conv_tflops_end_to_end       those FLOPs over the whole forward's time
  shares                       kernel-time shares per family from a separate torch.profiler run of eager forwards: implicit-GEMM convs,
                               pools (max and count-exclusive average), stem, other (BatchNorm folds and packs are cached, so none run)
and the card's name, power limit and max SM clock read in the same run (nvidia-smi query).  With --cpu it only prints the FLOP table.

    python tools/bench_inception4.py --steps 20

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

import inception4_oracle as I  # noqa: E402  (the architecture table)

B, H, W = 32, 416, 416


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def out_size(n, k, s, p):
    return (n + 2 * p - k) // s + 1


def unit_shapes(h, w):
    """[(key, cin, cout, kh, kw, stride, pad_h, pad_w, out_h, out_w)] of every conv and the head for one h x w image.  A block's unit reads the
    block input (or its average pool, same size) or its source unit's output; the last unit of every block ends at the block's output size."""
    widths = I.widths()
    cin, c_last = I.in_channels(widths)
    out, size, block, cur = [], {}, None, (h, w)
    for key, (kh, kw, s, ph, pw, src) in I.GEOM.items():
        stem = key.count('.') == 1
        prefix = '.'.join(key.split('.')[:2])
        if not stem and prefix != block:
            block, block_in = prefix, cur
        ih, iw = cur if stem else block_in if src in (None, 'avg') else size[src]
        cur = size[key] = (out_size(ih, kh, s, ph), out_size(iw, kw, s, pw))
        out.append((key, cin[key], widths[key], kh, kw, s, ph, pw) + cur)
    out.append((I.HEAD, c_last, 125, 1, 1, 1, 0, 0) + cur)
    return out


def geometry(u):
    return '%dx%d s%d p%d,%d' % (u[3], u[4], u[5], u[6], u[7])


def flops(u):
    return 2.0 * u[1] * u[2] * u[3] * u[4] * u[8] * u[9]


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
    line = dict(net='inception4', batch=B, size=[H, W], gflop_per_image=round(total, 3), gflop_by_geometry=by)
    if args.cpu:
        print(json.dumps(line))
        return
    import torch
    import model
    import model.inception4
    from oracle import yolo2_oracle as O
    assert torch.cuda.is_available(), 'bench_inception4 needs a GPU'
    line['gpu'] = gpu_info()
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'}})
    net = model.inception4.Inception4(model.ConfigChannels(cfg), O.anchors_yolo_voc(), 20)
    net.load_state_dict(I.make_state_dict(0), strict=False)
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
    line['conv_tflops_end_to_end'] = round(total * B / ms, 1)         # GFLOP / ms = TFLOP/s
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
    tot = sum(fam.values())
    line['shares'] = {k: round(v / tot, 3) for k, v in fam.items()}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
