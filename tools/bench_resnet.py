#!/usr/bin/env python
"""ResNet inference throughput on one GPU at batch 32, 416x416 (default: resnet101 and resnet152).  Prints ONE JSON line with a record per net:

  ms_per_batch / images_per_s  the eval forward captured in a CUDA graph after one warm-up call, CUDA events over --steps replays
  gflop_per_image              algorithmic conv FLOPs from the shapes (2 Cin Cout k^2 per OUTPUT pixel, stride-2 convs at their real output
                               resolution, not the 4x the stride-1 + even-pixel-selection form executes), stem and head included
  conv_tflops_end_to_end       those FLOPs over the whole forward's time
  peak_mem_gb                  torch.cuda.max_memory_allocated over the eager warm-up and the capture
and the card's name, power limit and max SM clock read in the same run (nvidia-smi query).

    python tools/bench_resnet.py --steps 20 [--nets resnet50,resnet101,resnet152]

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

B, H, W = 32, 416, 416


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def gflop_forward(net, h, w):
    """Algorithmic GFLOP of one image's eval forward (see the module docstring)."""
    total = 2.0 * 3 * 64 * 49 * (h // 2) * (w // 2)
    h, w = h // 4, w // 4
    for lname in ('layer1', 'layer2', 'layer3', 'layer4'):
        for blk in getattr(net, lname).children():
            hin, win = h, w
            for _, conv, _, _ in blk.units():
                s = conv.stride[0]
                h, w = h // s, w // s
                total += 2.0 * conv.in_channels * conv.out_channels * conv.kernel_size[0] ** 2 * h * w
            if blk.downsample is not None:
                conv = blk.downsample[0]
                s = conv.stride[0]
                total += 2.0 * conv.in_channels * conv.out_channels * (hin // s) * (win // s)
    total += 2.0 * net.conv.in_channels * net.conv.out_channels * h * w
    return total / 1e9


def run(name, steps):
    import torch
    import model
    import model.resnet
    import resnet_deep_oracle  # noqa: F401  (resnet101 / 152 in the oracle's ResNet table)
    from oracle import yolo2_oracle as O
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'}})
    net = getattr(model.resnet, name)(model.ConfigChannels(cfg), O.anchors_yolo_voc(), 20)
    net.load_state_dict(O.make_resnet_state_dict(name, 0), strict=False)
    net = net.cuda().eval()
    x = O.synth_images(B, H, W, seed=0).cuda()
    torch.cuda.reset_peak_memory_stats()
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
        for _ in range(steps):
            graph.replay()
        t1.record()
        torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    gflop = gflop_forward(net, H, W)
    rec = dict(ms_per_batch=round(ms, 3), images_per_s=round(B * 1000.0 / ms, 1), gflop_per_image=round(gflop, 3),
               conv_tflops_end_to_end=round(gflop * B / ms, 1), peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    del graph
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--nets', default='resnet101,resnet152')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_resnet.py needs a CUDA device (there is no CPU fallback)')
    torch.cuda.set_device(0)
    line = dict(metric='ResNet 416x416 inference images/sec', batch=B, size=[H, W], steps=args.steps, gpu=gpu_info(), dtype='f16')
    for name in args.nets.split(','):
        line[name] = run(name, args.steps)
        torch.cuda.empty_cache()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
