#!/usr/bin/env python
"""VGG-16 / VGG-16-BN inference and the VGG-16-BN training step on one GPU at batch 32, 416x416.  Prints ONE JSON line:

  ms_per_batch / images_per_s  per network, the forward captured in a CUDA graph after one warm-up call, CUDA events over --steps replays
  gflop_per_image              algorithmic conv FLOPs from the shapes (2 Cin Cout 9 per output pixel, 2 Cin Cout for the head), in total and
                               per conv geometry (Cin -> Cout at the output size), with the first layer's share
  conv_tflops_end_to_end       those FLOPs over the whole forward's time
  shares                       kernel-time shares per family from a separate torch.profiler run of eager vgg16_bn forwards: the first layer
                               (conv0_c64_kernel), the implicit-GEMM convs, the max-pools, other (BatchNorm folds and packs are cached, so
                               none run)
  vgg16_bn_train               train.GraphedStep (train-mode forward, region loss, backward, SGD) replayed --steps times, CUDA events; and
                               kernel-time shares of eager steps under the profiler: first layer forward and weight gradient, implicit-GEMM
                               convs (forward and data gradient), weight gradients, BatchNorm / ReLU / pool training ops, other
and the card's name, power limit and max SM clock read in the same run (nvidia-smi query).  With --cpu it only prints the FLOP table.

    python tools/bench_vgg.py --steps 20

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

import vgg_oracle as V  # noqa: E402  (the architecture table)

B, H, W = 32, 416, 416
NETS = ('vgg16', 'vgg16_bn')


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def unit_shapes(name, h, w):
    """[(cin, cout, k, out_h, out_w)] of every conv and the head for one h x w image."""
    out, cin = [], 3
    for kind, _, c in V.layers(name):
        if kind == 'conv':
            out.append((cin, c, 3, h, w))
            cin = c
        elif kind == 'pool':
            h, w = h // 2, w // 2
    out.append((cin, 125, 1, h, w))
    return out


def flop_table(name, h, w):
    shapes = unit_shapes(name, h, w)
    by = {}
    for cin, cout, k, oh, ow in shapes:
        key = '%dx%d %d->%d @%dx%d' % (k, k, cin, cout, oh, ow)
        by[key] = by.get(key, 0.0) + 2.0 * cin * cout * k * k * oh * ow / 1e9
    total = sum(by.values())
    first = 2.0 * 3 * 64 * 9 * h * w / 1e9
    return total, first / total, {k: round(v, 3) for k, v in by.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--cpu', action='store_true', help='print the FLOP table only')
    args = ap.parse_args()
    total, first_share, by = flop_table('vgg16', H, W)
    line = dict(net='vgg16', batch=B, size=[H, W], gflop_per_image=round(total, 3), first_layer_flop_share=round(first_share, 4),
                gflop_by_geometry=by)
    if args.cpu:
        print(json.dumps(line))
        return
    import torch
    import model
    import model.vgg
    from oracle import yolo2_oracle as O
    assert torch.cuda.is_available(), 'bench_vgg needs a GPU'
    line['gpu'] = gpu_info()
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'}})
    x = O.synth_images(B, H, W, seed=0).cuda()
    nets = {}
    for name in NETS:
        net = getattr(model.vgg, name)(model.ConfigChannels(cfg), O.anchors_yolo_voc(), 20)
        net.load_state_dict(V.make_state_dict(name), strict=False)
        nets[name] = net = net.cuda().eval()
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
        del graph
        line[name] = dict(ms_per_batch=round(ms, 3), images_per_s=round(B * 1000.0 / ms, 1),
                          conv_tflops_end_to_end=round(total * B / ms, 1))         # GFLOP / ms = TFLOP/s
    # kernel-time shares, eager forwards under the profiler
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            nets['vgg16_bn'](x)
        torch.cuda.synchronize()
    fam = {'first_layer': 0.0, 'conv': 0.0, 'pool': 0.0, 'other': 0.0}
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        n = e.key
        if 'conv0_c64_kernel' in n:
            fam['first_layer'] += t
        elif 'conv_igemm_kernel' in n or 'conv_wide_kernel' in n or 'conv_c32_kernel' in n:
            fam['conv'] += t
        elif 'pool' in n:
            fam['pool'] += t
        else:
            fam['other'] += t
    tot = sum(fam.values())
    line['shares_vgg16_bn'] = {k: round(v / tot, 3) for k, v in fam.items()}
    line['first_layer_ms_per_batch'] = round(fam['first_layer'] / 3 / 1000.0, 3)
    del nets
    line['vgg16_bn_train'] = train_step(args.steps)
    print(json.dumps(line))


def train_step(steps):
    import torch
    import model
    import model.vgg
    import train as yb_train
    from oracle import yolo2_oracle as O
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                   'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                   'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    anchors = O.anchors_yolo_voc()
    net = model.vgg.vgg16_bn(model.ConfigChannels(cfg), anchors, 20)
    net.load_state_dict(V.make_state_dict('vgg16_bn'), strict=False)
    net = net.cuda().train()
    inference = model.Inference(cfg, net, anchors).train()
    opt = torch.optim.SGD(net.parameters(), 1e-4, momentum=0.9)
    t = O.synth_targets(B, H, W, slots=8, seed=1)
    batch = dict(tensor=O.synth_images(B, H, W, seed=1).cuda(), yx_min=t['yx_min'].cuda(), yx_max=t['yx_max'].cuda(), cls=t['cls'].cuda())
    step = yb_train.GraphedStep(inference, opt, anchors, cfg)
    step(batch)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        out = step(batch)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    res = dict(ms_per_step=round(ms, 3), images_per_s=round(B * 1000.0 / ms, 1), loss_total=round(float(out['loss_total']), 4))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            yb_train.iterate(inference, opt, anchors, cfg, batch)
        torch.cuda.synchronize()
    fam = {'first_layer_fwd': 0.0, 'first_layer_wgrad': 0.0, 'conv': 0.0, 'wgrad': 0.0, 'bn_relu_pool': 0.0, 'other': 0.0}
    for e in prof.key_averages():
        tm = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        n = e.key
        if 'conv0_c64_wgrad_kernel' in n:
            fam['first_layer_wgrad'] += tm
        elif 'conv0_c64_kernel' in n:
            fam['first_layer_fwd'] += tm
        elif 'conv_wgrad_kernel' in n or 'unpack_wgrad' in n:
            fam['wgrad'] += tm
        elif 'conv_igemm_kernel' in n or 'conv_wide_kernel' in n or 'conv_c32_kernel' in n:
            fam['conv'] += tm
        elif 'bn_' in n or 'pool' in n:
            fam['bn_relu_pool'] += tm
        else:
            fam['other'] += tm
    tot = sum(fam.values())
    res['shares'] = {k: round(v / tot, 3) for k, v in fam.items()}
    return res


if __name__ == '__main__':
    main()
