#!/usr/bin/env python
"""The DenseNet training step (densenet121 / 169 / 201) on one GPU at batch 32, 416x416.  Prints ONE JSON line with one entry per network:

  graphed       train.GraphedStep (train-mode forward, region loss, backward, SGD) replayed --steps times after one warm-up step, CUDA events:
                ms per step and images/s
  eager         train.iterate (the same step issued from Python every time), --steps times after one warm-up step, CUDA events
  launches      C-ABI launches of one eager step: in total, and those of the per-step weight re-pack (forward and data-gradient operands of
                every conv); the re-pack alone captured in a CUDA graph and replayed, ms
  shares        kernel-time shares of eager steps under torch.profiler (a separate run): implicit-GEMM convs (forward and data gradient),
                weight gradients (plain and pre-activation), BatchNorm training ops, pools, weight packs, other
and the card's name, power limit and max SM clock read in the same run (nvidia-smi query).

    python tools/bench_densenet_train.py --steps 10 [--nets densenet121,densenet169]

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


def timed(fn, steps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        out = fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps, out


def bench(name, b, steps):
    import torch
    import model
    import model.densenet
    import train as yb_train
    import densenet_oracle as D
    from b200 import ops
    from oracle import yolo2_oracle as O
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'threshold': '0.6', 'pretrained': '0'},
                   'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'},
                   'hparam': {k: str(v) for k, v in O.HPARAM_DEFAULT.items()}, 'train': {'cross_entropy': '1'}})
    anchors = O.anchors_yolo_voc()
    net = getattr(model.densenet, name)(model.ConfigChannels(cfg), anchors, 20)
    net.load_state_dict(D.make_densenet_state_dict(name, 0), strict=False)
    net = net.cuda().train()
    inference = model.Inference(cfg, net, anchors).train()
    opt = torch.optim.SGD(net.parameters(), 1e-4, momentum=0.9)
    t = O.synth_targets(b, H, W, slots=8, seed=1)
    batch = dict(tensor=O.synth_images(b, H, W, seed=1).cuda(), yx_min=t['yx_min'].cuda(), yx_max=t['yx_max'].cuda(), cls=t['cls'].cuda())
    res = {}
    ms, out = timed(lambda: yb_train.iterate(inference, opt, anchors, cfg, batch), steps)
    res['eager'] = dict(ms_per_step=round(ms, 3), images_per_s=round(b * 1000.0 / ms, 1), loss_total=round(float(out['loss_total']), 4))
    step = yb_train.GraphedStep(inference, opt, anchors, cfg)
    ms, out = timed(lambda: step(batch), steps)
    res['graphed'] = dict(ms_per_step=round(ms, 3), images_per_s=round(b * 1000.0 / ms, 1), loss_total=round(float(out['loss_total']), 4),
                          launches=step.launches, found_inf=float(net.trainer.found_inf))
    del step

    n0 = ops.launch_count
    yb_train.iterate(inference, opt, anchors, cfg, batch)
    torch.cuda.synchronize()
    total = ops.launch_count - n0
    n0 = ops.launch_count
    net.trainer._repack(torch.device('cuda'))
    res['launches'] = dict(per_eager_step=total, repack=ops.launch_count - n0)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            yb_train.iterate(inference, opt, anchors, cfg, batch)
        torch.cuda.synchronize()
    fam = {'conv': 0.0, 'wgrad': 0.0, 'bn': 0.0, 'pool': 0.0, 'pack': 0.0, 'other': 0.0}
    for e in prof.key_averages():
        tm = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        n = e.key
        if 'conv_wgrad_kernel' in n or 'unpack_wgrad' in n or 'stem7x7_wgrad' in n:
            fam['wgrad'] += tm
        elif 'conv_igemm_kernel' in n or 'conv_wide_kernel' in n or 'conv_preact_kernel' in n or 'conv_c32_kernel' in n or 'stem7x7' in n:
            fam['conv'] += tm
        elif 'pack_weight' in n:
            fam['pack'] += tm
        elif 'bn_' in n:
            fam['bn'] += tm
        elif 'pool' in n:
            fam['pool'] += tm
        else:
            fam['other'] += tm
    tot = sum(fam.values())
    res['shares'] = {k: round(v / tot, 3) for k, v in fam.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--batch', type=int, default=B)
    ap.add_argument('--nets', default='densenet121,densenet169,densenet201')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_densenet_train: needs a GPU')
    res = dict(gpu=gpu_info(), batch=args.batch, size=[H, W])
    for name in args.nets.split(','):
        res[name] = bench(name, args.batch, args.steps)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
