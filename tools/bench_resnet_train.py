#!/usr/bin/env python
"""ResNet training throughput on one GPU: resnet18 (64 images) and resnet50 (32 images) at 416x416 by default, resnet34, resnet101 and
resnet152 (32 images each) with --nets, train-mode forward + region loss + backward + fused capturable Adam, one CUDA graph per step
(train.GraphedStep).  Prints ONE JSON line with a record per net:

  value / ms_per_step   images/s and the graphed step time (CUDA events over --steps replays after --warmup)
  gflop_per_image       algorithmic training FLOPs: 2 Cin Cout k^2 per OUTPUT pixel of every conv (stride-2 convs at their real output
                        resolution, not the 4x the stride-1 + even-pixel-selection form executes), x3 for forward, data and weight gradient,
                        minus the stem's data gradient (the image needs none)
  stem_*_ms / _share    the stem's two CUDA-core kernels (raw forward, weight gradient) timed alone with CUDA events on the step's shapes,
                        and that time over the graphed step
  saved_gb              device memory held between one eager train-mode forward and its backward (the activations saved for the backward)
  peak_mem_gb           torch.cuda.max_memory_allocated over the whole run of the net (eager forward, capture, replays)
  grad_scale            the trainer's static loss scale

    python tools/bench_resnet_train.py --steps 50 --warmup 5 [--nets resnet101,resnet152]

Writes nothing to the source tree.  Reuses bench.py's workload helpers (config, anchors, synthetic batches, peak figures).
"""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the product package on sys.path)

# batch sizes chosen to fit comfortably in 80 GB at 416x416 (resnet152 at 32 images saves 9.1 GB of activations for its backward, DESIGN §6)
BATCH = {'resnet18': 64, 'resnet34': 32, 'resnet50': 32, 'resnet101': 32, 'resnet152': 32}


def gflop_train(net, H, W):
    """Algorithmic GFLOP of one ResNet training image (see the module docstring)."""
    stem = 2.0 * 3 * 64 * 49 * (H // 2) * (W // 2)
    fwd = stem
    h, w = H // 4, W // 4
    for lname in ('layer1', 'layer2', 'layer3', 'layer4'):
        for blk in getattr(net, lname).children():
            hin, win = h, w
            for _, conv, _, _ in blk.units():
                s = conv.stride[0]
                h, w = h // s, w // s
                fwd += 2.0 * conv.in_channels * conv.out_channels * conv.kernel_size[0] ** 2 * h * w
            if blk.downsample is not None:
                conv = blk.downsample[0]
                s = conv.stride[0]
                fwd += 2.0 * conv.in_channels * conv.out_channels * (hin // s) * (win // s)
    fwd += 2.0 * net.conv.in_channels * net.conv.out_channels * h * w
    return (3 * fwd - stem) / 1e9


def run(name, B, steps, warmup, peaks, generator):
    import torch
    import model
    import model.resnet
    import train as yb_train
    from b200 import ops
    device = torch.device('cuda', torch.cuda.current_device())
    H = W = 416
    config = bench.make_config()
    config.read_dict({'model': {'pretrained': '0'}, 'hparam': {'foreground': '5', 'background': '1', 'center': '1', 'size': '1', 'cls': '1'},
                      'train': {'cross_entropy': '1'}})
    anchors = torch.tensor(bench.ANCHORS_HW, dtype=torch.float32)
    torch.manual_seed(0)
    net = getattr(model.resnet, name)(model.ConfigChannels(config), anchors, 20).to(device).train()
    inference = model.Inference(config, net, anchors).train()
    optimizer = torch.optim.Adam(net.parameters(), 1e-5, betas=(0.9, 0.999), eps=1e-8, capturable=True, fused=True)
    batches = bench._train_batches(B, H, W, device, generator)
    torch.cuda.reset_peak_memory_stats()
    step = yb_train.GraphedStep(inference, optimizer, anchors, config)
    for i in range(warmup):
        step(batches[i % 2])
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        out = step(batches[i % 2])
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / steps
    loss = float(out['loss_total'].item())
    # the stem kernels alone on this step's shapes
    x = batches[0]['tensor']
    z = torch.empty(B, H // 2, W // 2, 64, dtype=torch.float16, device=device)
    dz = torch.randn(B, H // 2, W // 2, 64, device=device).half()
    dw = torch.empty(64, 3, 7, 7, dtype=torch.float32, device=device)
    w7 = net.conv1.weight.detach().contiguous()
    kernel_ms = {}
    for kname, fn in (('stem_fwd', lambda: ops.call('yb_stem7x7_raw_fwd', x, w7, z, B, H, W)),
                      ('stem_wgrad', lambda: ops.call('yb_stem7x7_wgrad', x, dz, dw, B, H, W))):
        for _ in range(3):
            fn()
        reps = max(5, min(steps, 20))
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        kernel_ms[kname] = s.elapsed_time(e) / reps
    # after the timed replays, so the graphed step starts from the same state as without this measurement
    held = torch.cuda.memory_allocated()
    feature = net(x)
    torch.cuda.synchronize()
    saved_gb = (torch.cuda.memory_allocated() - held) / 2 ** 30
    del feature
    gflop = gflop_train(net, H, W)
    tfl = B / (ms / 1e3) * gflop / 1e3
    rec = dict(metric='%s 416x416 training images/sec' % name, value=B / (ms / 1e3), unit='images/s', ms_per_step=ms, per_gpu_batch=B,
               steps=steps, warmup=warmup, gflop_per_image=gflop, tflops=tfl, frac_of_tensor_peak=tfl / peaks['tflops'],
               stem_fwd_ms=kernel_ms['stem_fwd'], stem_wgrad_ms=kernel_ms['stem_wgrad'],
               stem_fwd_share=kernel_ms['stem_fwd'] / ms, stem_wgrad_share=kernel_ms['stem_wgrad'] / ms, loss_total=loss, cuda_graph=True,
               saved_gb=saved_gb, peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30, grad_scale=net.trainer.grad_scale,
               workload='%s 416x416 batch-%d training step: train-mode fwd + region loss + bwd + fused Adam' % (name, B))
    step.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--nets', default='resnet18,resnet50', help='comma-separated constructor names of model.resnet')
    args = ap.parse_args()
    nets = args.nets.split(',')
    unknown = [n for n in nets if n not in BATCH]
    if unknown:
        raise SystemExit('bench_resnet_train.py: unknown net(s) %s; choose from %s' % (unknown, sorted(BATCH)))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_resnet_train.py needs a CUDA device (there is no CPU fallback)')
    torch.cuda.set_device(0)
    peaks = bench.measured_peaks()
    g = torch.Generator().manual_seed(300)
    warmup = max(3, args.warmup)
    line = dict(metric='ResNet 416x416 training images/sec', n_gpus=1, steps=args.steps, warmup=warmup, dtype='f16', data='synthetic')
    for name in nets:
        line[name] = run(name, BATCH[name], args.steps, warmup, peaks, g)
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
