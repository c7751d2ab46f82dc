#!/usr/bin/env python
"""DenseNet inference throughput on one GPU: densenet121 / 169 / 201 at batch 32, 416x416.  Prints ONE JSON line with a record per net:

  ms_per_batch / images_per_s  the forward captured in a CUDA graph after one warm-up call, CUDA events over --steps replays
  gflop_per_image              algorithmic FLOPs from the shapes (2 Cin Cout k^2 per output pixel; transition convs at the resolution the
                               reference runs them, before its pool), and the share of the 1x1 and 3x3 convs
  shares                       kernel-time shares per family from a separate torch.profiler run of eager forwards: pre-activation GEMM
                               (conv_preact_kernel), plain implicit-GEMM conv, pool kernels, stem
  preact_*                     the pre-activation GEMM's achieved TFLOP/s and HBM bytes/s (A read once, weights, output written), and which
                               of the two data-sheet bounds (989 TFLOP/s dense fp16, 3.35 TB/s) is closer
and, for densenet121's dense-layer 1x1 shapes (all 58 at batch 32, 416x416), the A/B behind the kernel: the fused form
(yb_conv1x1_preact_fwd) against writing relu(bn(x)) with yb_bn_act_apply (running statistics) and running the plain conv on that copy,
each form captured in a CUDA graph,
alternated --pairs times.  The card's name, power limit and max SM clock are read in the same run (nvidia-smi query).

    python tools/bench_densenet.py --steps 20 --pairs 5

Writes nothing to the source tree.
"""
import argparse
import configparser
import ctypes
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, 'yolo2-pytorch_b200'), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

NAMES = ('densenet121', 'densenet169', 'densenet201')
B, H, W = 32, 416, 416
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35        # H100 SXM data sheet (dense fp16, 700 W card): denominators, not reached figures
FAMILIES = (('preact_gemm', ('conv_preact_kernel',)), ('plain_conv', ('conv_igemm_kernel', 'conv_wide_kernel', 'conv_c32_kernel')),
            ('pool', ('maxpool3x3_s2_ld_kernel', 'bn_relu_avgpool2x2_kernel')), ('stem', ('stem7x7_kernel',)))


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def layer_shapes(net, h, w):
    """[(kind, cin, cout, k, pixels)] of every conv of one image, in the reference's order."""
    out = [('stem', 3, 64, 7, (h // 2) * (w // 2))]
    hh, ww = h // 4, w // 4
    for i, n in enumerate(net.block_config):
        cin0 = net.block_channels[i][0]
        for j in range(n):
            out.append(('preact1x1', cin0 + j * net.growth_rate, net.bn_size * net.growth_rate, 1, hh * ww))
            out.append(('conv3x3', net.bn_size * net.growth_rate, net.growth_rate, 3, hh * ww))
        if i + 1 < len(net.block_config):
            c = net.block_channels[i][1]
            out.append(('transition1x1', c, c // 2, 1, hh * ww))
            hh, ww = hh // 2, ww // 2
    out.append(('head1x1', net.block_channels[-1][1], net.features.conv.weight.shape[0], 1, hh * ww))
    return out


def timed(fn, n, torch):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def run(name, steps, torch):
    import model
    import model.densenet
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}, 'model': {'pretrained': '0'}})
    anchors = torch.tensor([[1.0, 1.0]] * 5)
    net = getattr(model.densenet, name)(model.ConfigChannels(cfg), anchors, 20).cuda().eval()
    g = torch.Generator().manual_seed(1)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
    x = torch.rand(B, 3, H, W, generator=g).cuda()
    shapes = layer_shapes(net, H, W)
    flop = {k: 0.0 for k in ('stem', 'preact1x1', 'conv3x3', 'transition1x1', 'head1x1')}
    for kind, cin, cout, k, pix in shapes:
        flop[kind] += 2.0 * cin * cout * k * k * pix
    total = sum(flop.values())
    with torch.no_grad():
        net(x)                                                     # warm-up: packs / folds the operands, loads the modules
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            net(x)
        graph.replay()
        torch.cuda.synchronize()
        ms = timed(graph.replay, steps, torch)
        # per-family kernel time, profiler run of its own (eager forwards)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                net(x)
            torch.cuda.synchronize()
    fam = {k: 0.0 for k, _ in FAMILIES}
    fam['other'] = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = ev.cuda_time_total
        if t <= 0:
            continue
        key = next((k for k, names in FAMILIES if any(n in ev.key for n in names)), 'other')
        fam[key] += t / 3.0 / 1000.0                              # ms per forward
    kern = sum(fam.values())
    pre_flop = flop['preact1x1'] + flop['head1x1']
    # fp16 A read once, fp16 weights; the dense layers write fp16, the head fp32
    pre_bytes = sum(B * pix * (2.0 * cin + (4.0 if kind == 'head1x1' else 2.0) * cout) + 2.0 * cin * cout
                    for kind, cin, cout, k, pix in shapes if kind in ('preact1x1', 'head1x1'))
    pre_ms = fam['preact_gemm']
    rec = dict(ms_per_batch=ms, images_per_s=B / ms * 1e3, gflop_per_image=total / 1e9, gflop_1x1=(flop['preact1x1'] + flop['transition1x1'] + flop['head1x1']) / 1e9,
               gflop_3x3=flop['conv3x3'] / 1e9, achieved_tflops_end_to_end=B * total / (ms * 1e-3) / 1e12,
               kernel_ms=fam, shares={k: v / kern for k, v in fam.items()} if kern > 0 else None)
    if pre_ms > 0:
        tf = B * pre_flop / (pre_ms * 1e-3) / 1e12
        tb = pre_bytes / (pre_ms * 1e-3) / 1e12
        rec.update(preact_tflops=tf, preact_tbytes_per_s=tb, preact_share_of_compute_bound=tf / PEAK_TFLOPS, preact_share_of_hbm_bound=tb / PEAK_TBS,
                   preact_bound='hbm' if pre_bytes / (PEAK_TBS * 1e12) > B * pre_flop / (PEAK_TFLOPS * 1e12) else 'compute')
    del graph
    return net, rec


def ab_fused_vs_materialised(net, pairs, torch):
    """densenet121's 58 dense-layer 1x1 convs at batch 32, 416x416: fused pre-activation GEMM vs yb_bn_act_apply + plain conv."""
    from b200 import ops
    g = torch.Generator().manual_seed(2)
    cases = []
    hh = H // 4
    for i, n in enumerate(net.block_config):
        cin0, cend = net.block_channels[i]
        buf = (torch.randn(B, hh, hh, cend, generator=g) * 0.5).half().cuda()
        for j in range(n):
            cin = cin0 + j * net.growth_rate
            w = ops.pack_weight_f16((torch.randn(128, cin, 1, 1, generator=g) * (2.0 / cin) ** 0.5).cuda())
            mean, var = (torch.randn(cin, generator=g) * 0.1).cuda(), (torch.rand(cin, generator=g) + 0.5).cuda()
            gamma, beta = (torch.rand(cin, generator=g) + 0.5).cuda(), (torch.randn(cin, generator=g) * 0.1).cuda()
            invstd = torch.rsqrt(var + 1e-5)
            ps, pb = ops.bn_fold(gamma, beta, mean, var)
            cases.append(dict(buf=buf, cin=cin, w=w, mean=mean, invstd=invstd, gamma=gamma, beta=beta, ps=ps, pb=pb, h=hh))
        hh //= 2
    one, zero = torch.ones(128, device='cuda'), torch.zeros(128, device='cuda')
    outs = {hw: torch.empty(B, hw, hw, 128, dtype=torch.float16, device='cuda') for hw in {c['h'] for c in cases}}
    for c in cases:
        c['a'] = torch.empty(B, c['h'], c['h'], c['cin'], dtype=torch.float16, device='cuda')

    def fused():
        for c in cases:
            ops.conv1x1_preact(c['buf'], c['w'], c['ps'], c['pb'], True, one, zero, 1.0, out=outs[c['h']], cin=c['cin'])

    def materialised():
        for c in cases:
            # yb_bn_act_apply takes 32, 64, ..., 2048 channels per launch (C / 8 must divide its 256 threads): Cin as a sum of such pieces
            off, rest = 0, c['cin']
            while rest:
                piece = 32
                while piece * 2 <= rest:
                    piece *= 2
                ops.call('yb_bn_act_apply', ctypes.c_void_p(c['buf'].data_ptr() + 2 * off), c['buf'].shape[-1], c['mean'][off:], c['invstd'][off:],
                         c['gamma'][off:], c['beta'][off:], 0.0, c['a'], c['cin'], off, B, c['h'], c['h'], piece, 0)
                off += piece
                rest -= piece
            ops.conv_bn_act(c['a'], c['w'], one, zero, 1.0, out=outs[c['h']])

    # each variant captured in a CUDA graph, so the timed replays measure device work, not the host's launch rate
    graphs = {}
    for key, fn in (('fused', fused), ('materialised', materialised)):
        fn()
        torch.cuda.synchronize()
        graphs[key] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[key]):
            fn()
        graphs[key].replay()
    torch.cuda.synchronize()
    f_ms, m_ms = [], []
    for _ in range(pairs):
        f_ms.append(timed(graphs['fused'].replay, 3, torch))
        m_ms.append(timed(graphs['materialised'].replay, 3, torch))
    return dict(layers=len(cases), fused_ms=f_ms, materialised_ms=m_ms, fused_median_ms=sorted(f_ms)[len(f_ms) // 2],
                materialised_median_ms=sorted(m_ms)[len(m_ms) // 2], speedup=sorted(m_ms)[len(m_ms) // 2] / sorted(f_ms)[len(f_ms) // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--pairs', type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_densenet.py needs a CUDA device (there is no CPU fallback)')
    torch.cuda.set_device(0)
    line = dict(metric='DenseNet 416x416 batch-32 inference images/sec', gpu=gpu_info(), batch=B, steps=args.steps, dtype='f16 operands, fp32 accumulate')
    for name in NAMES:
        net, rec = run(name, args.steps, torch)
        line[name] = rec
        if name == 'densenet121':
            line['ab_dense_1x1_fused_vs_materialised'] = ab_fused_vs_materialised(net, max(3, args.pairs), torch)
        del net
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
