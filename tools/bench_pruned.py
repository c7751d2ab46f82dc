#!/usr/bin/env python
"""Channel-pruned Darknet-19 on one GPU at batch 32, 416x416.  Prints ONE JSON line with:

  images_per_s     {'full': full-width Darknet-19, 'pruned': the pruned checkpoint of tests/golden/pruned.npz}: the eval forward
                   captured in a CUDA graph after two warm-up calls, CUDA events over --steps replays, the two models alternated --rounds
                   times (median of the rounds)
  tail_layers      per unit of the pruned model that runs on the channel-tail entry (yb_conv_bn_act_tail_fwd): its shape, the tail
                   launch's time and the time of the same layer on the plain entry with its input materialised with zeros up to
                   cin_pad (same tile: the library's own choice for the padded shape, no stream-K), CUDA events over --iters launches,
                   medians of --rounds alternated rounds
and the card's name, power limit and SM clocks read in the same run (nvidia-smi query).

    python tools/bench_pruned.py [--steps 50] [--iters 200] [--rounds 5]

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
for _p in (os.path.join(ROOT, 'yolo2-pytorch_b200'), ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

B, H, W = 32, 416, 416


def gpu_info():
    q = 'name,power.limit,clocks.max.sm,clocks.sm'
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True)
    vals = [v.strip() for v in r.stdout.strip().split(',')] if r.returncode == 0 else []
    return dict(zip(q.split(','), vals)) if len(vals) == 4 else dict(error=r.stderr.strip())


def build(sd):
    import model
    import model.yolo2
    from oracle import yolo2_oracle as O
    cfg = configparser.ConfigParser()
    cfg.read_dict({'batch_norm': {'enable': '1'}})
    dnn = model.yolo2.Darknet(model.ConfigChannels(cfg, sd), O.anchors_yolo_voc(), 20)
    dnn.load_state_dict(sd, strict=False)
    return dnn.cuda().eval()


def graphed(dnn, x):
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            dnn.engine.forward(x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        dnn.engine.forward(x)
    return g


def time_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def tail_launches(dnn, x):
    """(key, unit, input) of every launch of one eager forward that goes to the channel-tail entry."""
    from b200 import ops
    eng = dnn.engine
    by_w = {id(u.w16): (k, u) for k, u in zip(eng.unit_keys(), eng.all_units())}
    calls = []
    orig = ops.conv_bn_act_tail

    def rec(xx, w, *a, **kw):
        k, u = by_w[id(w)]
        calls.append((k, u, xx, kw))
        return orig(xx, w, *a, **kw)
    ops.conv_bn_act_tail = rec
    try:
        eng.forward(x)
    finally:
        ops.conv_bn_act_tail = orig
    return calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_pruned.py needs a CUDA device (there is no CPU fallback)')
    from b200 import ops
    from oracle import yolo2_oracle as O
    import pruned_oracle as PO
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'pruned.npz'))
    x = O.synth_images(B, H, W, seed=0).cuda()
    nets = {'full': build(O.make_state_dict(0)), 'pruned': build(PO.darknet_pruned_state_dict(PO.keep_from_npz(g, 'darknet_')))}
    graphs = {k: graphed(d, x) for k, d in nets.items()}
    for gr in graphs.values():
        time_ms(gr.replay, 3)
    ips = {k: [] for k in nets}
    for _ in range(args.rounds):
        for k, gr in graphs.items():
            ips[k].append(B * 1000.0 / time_ms(gr.replay, args.steps))

    layers = []
    ws = ops.conv_workspace('cuda')
    for key, u, xx, kw in tail_launches(nets['pruned'], x):
        cin, cin_pad = u.in_ch, u.k_ch
        x_pad = torch.zeros(*xx.shape[:3], cin_pad, dtype=torch.float16, device='cuda')
        x_pad[..., :cin] = xx[..., :cin]
        out_mode = kw.get('out_mode', ops.OUT_F16_NHWC)
        y = kw['out']
        off = kw.get('y_ch_off', 0)
        flags = ops.CONV_NO_STREAMK | ops.CONV_NO_SMALLK

        def tail():
            ops.conv_bn_act_tail(xx, u.w16, u.scale, u.shift, u.slope, cin, out=y, out_mode=out_mode, y_ch_off=off)

        def padded():
            ops.conv_bn_act(x_pad, u.w16, u.scale, u.shift, u.slope, out=y, out_mode=out_mode, y_ch_off=off, workspace=ws, flags=flags)
        for fn in (tail, padded):
            time_ms(fn, 5)
        t_tail, t_pad = [], []
        for _ in range(args.rounds):
            t_tail.append(time_ms(tail, args.iters) * 1000.0)
            t_pad.append(time_ms(padded, args.iters) * 1000.0)
        b, h, w, _ = xx.shape
        layers.append(dict(unit=key, shape='%dx%dx%d cin %d (pad %d) -> %d, k%d' % (b, h, w, cin, cin_pad, u.out_ch, u.ksize),
                           tail_us=round(statistics.median(t_tail), 2), padded_operand_us=round(statistics.median(t_pad), 2),
                           tail_over_padded=round(statistics.median(t_tail) / statistics.median(t_pad), 4)))
    widths = {k: u.cout for k, u in zip(nets['pruned'].engine.unit_keys(), nets['pruned'].engine.all_units())}
    line = dict(tool='bench_pruned', workload='Darknet-19 eval forward, batch %d, %dx%d, CUDA graph, precision fast' % (B, H, W), gpu=gpu_info(),
                images_per_s={k: round(statistics.median(v), 1) for k, v in ips.items()},
                images_per_s_rounds={k: [round(t, 1) for t in v] for k, v in ips.items()},
                pruned_widths=widths, tail_layers=layers)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
