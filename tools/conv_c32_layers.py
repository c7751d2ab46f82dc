#!/usr/bin/env python
"""Per-launch A/B of the Cin = 32 halo-tile conv: conv_c32_kernel (weights as the register A operand, two consumer warpgroups)
against its first form conv_c32_kernel_v1 (YB_CONV_C32_V1=1), on layers1.2 of the C2 forward (208x208, 32 -> 64, batch 32), with
the fused 2x2 max-pool as the forward runs it and without.

YB_CONV_C32_V1 is read once per process, so each form lives in its own child process that stays resident for the whole run; the
parent alternates timing rounds between the two and reports medians.  In a round a form replays a CUDA graph of --reps
back-to-back launches --iters times between CUDA events.  The children also write their outputs, which must be equal bit for bit,
and trace one launch (yb_conv_set_trace, block 0): per tile of the CTA, the first wgmma issue, and for conv_c32_kernel the MMAs'
retirement and its store issue.  From those: the CTA's tile period, and (conv_c32_kernel) each tile's MMA span and epilogue, and the
share of the CTA's time in which some tile's MMAs are in flight.  Prints ONE JSON line (gpu: name, power limit, max and current SM
clock read in the same run) with the compute bound (data sheet FP16 dense rate) and the HBM bound (input + output bytes at the data
sheet bandwidth) beside the times.

    python tools/conv_c32_layers.py

Writes nothing to the source tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layers import gpu_info  # noqa: E402  (puts the product package on sys.path)

B, HW, CIN, COUT = 32, 208, 32, 64
CASES = ('pool', 'plain')
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35      # H100 SXM data sheet: dense FP16, HBM3


def child(args):
    import torch
    from b200 import lib, ops
    torch.cuda.set_device(0)
    dev = 'cuda'
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(B, HW, HW, CIN, generator=gen).half().to(dev)
    w16 = ops.pack_weight_f16((torch.randn(COUT, CIN, 3, 3, generator=gen) * (2.0 / (CIN * 9)) ** 0.5).to(dev))
    scale = (torch.rand(COUT, generator=gen) + 0.5).to(dev)
    shift = (torch.randn(COUT, generator=gen) * 0.1).to(dev)
    outs = {'pool': torch.empty(B, HW // 2, HW // 2, COUT, dtype=torch.float16, device=dev),
            'plain': torch.empty(B, HW, HW, COUT, dtype=torch.float16, device=dev)}
    fns = {c: (lambda c=c: ops.conv_bn_act(x, w16, scale, shift, 0.1, out=outs[c], flags=ops.CONV_POOL2X2 if c == 'pool' else 0))
           for c in CASES}
    graphs = {}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for c, fn in fns.items():
            fn()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                for _ in range(args.reps):
                    fn()
            graphs[c] = g
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    # one traced launch per case: role 1 slot i = tile i's first wgmma, role 2 slot 2i (conv_c32_kernel) = its MMAs retired
    trace = torch.zeros(3 * 256, dtype=torch.int64, device=dev)
    traces = {}
    for c, fn in fns.items():
        trace.zero_()
        torch.cuda.synchronize()
        lib.load().yb_conv_set_trace(trace.data_ptr())
        try:
            fn()
            torch.cuda.synchronize()
        finally:
            lib.load().yb_conv_set_trace(None)
        traces[c] = trace.view(3, 256).cpu().tolist()
    for c in CASES:
        torch.save(outs[c].view(torch.int16).cpu(), os.path.join(args.child, c + '.pt'))
    print(json.dumps(dict(ready=True, traces=traces)), flush=True)
    for line in sys.stdin:
        if line.strip() != 'round':
            break
        us = {}
        for c, g in graphs.items():
            g.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                g.replay()
            e1.record()
            e1.synchronize()
            us[c] = e0.elapsed_time(e1) * 1e3 / (args.iters * args.reps)
        print(json.dumps(us), flush=True)


def trace_stats(buf, v1):
    first = [int(v) for v in buf[1] if int(v) != 0]
    out = dict(tiles=len(first))
    if len(first) > 1:
        out['tile_period_cycles'] = (first[-1] - first[0]) / (len(first) - 1)
    if not v1:
        spans = sorted((int(buf[1][i]), int(buf[2][2 * i])) for i in range(min(len(first), 128)) if int(buf[2][2 * i]) != 0)
        if spans:
            busy, cur_s, cur_e = 0, spans[0][0], spans[0][1]
            for s, e in spans[1:]:
                if s > cur_e:
                    busy += cur_e - cur_s
                    cur_s, cur_e = s, e
                else:
                    cur_e = max(cur_e, e)
            busy += cur_e - cur_s
            out['mma_cycles_per_tile'] = statistics.mean(e - s for s, e in spans)
            epi = [int(buf[2][2 * i + 1]) - int(buf[2][2 * i]) for i in range(min(len(first), 128)) if int(buf[2][2 * i + 1]) != 0]
            out['epilogue_cycles_per_tile'] = statistics.mean(epi) if epi else None
            out['mma_busy_share'] = busy / (spans[-1][1] - spans[0][0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--child', default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args)
        return
    import torch
    forms = {'v1': '1', 'regs': '0'}
    with tempfile.TemporaryDirectory() as tmp:
        procs, ready = {}, {}
        for f, v in forms.items():
            os.makedirs(os.path.join(tmp, f))
            cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), '--child', os.path.join(tmp, f),
                                                                                      '--reps', str(args.reps), '--iters', str(args.iters)]
            procs[f] = subprocess.Popen(cmd, env=dict(os.environ, YB_CONV_C32_V1=v), stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        try:
            for f, pr in procs.items():
                line = pr.stdout.readline()
                if not line:
                    raise SystemExit('child %s failed' % f)
                ready[f] = json.loads(line)
            times = {f: {c: [] for c in CASES} for f in forms}
            for _ in range(args.rounds):
                for f, pr in procs.items():
                    pr.stdin.write('round\n')
                    pr.stdin.flush()
                    for c, v in json.loads(pr.stdout.readline()).items():
                        times[f][c].append(v)
            gpu = gpu_info()              # read while the clocks are still up
        finally:
            for pr in procs.values():
                try:
                    pr.stdin.write('quit\n')
                    pr.stdin.flush()
                except OSError:
                    pass
                pr.wait(timeout=60)
        same = {c: bool(torch.equal(torch.load(os.path.join(tmp, 'v1', c + '.pt')), torch.load(os.path.join(tmp, 'regs', c + '.pt'))))
                for c in CASES}
    flops = 2.0 * B * HW * HW * COUT * 9 * CIN
    layers = []
    for c in CASES:
        out_px = (HW // 2) ** 2 if c == 'pool' else HW * HW
        nbytes = B * HW * HW * CIN * 2 + B * out_px * COUT * 2
        row = dict(layer='layers1.2' + (' + 2x2 max-pool' if c == 'pool' else ''), shape='%dx%d cin%d cout%d k3 batch %d' % (HW, HW, CIN, COUT, B),
                   bit_identical=same[c], compute_bound_us=flops / PEAK_TFLOPS / 1e6, hbm_bound_us=nbytes / PEAK_TBS / 1e6, hbm_mb=nbytes / 1e6)
        for f in forms:
            v = times[f][c]
            row[f] = dict(us=statistics.median(v), us_min_max=[min(v), max(v)], tflops=flops / statistics.median(v) / 1e6,
                          trace=trace_stats(ready[f]['traces'][c], f == 'v1'))
        row['speedup'] = row['v1']['us'] / row['regs']['us']
        layers.append(row)
    print(json.dumps(dict(tool='conv_c32_layers', gpu=gpu, rounds=args.rounds, reps=args.reps, iters=args.iters, layers=layers)))


if __name__ == '__main__':
    main()
