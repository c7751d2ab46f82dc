#!/usr/bin/env python
"""Per-launch timing of the implicit-GEMM conv family in the C2 forward (Darknet-19, 416x416, batch 32, precision 'fast').

The 22 conv launches of one forward (21 implicit-GEMM launches and the Cin = 32 halo-tile launch) are recorded from an eager
pass of bench.py's model; each is then timed ALONE: a CUDA graph of --reps back-to-back launches of it, replayed --iters times
between CUDA events.  Prints ONE JSON line:

  gpu         name, power limit and max SM clock (nvidia-smi --query-gpu, read in the same run)
  layers[]    per launch: shape, the library's choice (yb_conv_choice: kernel, BK, BLOCK_N, rows per tile, stream-K, grid,
              waves = tiles / SMs), us, algorithmic TFLOP/s (2 Cin Cout k^2 per output pixel)
  --force S   time the tile shape S instead of the library's choice on every implicit-GEMM launch: BNxROWS with an optional
              "sk" (stream-K forced) suffix, e.g. 128x128, 128x256sk; the existing force flags, nothing else changes
  --all       also time every shape (64x128, 128x128, 64x256, 128x256, each with and without stream-K) of every launch
  --ab        alternate the library's choice with the shape the one-warpgroup kernel's model picked before the 256 x 128 tile
              existed (PRE_CHANGE below) on every launch, --rounds times in the same process

    python tools/conv_layers.py --ab

Writes nothing to the source tree.  Reuses bench.py's build_model (bench.py itself is unchanged).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the product package on sys.path)

B, SIZE = 32, 416
# (BLOCK_N, rows per tile, stream-K) the dispatcher chose for the 21 implicit-GEMM launches of C2, in launch order, before the
# two-consumer kernel existed: its cost model evaluated for 132 SMs with a stream-K workspace
PRE_CHANGE = [(128, 128, 0), (64, 256, 0), (128, 128, 0),                            # 104x104
              (128, 128, 0), (128, 128, 0), (128, 128, 0),                           # 52x52
              (128, 128, 0), (128, 128, 0), (128, 128, 0), (128, 128, 0), (128, 128, 0), (64, 256, 0),    # 26x26, passthrough
              (128, 128, 0), (128, 128, 0), (128, 128, 0), (128, 128, 0), (128, 128, 0), (128, 128, 0),   # 13x13 trunk
              (128, 128, 0), (128, 128, 0), (128, 128, 1)]                          # layers3: 3x3 on the concat, the head
ALL_SHAPES = [(bn, rows, sk) for bn, rows in ((64, 128), (128, 128), (64, 256), (128, 256)) for sk in (0, 1)]


def gpu_info():
    q = 'name,power.limit,clocks.max.sm,clocks.sm'
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True)
    vals = [v.strip() for v in r.stdout.strip().split(',')] if r.returncode == 0 else []
    return dict(zip(q.split(','), vals)) if len(vals) == 4 else dict(error=r.stderr.strip())


def shape_flags(ops, bn, rows, sk):
    return ops.conv_force_bn(bn) | ops.conv_force_mt(rows // 128) | (ops.CONV_FORCE_STREAMK if sk else ops.CONV_NO_STREAMK)


def parse_shape(s):
    sk = s.endswith('sk')
    bn, rows = s[:-2 if sk else None].split('x')
    return int(bn), int(rows), int(sk)


def record_launches(dnn, x):
    """(key, positional args, keyword args) of every ops.conv_bn_act call of one eager forward, in order."""
    from b200 import ops
    calls = []
    orig = ops.conv_bn_act

    def rec(*a, **kw):
        calls.append((a, dict(kw)))
        return orig(*a, **kw)
    ops.conv_bn_act = rec
    try:
        dnn.engine.forward(x)
    finally:
        ops.conv_bn_act = orig
    e = dnn.engine
    keys = e._k1[1:] + ['passthrough'] + e._k2 + ['layers3.0', 'layers3.1']      # launch order of DarknetEngine.forward
    if len(calls) != len(keys):
        raise RuntimeError('expected %d conv launches, recorded %d' % (len(keys), len(calls)))
    return list(zip(keys, calls))


def time_launch(call, flags, reps, iters):
    import torch
    from b200 import ops
    a, kw = call
    kw = dict(kw, flags=kw.get('flags', 0) | flags)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            ops.conv_bn_act(*a, **kw)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(reps):
                ops.conv_bn_act(*a, **kw)
        g.replay()
        s.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(iters):
            g.replay()
        e1.record(s)
        e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--force', default=None)
    ap.add_argument('--all', action='store_true')
    ap.add_argument('--ab', action='store_true')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('conv_layers.py needs a CUDA device (there is no CPU fallback)')
    torch.cuda.set_device(0)
    from b200 import ops
    device = torch.device('cuda', 0)
    _, dnn, _ = bench.build_model(device)
    x = torch.rand(B, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(1)).to(device)
    launches = record_launches(dnn, x)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    forced = parse_shape(args.force) if args.force else None
    layers = []
    igemm = 0
    for key, call in launches:
        a, kw = call
        xx, w = a[0], a[1]
        b, h, wd, _ = xx.shape
        cout, k, _, cin = w.shape
        out_mode = kw.get('out_mode', ops.OUT_F16_NHWC)
        base = kw.get('flags', 0)
        flops = 2.0 * b * h * wd * cin * cout * k * k
        halo = cin == 32 and k == 3 and (base & ops.CONV_POOL2X2)
        flags = 0 if (forced is None or halo) else shape_flags(ops, *forced)
        try:
            ch = ops.conv_choice(b, h, wd, cin, cout, k, out_mode, base | flags, workspace=kw.get('workspace') is not None)
        except RuntimeError:
            # the forced shape is not a form of this launch (e.g. 128 x 256 on the fp32 head): time the library's choice
            flags = 0
            ch = ops.conv_choice(b, h, wd, cin, cout, k, out_mode, base, workspace=kw.get('workspace') is not None)
        if forced is not None and not halo:
            ch['forced'] = flags != 0
        tiles = -(-b * h * wd // ch['rows']) * -(-cout // ch['bn'])
        rec = dict(layer=key, shape='%dx%d cin%d cout%d k%d' % (h, wd, cin, cout, k), batch=b, choice=ch, tiles=tiles, waves=tiles / sms,
                   cluster=False, gflop=flops / 1e9)
        us = time_launch(call, flags, args.reps, args.iters)
        rec.update(us=us, tflops=flops / us / 1e6)
        if args.all and not halo:
            rec['shapes'] = {}
            for bn, rows, sk in ALL_SHAPES:
                f = shape_flags(ops, bn, rows, sk)
                try:
                    c = ops.conv_choice(b, h, wd, cin, cout, k, out_mode, base | f, workspace=kw.get('workspace') is not None)
                except RuntimeError:
                    continue      # not a shape of this launch (e.g. 128 x 256 on the fp32 head)
                if (c['bn'], c['rows'], int(c['streamk'])) != (bn, rows, sk):
                    continue      # stream-K refused (too few K-blocks per CTA)
                rec['shapes']['%dx%d%s' % (bn, rows, 'sk' if sk else '')] = time_launch(call, f, args.reps, args.iters)
        if args.ab and not halo:
            pre_shape = PRE_CHANGE[igemm]
            pre = shape_flags(ops, *pre_shape)
            chosen, before = [], []
            for _ in range(args.rounds):
                chosen.append(time_launch(call, 0, args.reps, args.iters))
                before.append(time_launch(call, pre, args.reps, args.iters))
            rec['ab'] = dict(pre_change_shape='%dx%d%s' % (pre_shape[0], pre_shape[1], 'sk' if pre_shape[2] else ''),
                             chosen_us=chosen, pre_change_us=before, speedup=min(before) / min(chosen))
        igemm += 0 if halo else 1
        layers.append(rec)
    total_us = sum(r['us'] for r in layers)
    total_gflop = sum(r['gflop'] for r in layers)
    line = dict(tool='conv_layers', workload='C2 forward convs, Darknet-19 %dx%d batch %d, precision fast' % (SIZE, SIZE, B), gpu=gpu_info(),
                sms=sms, force=args.force, total_us=total_us, total_tflops=total_gflop / total_us * 1e3, layers=layers)
    if args.ab:
        line['ab_total'] = dict(chosen_us=sum(min(r['ab']['chosen_us']) for r in layers if 'ab' in r),
                                pre_change_us=sum(min(r['ab']['pre_change_us']) for r in layers if 'ab' in r))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
