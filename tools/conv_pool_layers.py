#!/usr/bin/env python
"""Per-launch timing of the fused conv + 2x2 max-pool (conv_wide_pool_kernel) against the conv followed by yb_maxpool2x2_f16, for the
two pooled 3x3 layers of the C2 forward that run on the two-consumer tile: layers1.6 (104x104, 64 -> 128) and layers1.10 (52x52,
128 -> 256), batch 32, seeded inputs and weights.

Each form is a CUDA graph of --reps back-to-back launches, replayed --iters times between CUDA events; the forms alternate over --rounds
rounds in one process and the median per launch is reported.  Also checks that the fused output equals conv + pool bit for bit.
Prints ONE JSON line (gpu: name, power limit, max and current SM clock read in the same run).

    python tools/conv_pool_layers.py

Writes nothing to the source tree.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layers import gpu_info  # noqa: E402  (puts the product package on sys.path)

LAYERS = [('layers1.6', 104, 64, 128), ('layers1.10', 52, 128, 256)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    import torch
    from b200 import ops
    dev = 'cuda'
    gen = torch.Generator().manual_seed(0)
    out = dict(gpu=gpu_info(), batch=args.batch, layers=[])
    for name, hw, cin, cout in LAYERS:
        b = args.batch
        x = (torch.randn(b, hw, hw, cin, generator=gen)).half().to(dev)
        w = (torch.randn(cout, cin, 3, 3, generator=gen) * (2.0 / (cin * 9)) ** 0.5).to(dev)
        w16 = ops.pack_weight_f16(w)
        scale = (torch.rand(cout, generator=gen) + 0.5).to(dev)
        shift = (torch.randn(cout, generator=gen) * 0.1).to(dev)
        full = torch.empty(b, hw, hw, cout, dtype=torch.float16, device=dev)
        pooled = torch.empty(b, hw // 2, hw // 2, cout, dtype=torch.float16, device=dev)
        fused = torch.empty_like(pooled)
        ws = ops.conv_workspace(dev)
        forms = {
            'conv': lambda: ops.conv_bn_act(x, w16, scale, shift, 0.1, out=full, workspace=ws),
            'pool': lambda: ops.maxpool2x2(full, out=pooled),
            'fused': lambda: ops.conv_bn_act(x, w16, scale, shift, 0.1, out=fused, flags=ops.CONV_POOL2X2, workspace=ws),
        }
        graphs = {}
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for k, fn in forms.items():
                fn()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    for _ in range(args.reps):
                        fn()
                graphs[k] = g
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        same = bool(torch.equal(fused.view(torch.int16), pooled.view(torch.int16)))
        times = {k: [] for k in forms}
        for _ in range(args.rounds):
            for k, g in graphs.items():
                g.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    g.replay()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / (args.iters * args.reps))
        us = {k: statistics.median(v) for k, v in times.items()}
        spread = {k: [min(v), max(v)] for k, v in times.items()}
        pool_bytes = b * hw * hw * cout * 2 * 5 // 4
        out['layers'].append(dict(layer=name, shape='%dx%d cin%d cout%d k3' % (hw, hw, cin, cout), choice=ops.conv_choice(b, hw, hw, cin, cout, 3,
                                  flags=ops.CONV_POOL2X2), bit_identical=same, us=us, us_min_max=spread,
                                  conv_plus_pool_us=us['conv'] + us['pool'], saved_us=us['conv'] + us['pool'] - us['fused'],
                                  pool_gbs=pool_bytes / us['pool'] / 1e3))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
