#!/usr/bin/env python
"""Per-launch timing of a conv with the following 1x1 unit run in its epilogue (conv_wide_chain_kernel) against the two separate
launches, for the pair of the C2 forward that has the fused form: layers1.4 (104x104, 3x3, 64 -> 128) -> layers1.5 (1x1, 128 -> 64),
batch 32, seeded inputs and weights.

Each form is a CUDA graph of --reps back-to-back launches, replayed --iters times between CUDA events; the forms alternate over --rounds
rounds in one process and the median per launch is reported.  Also checks that the fused output equals the two launches bit for bit.
Prints ONE JSON line (gpu: name, power limit, max and current SM clock read in the same run).

    python tools/conv_chain_layers.py

Writes nothing to the source tree.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layers import gpu_info  # noqa: E402  (puts the product package on sys.path)

# name of the pair, H = W, producer k, Cin, Cout, consumer Cout
PAIRS = [('layers1.4+layers1.5', 104, 3, 64, 128, 64)]


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
    out = dict(gpu=gpu_info(), batch=args.batch, pairs=[])

    def unit(cin, cout, k):
        w = (torch.randn(cout, cin, k, k, generator=gen) * (2.0 / (cin * k * k)) ** 0.5).to(dev)
        return ops.pack_weight_f16(w), (torch.rand(cout, generator=gen) + 0.5).to(dev), (torch.randn(cout, generator=gen) * 0.1).to(dev)

    for name, hw, k, cin, cout, cout2 in PAIRS:
        b = args.batch
        x = (torch.randn(b, hw, hw, cin, generator=gen)).half().to(dev)
        wa, sa, ha = unit(cin, cout, k)
        wc, sc, hc = unit(cout, cout2, 1)
        mid = torch.empty(b, hw, hw, cout, dtype=torch.float16, device=dev)
        sep = torch.empty(b, hw, hw, cout2, dtype=torch.float16, device=dev)
        fused = torch.empty_like(sep)
        ws = ops.conv_workspace(dev)
        forms = {
            'first': lambda: ops.conv_bn_act(x, wa, sa, ha, 0.1, out=mid, workspace=ws),
            'second': lambda: ops.conv_bn_act(mid, wc, sc, hc, 0.1, out=sep, workspace=ws),
            'fused': lambda: ops.conv_bn_act(x, wa, sa, ha, 0.1, out=fused, workspace=ws, chain=(wc, sc, hc, 0.1)),
        }
        graphs = {}
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for key, fn in forms.items():
                fn()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    for _ in range(args.reps):
                        fn()
                graphs[key] = g
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        same = bool(torch.equal(fused.view(torch.int16), sep.view(torch.int16)))
        times = {key: [] for key in forms}
        for _ in range(args.rounds):
            for key, g in graphs.items():
                g.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    g.replay()
                e1.record()
                e1.synchronize()
                times[key].append(e0.elapsed_time(e1) * 1e3 / (args.iters * args.reps))
        us = {key: statistics.median(v) for key, v in times.items()}
        spread = {key: [min(v), max(v)] for key, v in times.items()}
        out['pairs'].append(dict(pair=name, shape='%dx%d cin%d k%d -> %d -> 1x1 -> %d' % (hw, hw, cin, k, cout, cout2),
                                 choice=ops.conv_choice(b, hw, hw, cin, cout, k, flags=ops.CONV_CHAIN1X1), bit_identical=same, us=us,
                                 us_min_max=spread, separate_us=us['first'] + us['second'], saved_us=us['first'] + us['second'] - us['fused']))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
