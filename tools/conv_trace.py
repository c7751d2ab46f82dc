#!/usr/bin/env python
"""Per-tile pipeline trace of the two-consumer conv tile (conv_wide_kernel) on the C2 forward (Darknet-19, 416x416, batch 32,
precision 'fast').

Every implicit-GEMM launch of one forward that runs on conv_wide_kernel is made once with the trace buffer set
(yb_conv_set_trace), after a warm-up of the same launch.  Block 0 records clock64() at, per tile of its work list:

  producer   role 0: every stage issue (after its empty-barrier wait)
  consumer   role 1: the last K-block's full-barrier wait, the first wgmma issue
             role 2: the K-loop end (every MMA of the tile retired), the epilogue end

(consumer events from consumer 0's first thread).  Prints ONE JSON line:

  gpu        name, power limit, max and current SM clock (nvidia-smi, read right after the traced launches)
  layers[]   per launch: shape, tiles of block 0, K-blocks per tile, per-tile K-loop (first wgmma -> K-loop end), epilogue
             (K-loop end -> epilogue end) and gap (K-loop end -> the next tile's first wgmma: the tensor cores' idle time
             between two tiles) in cycles, and their means in ns at the sampled SM clock
  gap_ns     the mean gap over all traced tiles

    python tools/conv_trace.py
    YB_LIB_PATH=/path/to/other/libyolo2_b200.so python tools/conv_trace.py      # the same on another build

Writes nothing to the source tree.  Reuses bench.py's build_model and conv_layers.py's launch recorder.
"""
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import bench  # noqa: E402  (puts the product package on sys.path)
import conv_layers  # noqa: E402

SLOTS = 256          # per role (include/yolo2_b200.h: 768 x uint64)


def per_tile(buf):
    """Per-tile event times of block 0 from the trace buffer [3][256] (0 = not written)."""
    prod, cons, epi = buf[0], buf[1], buf[2]
    tiles = []
    for i in range(SLOTS // 2):
        first, kend = int(cons[2 * i + 1]), int(epi[2 * i])
        if first == 0 or kend == 0:
            break
        tiles.append(dict(last_full=int(cons[2 * i]), first_wgmma=first, kloop_end=kend, epi_end=int(epi[2 * i + 1])))
    issues = [int(v) for v in prod if int(v) != 0]
    return tiles, issues


def mean_ns(cycles, mhz):
    return sum(cycles) / len(cycles) * 1e3 / mhz if cycles and mhz else None


def trace_launch(call, trace, warm):
    import torch
    from b200 import lib, ops
    a, kw = call
    for _ in range(warm):
        ops.conv_bn_act(*a, **kw)
    trace.zero_()
    torch.cuda.synchronize()
    lib.load().yb_conv_set_trace(ctypes.c_void_p(trace.data_ptr()))
    try:
        ops.conv_bn_act(*a, **kw)
        torch.cuda.synchronize()
    finally:
        lib.load().yb_conv_set_trace(None)
    return trace.view(3, SLOTS).cpu().numpy().astype('uint64')


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('conv_trace.py needs a CUDA device (there is no CPU fallback)')
    torch.cuda.set_device(0)
    from b200 import ops
    device = torch.device('cuda', 0)
    _, dnn, _ = bench.build_model(device)
    x = torch.rand(conv_layers.B, 3, conv_layers.SIZE, conv_layers.SIZE, generator=torch.Generator().manual_seed(1)).to(device)
    launches = conv_layers.record_launches(dnn, x)
    trace = torch.zeros(3 * SLOTS, dtype=torch.int64, device=device)
    raw = []
    for key, call in launches:
        a, kw = call
        xx, w = a[0], a[1]
        b, h, wd, _ = xx.shape
        cout, k, _, cin = w.shape
        ch = ops.conv_choice(b, h, wd, cin, cout, k, kw.get('out_mode', ops.OUT_F16_NHWC), kw.get('flags', 0),
                             workspace=kw.get('workspace') is not None)
        if ch['kernel'] != 'conv_wide_kernel':
            continue
        raw.append((key, '%dx%d cin%d cout%d k%d' % (h, wd, cin, cout, k), ch, k * k * cin // ch['bk'], trace_launch(call, trace, 20)))
    gpu = conv_layers.gpu_info()          # read while the clocks are still up
    mhz = float(gpu.get('clocks.sm') or 0) or float(gpu.get('clocks.max.sm') or 0)
    layers, gaps_all = [], []
    for key, shape, ch, num_kb, buf in raw:
        tiles, issues = per_tile(buf)
        kloop = [t['kloop_end'] - t['first_wgmma'] for t in tiles]
        epi = [t['epi_end'] - t['kloop_end'] for t in tiles if t['epi_end']]
        gaps = [tiles[i + 1]['first_wgmma'] - tiles[i]['kloop_end'] for i in range(len(tiles) - 1)]
        gaps_all += gaps
        layers.append(dict(layer=key, shape=shape, choice=ch, kb_per_tile=num_kb, tiles=len(tiles), stage_issues=len(issues),
                           kloop_cycles=kloop, epi_cycles=epi, gap_cycles=gaps,
                           kloop_ns=mean_ns(kloop, mhz), epi_ns=mean_ns(epi, mhz), gap_ns=mean_ns(gaps, mhz)))
    line = dict(tool='conv_trace', lib=os.environ.get('YB_LIB_PATH') or 'in-tree', gpu=gpu, sm_mhz=mhz,
                workload='C2 forward convs on conv_wide_kernel, Darknet-19 %dx%d batch %d, precision fast' % (conv_layers.SIZE, conv_layers.SIZE,
                                                                                                               conv_layers.B),
                gap_ns=mean_ns(gaps_all, mhz), layers=layers)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
