#!/usr/bin/env python
"""Cost of dynamic loss scaling on one GPU.  Prints ONE JSON line:

  step_ms       the graphed Darknet-19 training step (64 images at 416x416, fused capturable Adam, train.GraphedStep) in static mode and in
                dynamic mode at factor 1 (the arena pass writes nothing) and at factor 2 (it rescales the whole gradient arena).  One graph
                per mode on the same model; the modes are timed alternately, --rounds times --steps replays each (CUDA events), and the
                median per mode is reported with every round's figure.  found_inf of each mode's last replay is reported too: an
                overflowed step skips the Adam update and is not the step being measured.
  pass_us       the gradient arena guard alone on the step's arena (50.6 M fp32 values): yb_grad_guard, and yb_grad_unscale_guard at
                factor 1 and 2, CUDA events over --passes launches; `pass_gbps` is the bytes each must move (4 per value read, 4 more per
                value read and written when the factor is not 1) over that time, `pass_share_of_hbm` that rate over 3.35 TB/s (H100 SXM data
                sheet).
  gpu           the card's name and power limit, read in the same run.

    python tools/bench_loss_scale.py [--steps 20 --rounds 5 --warmup 3 --passes 200]

Writes nothing to the source tree.  Reuses bench.py's workload helpers (model, config, synthetic batches).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the product package on sys.path)

HBM_BYTES_PER_S = 3.35e12


def gpu_info(index):
    import torch
    info = dict(name=torch.cuda.get_device_name(index))
    try:
        r = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        info['power_limit_and_max_sm_clock'] = r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        info['power_limit_and_max_sm_clock'] = 'unavailable: %s' % ex
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--passes', type=int, default=200)
    args = ap.parse_args()
    import torch
    import train as yb_train
    from b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit('bench_loss_scale: needs a CUDA device')
    device = torch.device('cuda', torch.cuda.current_device())
    config, dnn, inference, anchors, optimizer = bench._train_setup(device, capturable=True)
    batches = bench._train_batches(64, 416, 416, device, torch.Generator().manual_seed(200))
    trainer = dnn.trainer
    modes = [('static', None), ('dynamic_f1', 1.0), ('dynamic_f2', 2.0)]
    steps = {}
    for name, f in modes:
        cfg = bench.make_config()
        cfg.read_dict({s: dict(config.items(s)) for s in config.sections()})
        if f is not None:
            cfg.read_dict({'train': {'loss_scale': 'dynamic', 'loss_scale_growth_interval': str(1 << 30)}})
        steps[name] = yb_train.GraphedStep(inference, optimizer, anchors, cfg)

    def set_factor(f):
        if f is not None and trainer.loss_factor is not None:       # created when the first dynamic graph is captured
            trainer.loss_factor.fill_(f)
            trainer.growth_tracker.zero_()

    found = {}
    for name, f in modes:
        for i in range(args.warmup):
            set_factor(f)
            steps[name](batches[i % 2])
    torch.cuda.synchronize()
    times = {name: [] for name, _ in modes}
    for _ in range(args.rounds):
        for name, f in modes:
            set_factor(f)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for i in range(args.steps):
                steps[name](batches[i % 2])
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / args.steps)
            found[name] = float(trainer.found_inf.item())
    factor_after = float(trainer.loss_factor.item())
    for st in steps.values():
        st.close()

    # the arena pass alone, on a buffer the size of the step's arena
    n = trainer.arena.flat.numel()
    buf = torch.randn(n, device=device)
    flag = torch.zeros((), device=device)
    fac = torch.ones((), device=device)
    tracker = torch.zeros((), dtype=torch.int32, device=device)
    passes = {'grad_guard': (lambda: ops.call('yb_grad_guard', buf, n, flag, 1), 4.0),
              'unscale_guard_f1': (lambda: ops.call('yb_grad_unscale_guard', buf, n, flag, fac, tracker, 1 << 30), 4.0),
              'unscale_guard_f2': (lambda: ops.call('yb_grad_unscale_guard', buf, n, flag, fac, tracker, 1 << 30), 12.0)}
    pass_us, pass_gbps, pass_share = {}, {}, {}
    for name, (fn, bytes_per_value) in passes.items():
        fac.fill_(2.0 if name.endswith('f2') else 1.0)
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.passes):
            fn()
        e.record()
        torch.cuda.synchronize()
        us = s.elapsed_time(e) * 1e3 / args.passes
        pass_us[name] = round(us, 2)
        pass_gbps[name] = round(bytes_per_value * n / (us * 1e-6) / 1e9, 1)
        pass_share[name] = round(bytes_per_value * n / (us * 1e-6) / HBM_BYTES_PER_S, 3)
    assert flag.item() == 0.0

    med = {name: statistics.median(v) for name, v in times.items()}
    print(json.dumps(dict(
        workload='darknet19 train step, 64 x 416x416, GraphedStep, fused capturable Adam',
        step_ms={k: round(v, 3) for k, v in med.items()},
        step_ms_rounds={k: [round(x, 3) for x in v] for k, v in times.items()},
        dynamic_over_static={k: round(med[k] / med['static'], 4) for k in med},
        found_inf_last=found, factor_after=factor_after,
        arena_values=n, pass_us=pass_us, pass_gbps=pass_gbps, pass_share_of_hbm=pass_share,
        gpu=gpu_info(device.index))))


if __name__ == '__main__':
    main()
