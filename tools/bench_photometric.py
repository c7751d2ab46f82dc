#!/usr/bin/env python
"""Device time of the photometric chain in the reference's order (RandomBlur, BGR2HSV, RandomHue, RandomSaturation, RandomBrightness,
HSV2RGB, RandomGamma; one yb_photometric_batch_u8 launch) on a resized uint8 batch, against the same chain on one host core.

    python tools/bench_photometric.py [--batch 64] [--sizes 416 608] [--window 1.0]

Prints one JSON line: per size, the device time per batch from CUDA events (after a warm-up, over a window of at least `--window`
seconds), the bytes the launch moves (frames in and out, plus the parameter block) and the rate against 3.35 TB/s; the card and its
power limit, read in the same run; and the host time per image of the reference chain restated with cv2 + numpy on one thread."""
import argparse
import configparser
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'yolo2-pytorch_b200'))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
CANONICAL = ['RandomBlur', 'BGR2HSV', 'RandomHue', 'RandomSaturation', 'RandomBrightness', 'HSV2RGB', 'RandomGamma']
AUGMENTATION = {'random_blur': '5 5', 'random_hue': '0 25', 'random_saturation': '0.5 1.5', 'random_brightness': '0.5 1.5',
                'random_gamma': '0.9 1.5'}


def power_limit():
    try:
        idx = os.environ.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0] or '0'
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', idx], capture_output=True,
                             text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def device_time(chain, batch, height, width, window):
    import transform.image as ti
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randint(0, 256, (batch, height, width, 3), dtype=torch.uint8, device='cuda', generator=g)
    dst = torch.empty_like(x)
    seg = chain.segments[0]
    params = torch.from_numpy(chain.params(chain.draw(batch))[0]).cuda()
    for _ in range(20):
        ti.launch(x, dst, seg, params)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters, total_ms = 0, 0.0
    while total_ms < window * 1e3:
        start.record()
        for _ in range(100):
            ti.launch(x, dst, seg, params)
        end.record()
        end.synchronize()
        total_ms += start.elapsed_time(end)
        iters += 100
    per = total_ms / iters * 1e-3
    moved = 2 * x.numel() + params.numel()
    return dict(height=height, width=width, batch=batch, launches=len(chain.segments), device_us_per_batch=round(per * 1e6, 2),
                bytes_moved=int(moved), achieved_GBps=round(moved / per / 1e9, 1), fraction_of_3p35TBps=round(moved / per / HBM_PEAK, 3),
                iterations=iters, window_s=round(total_ms / 1e3, 2))


def host_chain_per_image(height, width, images=20):
    """The reference chain on one core: cv2.blur / cvtColor / split / merge and numpy float64 for the random adjustments and gamma."""
    import cv2
    cv2.setNumThreads(1)
    rng = np.random.RandomState(0)
    frames = [rng.randint(0, 256, (height, width, 3)).astype(np.uint8) for _ in range(images)]
    random.seed(0)

    def chain(image):
        image = cv2.blur(image, (random.randint(1, 5), random.randint(1, 5)))
        hsv = cv2.cvtColor(image, cv2.COLOR_BGR2HSV)
        h, s, v = cv2.split(hsv)
        h = np.clip(h.astype(int) + random.randint(0, 25), 0, 179).astype(np.uint8)
        hsv = cv2.merge((h, s, v))
        h, s, v = cv2.split(hsv)
        s = np.clip(s * random.uniform(0.5, 1.5), 0, 255).astype(np.uint8)
        hsv = cv2.merge((h, s, v))
        h, s, v = cv2.split(hsv)
        v = np.clip(v * random.uniform(0.5, 1.5), 0, 255).astype(np.uint8)
        image = cv2.cvtColor(cv2.merge((h, s, v)), cv2.COLOR_HSV2RGB)
        return np.uint8(((image / 255.0) ** random.uniform(0.9, 1.5)) * 255.0)

    chain(frames[0])
    t0 = time.perf_counter()
    for f in frames:
        chain(f)
    return (time.perf_counter() - t0) / images


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--sizes', type=int, nargs='+', default=[416, 608])
    ap.add_argument('--window', type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_photometric: no CUDA device (this measures the H100 kernel; there is nothing to time without one)')
    import transform
    cfg = configparser.ConfigParser()
    cfg.read_dict({'augmentation': AUGMENTATION})
    chain = transform.get_transform(cfg, ['transform.image.' + n for n in CANONICAL])
    random.seed(0)
    res = dict(metric='photometric_chain', gpu=torch.cuda.get_device_name(), power_limit_w=power_limit(),
               device=[device_time(chain, a.batch, s, s, a.window) for s in a.sizes])
    try:
        res['host_ms_per_image_one_thread'] = {str(s): round(host_chain_per_image(s, s) * 1e3, 2) for s in a.sizes}
    except ImportError:
        res['host_ms_per_image_one_thread'] = None      # cv2 not installed where this ran
    print(json.dumps(res))


if __name__ == '__main__':
    main()
