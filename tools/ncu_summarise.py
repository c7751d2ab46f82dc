#!/usr/bin/env python
"""Summarise `ncu --page raw --csv` tables (tools/ncu_capture.sh) into a compact markdown table:
    python tools/ncu_summarise.py gpurun_out/ncu_infer_raw.csv > profiles/rNN_ncu_infer_full.md"""
import csv
import re
import sys

COLS = [('gpu__time_duration.sum', 'us', 1e-3), ('sm__inst_executed_pipe_tensor.sum', None, None),
        ('sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active', 'tensor pipe %', 1.0),
        ('sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'tensor pipe %', 1.0),
        ('dram__bytes_read.sum', 'DRAM rd MB', None), ('dram__bytes_write.sum', 'DRAM wr MB', None),
        ('dram__throughput.avg.pct_of_peak_sustained_elapsed', 'dram %', 1.0), ('lts__throughput.avg.pct_of_peak_sustained_elapsed', 'L2 %', 1.0),
        ('sm__throughput.avg.pct_of_peak_sustained_elapsed', 'SM %', 1.0), ('launch__registers_per_thread', 'regs', 1.0)]


def to_bytes(value, unit):
    mult = {'byte': 1, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}.get(unit, 1)
    return float(value.replace(',', '')) * mult


def main(path):
    rows = list(csv.reader(open(path)))
    start = next(i for i, r in enumerate(rows) if r and r[0] == 'ID')
    header, units = rows[start], rows[start + 1]
    idx = {name: i for i, name in enumerate(header)}
    tensor_key = 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active'
    tensor_el = 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed'
    dram_key = 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed'
    print('| kernel | grid | us | tensor pipe % of peak while SM active | tensor pipe % of peak, whole launch | DRAM rd MB | DRAM wr MB | DRAM GB/s | dram % | L2 % | SM % | regs |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|')
    tot_us = tot_rd = tot_wr = 0.0
    n = 0
    conv = [0, 0.0, 0.0]      # launches, bytes, us of the wgmma conv family (conv_igemm + conv_c32)
    for r in rows[start + 2:]:
        if len(r) < len(header):
            continue
        name = re.sub(r'\(.*', '', r[idx['Kernel Name']]).replace('void yb::', '').replace('yb::', '')

        def num(key):
            return float(r[idx[key]].replace(',', '')) if key in idx and r[idx[key]] not in ('', 'n/a') else float('nan')
        dur = num('gpu__time_duration.sum')
        dur_us = dur / 1e3 if units[idx['gpu__time_duration.sum']] in ('ns', 'nsecond') else (dur if units[idx['gpu__time_duration.sum']] in ('us', 'usecond') else dur * 1e3)
        rd = to_bytes(r[idx['dram__bytes_read.sum']], units[idx['dram__bytes_read.sum']]) / 1e6
        wr = to_bytes(r[idx['dram__bytes_write.sum']], units[idx['dram__bytes_write.sum']]) / 1e6
        tens = num(tensor_key)
        if 'conv_igemm_kernel' in name or 'conv_c32_kernel' in name:
            conv[0] += 1; conv[1] += (rd + wr) * 1e6; conv[2] += dur_us
        print('| %s | %s | %.1f | %.1f | %.1f | %.1f | %.1f | %.0f | %.1f | %.1f | %.1f | %d |' % (
            name[:60], r[idx['Grid Size']], dur_us, tens, num(tensor_el), rd, wr, (rd + wr) * 1e6 / (dur_us * 1e-6) / 1e9 if dur_us > 0 else 0.0, num(dram_key),
            num('lts__throughput.avg.pct_of_peak_sustained_elapsed'), num('sm__throughput.avg.pct_of_peak_sustained_elapsed'),
            int(num('launch__registers_per_thread'))))
        tot_us += dur_us; tot_rd += rd; tot_wr += wr; n += 1
    print()
    print('Totals over %d launches: %.1f us, DRAM read %.1f MB + write %.1f MB = %.1f MB (%.1f MB per launch).' % (n, tot_us, tot_rd, tot_wr, tot_rd + tot_wr, (tot_rd + tot_wr) / max(n, 1)))
    if conv[0]:
        print('wgmma conv family (conv_igemm_kernel + conv_c32_kernel): %d launches, %.1f us = %.3f of the listed kernel time, DRAM %.1f MB per launch.'
              % (conv[0], conv[2], conv[2] / max(tot_us, 1e-9), conv[1] / conv[0] / 1e6))
    if len(sys.argv) > 2:       # traffic.json for bench.py's roofline.traffic
        import json
        with open(sys.argv[2], 'w') as f:
            json.dump(dict(conv_family_dram_bytes_per_launch=(conv[1] / conv[0]) if conv[0] else None, conv_family_launches=conv[0],
                           conv_family_share_of_listed_time=(conv[2] / tot_us) if tot_us else None,
                           source='%s: dram__bytes_read.sum + dram__bytes_write.sum of the wgmma conv launches of one B=32 inference step (ncu --set full)' % sys.argv[3]
                           if len(sys.argv) > 3 else None), f, indent=1)


if __name__ == '__main__':
    main(sys.argv[1])
