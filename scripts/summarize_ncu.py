#!/usr/bin/env python
"""Summarise ncu output under bench_out/ into small markdown files under bench_out/.

    python scripts/summarize_ncu.py <tag> [--rep bench_out/prof.ncu-rep] [--launches bench_out/launches.csv]
"""
import argparse
import csv
import io
import os
import subprocess
from collections import OrderedDict

KEYS = [
    'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
    'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
    'dram__throughput.avg.pct_of_peak_sustained_elapsed',
    'lts__t_bytes.sum', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
    'sm__warps_active.avg.pct_of_peak_sustained_active',
    'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active',
    'sm__inst_executed_pipe_fp64.sum', 'smsp__inst_executed.sum',
    'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
    'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum',
    'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic',
    'launch__grid_size', 'launch__block_size', 'launch__occupancy_limit_shared_mem',
    'smsp__cycles_active.avg', 'sm__cycles_elapsed.avg',
    'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
    'smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio',
    'smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio',
    'smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio',
    'smsp__average_warps_issue_stalled_wait_per_issue_active.ratio',
    'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('tag')
    ap.add_argument('--rep', default=None)
    ap.add_argument('--launches', default=None)
    args = ap.parse_args()
    os.makedirs('bench_out', exist_ok=True)
    if args.rep:
        raw = subprocess.run(['ncu', '-i', args.rep, '--page', 'raw', '--csv'],
                             capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(raw)))
        hdr, units = rows[0], rows[1]
        out = os.path.join('bench_out', args.tag + '_ncu_full.md')
        with open(out, 'w') as f:
            f.write('# ncu --set full capture: {}\n\n'.format(args.tag))
            f.write('source: `{}` (per launch; ncu serialises and replays, so compare shares, '
                    'not absolutes)\n\n'.format(args.rep))
            for r in rows[2:]:
                name = r[hdr.index('Kernel Name')]
                f.write('## {}\n\n| metric | value | unit |\n|---|---|---|\n'.format(name))
                for k in KEYS:
                    if k in hdr:
                        f.write('| {} | {} | {} |\n'.format(k, r[hdr.index(k)], units[hdr.index(k)]))
                f.write('\n')
        print('wrote', out)
    if args.launches:
        text = [l for l in open(args.launches) if not l.startswith('==')]
        rows = list(csv.reader(text))
        hdr = rows[0]
        ki = hdr.index('Kernel Name')
        vi = hdr.index('Metric Value')
        agg = OrderedDict()
        for r in rows[1:]:
            if len(r) <= vi:
                continue
            try:
                v = float(r[vi].replace(',', ''))
            except ValueError:
                continue
            a = agg.setdefault(r[ki], [0, 0.0])
            a[0] += 1
            a[1] += v
        total = sum(a[1] for a in agg.values()) or 1.0
        out = os.path.join('bench_out', args.tag + '_launches.md')
        with open(out, 'w') as f:
            f.write('# ncu launch list: {}\n\n'.format(args.tag))
            f.write('`ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, '
                    'serialised: shares matter, not absolutes)\n\n')
            f.write('| kernel | launches | total us | avg us | share |\n|---|---|---|---|---|\n')
            for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
                f.write('| `{}` | {} | {:.1f} | {:.1f} | {:.1%} |\n'.format(
                    k[:110], n, t / 1e3, t / n / 1e3, t / total))
        print('wrote', out)


if __name__ == '__main__':
    main()
