#!/usr/bin/env python3
"""Turns *.ncu-rep reports / launch CSVs into small text summaries.
usage: tools/ncu_summary.py launches <launches.csv> <out.txt>
       tools/ncu_summary.py kernel   <file.ncu-rep> <out.txt>"""
import csv, collections, re, subprocess, sys

METRICS = ['Kernel Name', 'Grid Size', 'Block Size', 'gpu__time_duration.sum', 'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic',
           'launch__occupancy_limit_shared_mem', 'launch__occupancy_limit_registers', 'sm__warps_active.avg.pct_of_peak_sustained_active',
           'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
           'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'lts__t_bytes.sum', 'lts__t_sector_hit_rate.pct',
           'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'smsp__inst_executed.sum',
           'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
           'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
           'sm__inst_executed_pipe_tensor.sum', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
           'smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio', 'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
           'smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio',
           'smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio',
           'smsp__average_warps_issue_stalled_wait_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio',
           'smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio']


def launches(src, dst):
    rows = [r for r in csv.reader(open(src, errors='ignore')) if len(r) > 5]
    hdr = None; data = []
    for r in rows:
        if r[0] == 'ID':
            hdr = r; continue
        if hdr and r[0].isdigit():
            data.append(dict(zip(hdr, r)))
    agg = collections.OrderedDict()
    for d in data:
        name = re.sub(r'^void ', '', re.sub(r'\(.*', '', d['Kernel Name']))
        t = float(d['Metric Value'].replace(',', '')); u = d['Metric Unit']
        t = t / 1e6 if u == 'ns' else t / 1e3 if u == 'us' else t * 1e3 if u == 's' else t
        key = (name, d['Grid Size'], d['Block Size'])
        a = agg.setdefault(key, [0, 0.0]); a[0] += 1; a[1] += t
    tot = sum(v[1] for v in agg.values())
    with open(dst, 'w') as f:
        f.write('# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised launches: compare SHARES)\n')
        f.write('# %d launches, %.3f ms total\n' % (len(data), tot))
        f.write('%-48s %-16s %-12s %6s %12s %10s %7s\n' % ('kernel', 'grid', 'block', 'n', 'total_ms', 'avg_ms', 'share'))
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write('%-48s %-16s %-12s %6d %12.3f %10.4f %6.1f%%\n' % (k[0][:48], k[1], k[2], v[0], v[1], v[1] / v[0], 100 * v[1] / tot))


def kernel(src, dst):
    out = subprocess.run(['ncu', '-i', src, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    with open(dst, 'w') as f:
        f.write('# ncu --set full --clock-control none --import-source on ; selected raw metrics per captured launch\n')
        for r in rows[2:]:
            f.write('-' * 100 + '\n')
            for m in METRICS:
                if m in idx:
                    f.write('%-82s %s %s\n' % (m, r[idx[m]], units[idx[m]]))


if __name__ == '__main__':
    {'launches': launches, 'kernel': kernel}[sys.argv[1]](sys.argv[2], sys.argv[3])
