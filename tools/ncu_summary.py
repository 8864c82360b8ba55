#!/usr/bin/env python
"""Summarise an .ncu-rep (or an ncu --csv launch list) into a small text file
for profiles/.   usage: ncu_summary.py <file.ncu-rep|launches.csv> [out.txt]"""
import collections
import csv
import io
import re
import subprocess
import sys

KEYS = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tensor.sum', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size',
        'launch__shared_mem_per_block_dynamic', 'launch__shared_mem_per_block_static',
        'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum',
        'smsp__inst_executed.sum', 'dram__cycles_active.avg.pct_of_peak_sustained_elapsed']


def rep_summary(path):
    raw = subprocess.run(['ncu', '-i', path, '--page', 'raw', '--csv'], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    out = ['# %s  (ncu --set full --clock-control none; per launch, cold cache, serialised)' % path]
    try:                                   # stamp: which kernel sources the summary was captured from (bench.kernel_source_hash)
        import os
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        from bench import kernel_source_hash
        out.append('# source_sha256: ' + kernel_source_hash())
    except Exception:
        pass
    for r in rows[2:]:
        out.append('kernel: ' + r[hdr.index('Kernel Name')][:150])
        for k in KEYS:
            if k in hdr:
                out.append('  %-70s %s %s' % (k, r[hdr.index(k)], units[hdr.index(k)]))
        out.append('')
    return '\n'.join(out)


def launches_summary(path):
    lines = [l for l in open(path) if not l.startswith('==')]
    agg = collections.OrderedDict()
    for row in csv.DictReader(lines):
        if row.get('Metric Name') != 'gpu__time_duration.sum':
            continue
        name = re.sub(r'\(.*', '', row['Kernel Name'])
        name = re.sub(r'void |<unnamed>::', '', name)[:70]
        v = float(row['Metric Value'].replace(',', ''))
        v *= {'ns': 1e-3, 'us': 1.0, 'ms': 1e3, 's': 1e6}.get(row['Metric Unit'], 1.0)
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(v[1] for v in agg.values()) or 1.0
    out = ['# %s  (ncu --metrics gpu__time_duration.sum --clock-control none; cold-cache serialised launches: compare SHARES)' % path,
           '%-72s %6s %12s %7s %10s' % ('kernel', 'n', 'total_us', 'share', 'avg_us')]
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        out.append('%-72s %6d %12.1f %6.1f%% %10.1f' % (k, v[0], v[1], 100 * v[1] / tot, v[1] / v[0]))
    return '\n'.join(out)


if __name__ == '__main__':
    p = sys.argv[1]
    text = rep_summary(p) if p.endswith('.ncu-rep') else launches_summary(p)
    if len(sys.argv) > 2:
        open(sys.argv[2], 'w').write(text + '\n')
    print(text)
