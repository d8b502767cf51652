#!/usr/bin/env python
"""Where a kernel's executed instructions and stall samples go, per CUDA source line and per SASS mnemonic, from a saved Nsight Compute report
(captured with --set full --import-source on; the kernels are built with -lineinfo).  Reads the report on the CPU:
    tools/ncu_source_breakdown.py step.ncu-rep sad_search_kernel [top_lines] > src_<kernel>.txt
The kernel is a regex on the demangled name, or id:N for the N-th launch in the report."""
import collections
import csv
import io
import re
import subprocess
import sys


def num(v):
    try:
        return int(v)
    except ValueError:
        return 0


def main():
    rep, kern = sys.argv[1], sys.argv[2]
    sel = ['--kernel-id', ':::' + kern[3:]] if kern.startswith('id:') else ['--kernel-name-base', 'demangled', '--kernel-name', 'regex:' + kern]
    top = int(sys.argv[3]) if len(sys.argv) > 3 else 40
    out = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--print-source', 'cuda,sass', '--csv'] + sel, capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    fpath = None; func = None; seen_funcs = []
    per_line = collections.OrderedDict(); mnem = collections.Counter(); mnem_s = collections.Counter()
    ci = cs = None; first_func = None
    for r in rows:
        if not r:
            continue
        if r[0] == 'File Path':
            fpath = r[1]; continue
        if r[0] == 'Function Name':
            func = r[1]
            if first_func is None:
                first_func = func
            seen_funcs.append(func); continue
        if r[0] == 'Line No':
            ci = r.index('Instructions Executed'); cs = r.index('# Samples'); continue
        if ci is None or func != first_func:
            continue
        if r[0].isdigit():                                   # aggregated source line
            key = (fpath, int(r[0]))
            if key in per_line:
                continue                                     # the report holds one section per launch: keep the first
            per_line[key] = [r[1].strip(), num(r[ci]), num(r[cs])]
    # SASS table of the first launch (sass view) for the mnemonic mix
    out2 = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv'] + sel, capture_output=True, text=True).stdout
    rows2 = list(csv.reader(io.StringIO(out2)))
    h = None; n_tables = 0
    for r in rows2:
        if r and r[0] == 'Address':
            n_tables += 1
            if n_tables > 1:
                break
            h = r; continue
        if h and r and r[0].startswith('0x'):
            m = re.match(r'\s*(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)', r[h.index('Source')])
            k = m.group(1) if m else '?'
            mnem[k] += num(r[h.index('Instructions Executed')]); mnem_s[k] += num(r[h.index('# Samples')])
    tot = sum(mnem.values()) or 1; samp = sum(mnem_s.values()) or 1
    print('# %s -- first launch of a kernel matching "%s"' % (rep, kern))
    print('# %s' % first_func)
    print('# warp instructions executed: %d ; stall samples: %d' % (tot, samp))
    print('\n## SASS mnemonic mix (share of executed warp instructions | share of stall samples)')
    for k, v in mnem.most_common(18):
        print('%-10s %6.2f %%   %6.2f %%' % (k, 100.0 * v / tot, 100.0 * mnem_s[k] / samp))
    ltot = sum(v[1] for v in per_line.values()) or 1; lsamp = sum(v[2] for v in per_line.values()) or 1
    print('\n## CUDA source lines, by executed warp instructions (share of instructions | share of stall samples | file:line | source)')
    print('# lines with correlation cover %.1f %% of the executed warp instructions%s' % (100.0 * ltot / tot, '' if ltot > 0.5 * tot else '  -- INCOMPLETE correlation for this launch: read the mnemonic mix only'))
    for (f, ln), (src, n, s) in sorted(per_line.items(), key=lambda kv: -kv[1][1])[:top]:
        print('%6.2f %%  %6.2f %%  %s:%d  %s' % (100.0 * n / ltot, 100.0 * s / lsamp, f.split('/')[-1], ln, src[:150]))


if __name__ == '__main__':
    main()
