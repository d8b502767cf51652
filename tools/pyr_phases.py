#!/usr/bin/env python3
"""phase split of the in-CTA SAD pyramid (pyramid_kernels.cuh) on the bench geometry (3840x2160, 8/16/32/64, +-32)

Builds the -DVVB_PYR_PHASES variant of the library into OUT (default: a temporary directory), runs vvb_sad_search_pyramid_dev on it like
tools/pyr_bench.py and prints, per root level, the mean microseconds per root of each phase (thread 0's %globaltimer at the CTA's barriers):
geometry, staging, prologue compute, candidate loop, argmin, results.  'cta_slot_us_per_root' is the call's wall time times the SM count over the
roots of all levels: what a root costs an SM, so the part of it no phase covers is CTA turnaround and the short last wave.  The phase build adds one
barrier per root (before the results mark); its call time is printed next to the phase sums and is not the shipped library's time.
usage: python tools/pyr_phases.py [--out DIR | --lib PHASE_BUILD.so] [--reps N]"""
import argparse, ctypes, json, os, re, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vvenc_b200', 'csrc')
PHASES = ('geometry', 'staging', 'prologue', 'candidates', 'argmin', 'results')


def build(out):
    mk = open(os.path.join(CSRC, 'Makefile')).read()
    var = {k: v.strip() for k, v in re.findall(r'^(\w+)\s*:?=\s*(.*)$', mk, flags=re.M)}
    flags = var['FLAGS'].replace('$(ARCH)', var['ARCH']).split()
    nvcc = os.environ.get('NVCC') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else 'nvcc')
    lib = os.path.abspath(os.path.join(out, 'libvvenc_b200_phases.so'))
    with open(os.path.join(out, 'build_phases.log'), 'w') as log:
        subprocess.check_call([nvcc] + flags + ['-DVVB_PYR_PHASES', '-shared', '-cudart', 'static', '-o', lib, 'capi.cu'], cwd=CSRC, stderr=log)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--lib', default=None, help='a phase build made earlier by this tool (skips the two-minute compile)')
    a = ap.parse_args()
    if a.lib:
        os.environ['VVENC_B200_LIB'] = os.path.abspath(a.lib)
    else:
        out = a.out or tempfile.mkdtemp(prefix='pyr_phases_')
        os.makedirs(out, exist_ok=True)
        os.environ['VVENC_B200_LIB'] = build(out)
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import bench as B
    import vvenc_b200 as V
    eng = V.CostEngine(0)
    lib = eng.lib
    lib.vvb_pyr_phases_read.restype = ctypes.c_int
    lib.vvb_pyr_phases_read.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    acc = np.zeros((3, len(PHASES) + 1), dtype=np.uint64)
    sets = []
    for s in range(4):
        org, ref, S = B.synth_picture_pair(1234 + 17 * s)
        dorg = torch.from_numpy(org).cuda(); dref = torch.from_numpy(ref).cuda()
        base = (B.MARGIN * S + B.MARGIN) * 2
        eng.bind_plane_dev(2 * s, dorg.data_ptr() + base, S, B.W, B.H, B.MARGIN, 10); eng.bind_plane_dev(2 * s + 1, dref.data_ptr() + base, S, B.W, B.H, B.MARGIN, 10)
        sets.append((dorg, dref))
    d_blocks, d_best, counts = [], [], []
    for n in B.SIZES:
        xs, ys = B.block_grid(n)
        b = np.zeros(len(xs), dtype=V.BLOCK_DT)
        b['x'] = xs; b['y'] = ys; b['left'] = -32; b['right'] = 32; b['top'] = -32; b['bottom'] = 32
        d_blocks.append(torch.from_numpy(np.frombuffer(b.tobytes(), dtype=np.uint8).copy()).cuda()); d_best.append(torch.empty(len(b) * 16, dtype=torch.uint8, device='cuda')); counts.append(len(b))
    pb = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in d_blocks]); po = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in d_best]); cn = (ctypes.c_int * 4)(*counts)
    me = eng.me_par(B.LAMBDA, 2, 0, 0, 1, 2)

    def run(i):
        s = i % 4
        rc = lib.vvb_sad_search_pyramid_dev(eng.h, 2 * s, 2 * s + 1, 4, pb, cn, 8, ctypes.byref(me), 65, 65, po)
        assert rc == 0, lib.vvb_last_error(eng.h)
    for i in range(4):
        run(i)
    assert lib.vvb_pyr_phases_read(eng.h, acc.ctypes.data) == 0           # drop the warm-up's sums
    ext = torch.cuda.ExternalStream(eng.stream)
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(ext):
        e0.record(ext)
        for i in range(a.reps):
            run(i)
        e1.record(ext)
    eng.synchronize(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.reps
    assert lib.vvb_pyr_phases_read(eng.h, acc.ctypes.data) == 0
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    roots_all = int(acc[:, -1].sum()) / a.reps
    res = {'gpu': torch.cuda.get_device_name(0), 'sms': sms, 'reps': a.reps, 'phase_build_call_ms': round(ms, 4),
           'cta_slot_us_per_root': round(ms * 1e3 * sms / max(roots_all, 1), 3), 'levels': {}}
    for lvl in range(3):
        n = int(acc[lvl, -1])
        if n == 0:
            continue
        us = {p: round(float(acc[lvl, k]) / n / 1e3, 3) for k, p in enumerate(PHASES)}
        tot = sum(us.values())
        res['levels']['%dx%d' % (16 << lvl, 16 << lvl)] = {'roots_per_call': n // a.reps, 'us_per_root': us, 'sum_us': round(tot, 3),
                                                          'share': {p: round(v / tot, 4) for p, v in us.items()}}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
