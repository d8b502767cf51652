#!/usr/bin/env python3
"""times vvb_cost_pattern_dev( DF_HAD ) alone on the bench geometry (3840x2160, 4 rotated picture sets, 8/16/32/64, the bench's 18-point ring at
pattern_radius 2, start vectors from one SAD pyramid search per set): tuning aid for had8_ring_kernel (search_kernels.cuh)
usage: python tools/had_bench.py [reps]"""
import ctypes, os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench as B
import vvenc_b200 as V

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
eng = V.CostEngine(0)
lib = eng.lib
ext = torch.cuda.ExternalStream(eng.stream)
P_ = ctypes.c_void_p
sets = []
for s in range(B.N_PICTURE_SETS):
    org, ref, S = B.synth_picture_pair(1234 + 17 * s)
    dorg = torch.from_numpy(org).cuda(); dref = torch.from_numpy(ref).cuda()
    base = (B.MARGIN * S + B.MARGIN) * 2
    eng.bind_plane_dev(2 * s, dorg.data_ptr() + base, S, B.W, B.H, B.MARGIN, B.BITDEPTH); eng.bind_plane_dev(2 * s + 1, dref.data_ptr() + base, S, B.W, B.H, B.MARGIN, B.BITDEPTH)
    sets.append((dorg, dref))
pts = B.refine_pattern()
pat = np.zeros(len(pts), dtype=V.MV_DT); pat['dx'] = [p[0] for p in pts]; pat['dy'] = [p[1] for p in pts]
K = len(pat)
d_pat = torch.from_numpy(np.frombuffer(pat.tobytes(), dtype=np.uint8).copy()).cuda()
me = eng.me_par(B.LAMBDA, 2, 0, 0, 1, 2)
nx = 2 * B.SEARCH_RANGE + 1
counts, d_blocks, d_best, d_cost = [], {}, {}, {}
for n in B.SIZES:
    xs, ys = B.block_grid(n)
    b = np.zeros(len(xs), dtype=V.BLOCK_DT)
    b['x'] = xs; b['y'] = ys; b['left'] = -B.SEARCH_RANGE; b['right'] = B.SEARCH_RANGE; b['top'] = -B.SEARCH_RANGE; b['bottom'] = B.SEARCH_RANGE
    counts.append(len(b))
    d_blocks[n] = [torch.from_numpy(np.frombuffer(b.tobytes(), dtype=np.uint8).copy()).cuda() for _ in sets]     # start vectors differ per set
    d_best[n] = torch.empty(len(b) * 16, dtype=torch.uint8, device='cuda')
    d_cost[n] = [torch.empty(len(b) * K, dtype=torch.int32, device='cuda') for _ in sets]
cn = (ctypes.c_int * len(B.SIZES))(*counts)


def chk(rc):
    assert rc == 0, lib.vvb_last_error(eng.h)


for s in range(len(sets)):                  # start vectors: one pyramid search per picture set
    pb = (P_ * len(B.SIZES))(*[d_blocks[n][s].data_ptr() for n in B.SIZES]); po = (P_ * len(B.SIZES))(*[d_best[n].data_ptr() for n in B.SIZES])
    chk(lib.vvb_sad_search_pyramid_dev(eng.h, 2 * s, 2 * s + 1, len(B.SIZES), pb, cn, B.SIZES[0], ctypes.byref(me), nx, nx, po))
    for n, c in zip(B.SIZES, counts):
        chk(lib.vvb_blocks_set_start_dev(eng.h, P_(d_blocks[n][s].data_ptr()), P_(d_best[n].data_ptr()), c))


def run(i, n, c):
    s = i % len(sets)
    chk(lib.vvb_cost_pattern_dev(eng.h, V.DF_HAD, 2 * s, 2 * s + 1, P_(d_blocks[n][s].data_ptr()), c, n, n, P_(d_pat.data_ptr()), K, ctypes.byref(me),
                                 P_(d_cost[n][s].data_ptr()), None))


for i in range(4):
    for n, c in zip(B.SIZES, counts):
        run(i, n, c)
eng.synchronize()
ms = {}
with torch.cuda.stream(ext):
    for n, c in zip(B.SIZES, counts):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(ext)
        for i in range(reps):
            run(i, n, c)
        e1.record(ext)
        e1.synchronize()
        ms[n] = e0.elapsed_time(e1) / reps
eng.synchronize(); torch.cuda.synchronize()
chk_sum = sum(int(t.to(torch.int64).sum().item()) for n in B.SIZES for t in d_cost[n])
print(json.dumps({'gpu': torch.cuda.get_device_name(0), 'ms': {str(n): round(ms[n], 4) for n in B.SIZES}, 'total_ms': round(sum(ms.values()), 4),
                  'tile_satd_per_s': sum(c * (n // 8) ** 2 * K for n, c in zip(B.SIZES, counts)) / (sum(ms.values()) * 1e-3), 'checksum': chk_sum}))
