"""Bi-predictive motion refinement of a whole 3840x2160 10-bit picture: vvb_bipred_search_dev against the reference's members.

Every 8x8 .. 128x128 PU of the picture.  The start vectors come from the device uni chain (vvb_tz_search_dev with the medium preset's settings, then
vvb_frac_search_dev; the quarter-pel result, in internal units, is written into the bi PU list on the device); the other list's prediction is a block of a
second picture.  HAD, fast_sub_pel 1, reduce_tap 2, at bipred search range 1 and 4.  Per range:
  bipred_ms   vvb_bipred_search_dev per shape and per picture, CUDA events around `reps` pictures after a warm-up picture
  member_ms   the member pair (refshim_pattern_search_member then refshim_frac_search_member over the target plane, with the replayed start selection) on
              one host thread, wall clock, Python driving included
  mismatches  PUs where any stage differs from its member (every PU is checked)
Prints one JSON line with the card name and power limit read in the same run.  Needs oracle/_ref (built by build() where the reference sources exist)."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

from me_bench_common import PW, PH, card, pictures, timed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))

CTU, LAM, RANGE = 128, 57.25, 384
MARGIN = CTU + 12                  # the margin the header states for every vector the clip rules allow
SHAPES = (8, 16, 32, 64, 128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    import torch
    import vvenc_b200 as V
    import test_gpu_bipred_search as T
    name, plim = card()
    org, cur, oth, S = pictures(MARGIN, third=True)
    eng = V.CostEngine(0)
    eng.upload_plane(0, org, PW, PH, MARGIN, bit_depth=10); eng.upload_plane(1, cur, PW, PH, MARGIN, bit_depth=10)
    from _libs import refshim
    R = T.ref_setup(refshim())
    stream = torch.cuda.ExternalStream(eng.stream)
    vp = ctypes.c_void_p
    T.LAM = LAM

    # start vectors from the uni chain, left on the device
    rs = np.random.RandomState(4096)
    me = eng.me_par(LAM, 2, 0)
    tz = eng.tz_par(RANGE, PW, PH, CTU, extended=0, fast=1, integer_et=0, first_search_stop=1, sub_shift_mode=1)
    fpar = eng.frac_par(LAM, V.DF_HAD, 2, False, 1)
    jobs = {}
    for s in SHAPES:
        ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
        n = xs.size
        pus = np.zeros(n, dtype=V.TZ_PU_DT)
        pus['x'] = xs.ravel(); pus['y'] = ys.ravel()
        pus['start_hor'] = rs.randint(-48 * 16, 48 * 16 + 1, size=n); pus['start_ver'] = rs.randint(-32 * 16, 32 * 16 + 1, size=n)
        q = lambda v: np.where(v >= 0, (v + 1) >> 2, (v + 2) >> 2)
        pus['pred_hor'] = q(pus['start_hor'].astype(np.int64)); pus['pred_ver'] = q(pus['start_ver'].astype(np.int64))
        d_pus = torch.from_numpy(pus.view(np.uint8).copy()).cuda()
        d_mv = torch.zeros(n * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        d_fr = torch.zeros(n * V.FRAC_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        assert eng.lib.vvb_tz_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), n, s, s, ctypes.byref(me), ctypes.byref(tz), None, 0, vp(d_mv.data_ptr())) == 0
        assert eng.lib.vvb_frac_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), vp(d_mv.data_ptr()), n, s, s, ctypes.byref(fpar), vp(d_fr.data_ptr())) == 0
        eng.synchronize()
        bi = np.zeros(n, dtype=V.BI_PU_DT)
        for f in ('x', 'y', 'pred_hor', 'pred_ver'):
            bi[f] = pus[f]
        bi['bits'] = 9; bi['bcw_idx'] = np.arange(n) % 5
        d_bi = torch.from_numpy(bi.view(np.uint8).copy()).cuda().view(n, 36)
        mvt = d_mv.view(torch.int32).view(-1, 8)[:, :2]
        frt = d_fr.view(torch.int16).view(-1, 8)[:, :4].to(torch.int32)
        d_bi[:, 8:16] = ((mvt * 4 + frt[:, 0:2] * 2 + frt[:, 2:4]) * 4).contiguous().view(torch.uint8).view(n, 8)
        bi = np.frombuffer(d_bi.cpu().numpy().tobytes(), dtype=V.BI_PU_DT).copy()
        pred = np.stack([oth[MARGIN + y:MARGIN + y + s, MARGIN + x:MARGIN + x + s] for x, y in zip(bi['x'], bi['y'])]).astype(np.int16)
        d_pred = torch.from_numpy(pred).cuda()
        d_out = torch.zeros(n * V.BI_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        jobs[s] = dict(n=n, bi=bi, pred=pred, d_bi=d_bi, d_pred=d_pred, d_out=d_out)
    torch.cuda.synchronize()

    res = {'metric': 'bipred_search_picture', 'picture': '%dx%d 10-bit' % (PW, PH), 'pus': int(sum(j['n'] for j in jobs.values())), 'card': name, 'power_limit': plim,
           'starts': 'vvb_tz_search_dev (fast, first-search stop, SearchRange %d) -> vvb_frac_search_dev' % RANGE, 'dfunc': 'HAD', 'fast_sub_pel': 1,
           'member_threads': 1, 'ranges': []}
    for rng in (1, 4):
        par = eng.bi_par(LAM, rng, PW, PH, CTU, V.DF_HAD, ref_list=1, fast_sub_pel=1, reduce_tap=2)

        def run(s):
            j = jobs[s]
            assert eng.lib.vvb_bipred_search_dev(eng.h, 0, 1, vp(j['d_bi'].data_ptr()), j['n'], s, s, ctypes.byref(par), None, 0, vp(j['d_pred'].data_ptr()),
                                                 vp(j['d_out'].data_ptr())) == 0
        row = {'search_range': rng, 'bipred_ms': {}, 'member_ms': {}, 'mismatches': {}}
        for s in SHAPES:
            row['bipred_ms'][s] = round(timed(eng, stream, lambda: run(s), a.reps), 3)
        row['bipred_picture_ms'] = round(timed(eng, stream, lambda: [run(s) for s in SHAPES], a.reps), 3)
        for s in SHAPES:
            run(s)
        eng.synchronize()
        for s in SHAPES:
            j = jobs[s]
            dev = np.frombuffer(j['d_out'].cpu().numpy().tobytes(), dtype=V.BI_BEST_DT)
            t = time.perf_counter()
            row['mismatches'][s] = T.check_call(R, org, cur, S, 10, j['bi'], np.zeros((0, 2), np.int32), j['pred'], s, s, par, dev)
            row['member_ms'][s] = round((time.perf_counter() - t) * 1e3, 1)
            print('range %d: %dx%d done' % (rng, s, s), file=sys.stderr, flush=True)
        res['ranges'].append(row)
    jobs.clear()
    torch.cuda.synchronize()
    eng.close()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
