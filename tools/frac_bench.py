"""Fractional motion refinement of a whole 3840x2160 10-bit picture: vvb_frac_search against the reference's own InterSearch::xPatternSearchFracDIF and the grid path.

Every 8x8 .. 128x128 PU of the picture; the integer vectors come from vvb_tz_search with the medium preset's settings (DIAMOND_FAST, first-search stop,
SearchRange 384) and stay on the device; HAD with reduce_tap 2, at fast_sub_pel 1 and 0.  Per setting:
  frac_ms     vvb_frac_search_dev per shape and per picture, CUDA events around `reps` pictures after a warm-up picture
  grid_ms     vvb_frac_cost_grid_dev on the same PUs (shapes up to 64, the grid's limit), and d2h_ms the copy of its 49-entry tables to the host
  member_ms   refshim_frac_search_member (oracle/_ref) over the same PUs on one host thread (the probe's rig shares one static VVEncCfg), wall clock
  mismatches  PUs whose half / quarter offsets or cost differ from the member's
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

CTU, LAM, RANGE = 128, 57.0, 384
MARGIN = CTU + 12                  # the margin the header states for every vector vvb_tz_search can return
SHAPES = (8, 16, 32, 64, 128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    import torch
    import vvenc_b200 as V
    from _libs import refshim, P, PO
    name, plim = card()
    org, cur, S = pictures(MARGIN)
    base = MARGIN * S + MARGIN
    eng = V.CostEngine(0)
    eng.upload_plane(0, org, PW, PH, MARGIN, bit_depth=10); eng.upload_plane(1, cur, PW, PH, MARGIN, bit_depth=10)
    R = refshim()
    R.refshim_frac_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    R.refshim_set_simd(b'AVX2')
    stream = torch.cuda.ExternalStream(eng.stream)
    vp = ctypes.c_void_p

    # integer vectors: vvb_tz_search_dev with the medium settings, left on the device
    rs = np.random.RandomState(4096)
    me = eng.me_par(LAM, 2, 0)
    tz = eng.tz_par(RANGE, PW, PH, CTU, extended=0, fast=1, integer_et=0, first_search_stop=1, sub_shift_mode=1)
    jobs = {}
    for s in SHAPES:
        ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
        pus = np.zeros(xs.size, dtype=V.TZ_PU_DT)
        pus['x'] = xs.ravel(); pus['y'] = ys.ravel()
        pus['start_hor'] = rs.randint(-48 * 16, 48 * 16 + 1, size=xs.size); pus['start_ver'] = rs.randint(-32 * 16, 32 * 16 + 1, size=xs.size)
        q = lambda v: np.where(v >= 0, (v + 1) >> 2, (v + 2) >> 2)
        pus['pred_hor'] = q(pus['start_hor'].astype(np.int64)); pus['pred_ver'] = q(pus['start_ver'].astype(np.int64))
        d_pus = torch.from_numpy(pus.view(np.uint8).copy()).cuda()
        d_mv = torch.zeros(len(pus) * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        d_out = torch.zeros(len(pus) * V.FRAC_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        assert eng.lib.vvb_tz_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), len(pus), s, s, ctypes.byref(me), ctypes.byref(tz), None, 0, vp(d_mv.data_ptr())) == 0
        eng.synchronize()
        mv = np.frombuffer(d_mv.cpu().numpy().tobytes(), dtype=V.TZ_BEST_DT)
        blk = np.zeros(len(pus), dtype=V.BLOCK_DT)                     # the grid path's blocks: integer vector as start
        blk['x'] = pus['x']; blk['y'] = pus['y']; blk['start_x'] = mv['mv_hor']; blk['start_y'] = mv['mv_ver']
        d_blk = torch.from_numpy(blk.view(np.uint8).copy()).cuda()
        d_tab = torch.zeros(len(pus) * 49, dtype=torch.int32, device='cuda') if s <= 64 else None
        h_tab = torch.zeros(len(pus) * 49, dtype=torch.int32, pin_memory=True) if s <= 64 else None
        mem_blk = np.zeros((len(pus), 8), dtype=np.int32)
        mem_blk[:, 0] = pus['x']; mem_blk[:, 1] = pus['y']; mem_blk[:, 2] = s; mem_blk[:, 3] = s
        mem_blk[:, 4] = mv['mv_hor']; mem_blk[:, 5] = mv['mv_ver']; mem_blk[:, 6] = pus['pred_hor']; mem_blk[:, 7] = pus['pred_ver']
        jobs[s] = dict(n=len(pus), d_pus=d_pus, d_mv=d_mv, d_out=d_out, d_blk=d_blk, d_tab=d_tab, h_tab=h_tab, mem_blk=mem_blk)
    torch.cuda.synchronize()

    res = {'metric': 'frac_search_picture', 'picture': '%dx%d 10-bit' % (PW, PH), 'pus': int(sum(j['n'] for j in jobs.values())), 'card': name, 'power_limit': plim,
           'tz': 'fast, first-search stop, SearchRange %d' % RANGE, 'dfunc': 'HAD', 'reduce_tap': 2, 'member_threads': 1, 'settings': []}
    for fast in (1, 0):
        par = eng.frac_par(LAM, V.DF_HAD, 2, False, fast)

        def frac(s):
            j = jobs[s]
            assert eng.lib.vvb_frac_search_dev(eng.h, 0, 1, vp(j['d_pus'].data_ptr()), vp(j['d_mv'].data_ptr()), j['n'], s, s, ctypes.byref(par), vp(j['d_out'].data_ptr())) == 0

        def grid(s):
            j = jobs[s]
            assert eng.lib.vvb_frac_cost_grid_dev(eng.h, V.DF_HAD, 0, 1, vp(j['d_blk'].data_ptr()), j['n'], s, s, 2, 0, vp(j['d_tab'].data_ptr())) == 0

        def d2h(s):
            j = jobs[s]
            j['h_tab'].copy_(j['d_tab'], non_blocking=True)

        row = {'fast_sub_pel': fast, 'frac_ms': {}, 'grid_ms': {}, 'd2h_ms': {}, 'member_ms': {}, 'mismatches': {}}
        for s in SHAPES:
            row['frac_ms'][s] = round(timed(eng, stream, lambda: frac(s), a.reps), 3)
            if s <= 64:
                row['grid_ms'][s] = round(timed(eng, stream, lambda: grid(s), a.reps), 3)
                with torch.cuda.stream(stream):
                    row['d2h_ms'][s] = round(timed(eng, stream, lambda: d2h(s), a.reps), 3)
        row['frac_picture_ms'] = round(timed(eng, stream, lambda: [frac(s) for s in SHAPES], a.reps), 3)
        row['grid_picture_ms_le64'] = round(timed(eng, stream, lambda: [grid(s) for s in SHAPES if s <= 64], a.reps), 3)
        row['frac_picture_ms_le64'] = round(timed(eng, stream, lambda: [frac(s) for s in SHAPES if s <= 64], a.reps), 3)
        for s in SHAPES:
            frac(s)
        eng.synchronize()
        for s in SHAPES:
            j = jobs[s]
            out = np.zeros((j['n'], 6), dtype=np.int32)
            t = time.perf_counter()
            R.refshim_frac_search_member(1, PO(org, base), S, PO(cur, base), S, P(j['mem_blk']), j['n'], 10, LAM, 2, 1, 0, fast, P(out))
            row['member_ms'][s] = round((time.perf_counter() - t) * 1e3, 1)
            got = np.frombuffer(j['d_out'].cpu().numpy().tobytes(), dtype=V.FRAC_BEST_DT)
            cost = (out[:, 4].astype(np.int64) & 0xffffffff) | (out[:, 5].astype(np.int64) << 32)
            same = (got['half_hor'] == out[:, 0]) & (got['half_ver'] == out[:, 1]) & (got['qter_hor'] == out[:, 2]) & (got['qter_ver'] == out[:, 3]) & \
                   (got['cost'].astype(np.int64) == cost)
            row['mismatches'][s] = int((~same).sum())
            print('fast %d: %dx%d done' % (fast, s, s), file=sys.stderr, flush=True)
        row['member_picture_ms'] = round(sum(row['member_ms'].values()), 1)
        res['settings'].append(row)
    # release the page-locked tables while the CUDA context is alive: torch's host cache would otherwise query their copy events at interpreter exit, after
    # the context is gone, and abort
    jobs.clear(); j = None
    torch.cuda.synchronize()
    torch._C._host_emptyCache()
    eng.close()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
