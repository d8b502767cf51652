"""AMVR integer refinement of a whole 3840x2160 10-bit picture: vvb_amvr_refine_dev after vvb_tz_search_dev, and the one-call bi branch
vvb_bipred_amvr_search_dev, against the restatement of xPatternSearchIntRefine in tests/test_gpu_amvr_refine.py.

Every 8x8 .. 128x128 PU of the picture, imv 1 (IMV_FPEL) and 2 (IMV_4PEL), HAD, two AMVP candidates per PU.
  tz_ms       vvb_tz_search_dev with the medium preset's settings (fast, first-search stop, SearchRange 384) and imv_shift 2 / 4, per shape
  refine_ms   vvb_amvr_refine_dev on its integer vectors, per shape (refine_over_tz: refine_ms / tz_ms)
  bi_ms       vvb_bipred_amvr_search_dev (bipred search range 4, list 1, every BCW index) with the uni result as start vector, per shape
  mismatches  PUs where the device differs from the restatement (uni) or from refshim_pattern_search_member and the restatement (bi); every PU is checked
Device times are CUDA events around `reps` calls after a warm-up call.  Prints one JSON line with the card name and power limit read in the same run.  Needs
oracle/_ref (built by build() where the reference sources exist)."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

from me_bench_common import PW, PH, card, pictures, timed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))

CTU, LAM, RANGE = 128, 57.25, 384
MARGIN = CTU + 12                  # the bi branch's integer stage needs ctu_size + 12; the refinement ctu_size + 7
SHAPES = (8, 16, 32, 64, 128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    import torch
    import vvenc_b200 as V
    import test_gpu_amvr_refine as T
    from _libs import refshim
    name, plim = card()
    org, cur, oth, S = pictures(MARGIN, third=True)
    assert T.M == MARGIN
    eng = V.CostEngine(0)
    eng.upload_plane(0, org, PW, PH, MARGIN, bit_depth=10); eng.upload_plane(1, cur, PW, PH, MARGIN, bit_depth=10)
    R = T.B.ref_setup(refshim())
    stream = torch.cuda.ExternalStream(eng.stream)
    vp = ctypes.c_void_p
    res = {'metric': 'amvr_refine_picture', 'picture': '%dx%d 10-bit' % (PW, PH), 'card': name, 'power_limit': plim, 'dfunc': 'HAD',
           'tz': 'fast, first-search stop, SearchRange %d, sub_shift_mode 1' % RANGE, 'imv': []}
    tz = eng.tz_par(RANGE, PW, PH, CTU, extended=0, fast=1, integer_et=0, first_search_stop=1, sub_shift_mode=1)
    for imv in (1, 2):
        s_ = 4 if imv == 1 else 6
        me = eng.me_par(LAM, 2, imv << 1)
        par = eng.amvr_par(LAM, V.DF_HAD, imv, (1, 1), PW, PH, CTU)
        bpar = eng.bi_par(LAM, 4, PW, PH, CTU, V.DF_HAD, ref_list=1, imv=imv)
        mb = np.array((1, 1), dtype=np.uint32)
        row = {'imv': imv, 'pus': 0, 'tz_ms': {}, 'refine_ms': {}, 'refine_over_tz': {}, 'bi_ms': {}, 'mismatches_uni': {}, 'mismatches_bi': {}}
        for s in SHAPES:
            rs = np.random.RandomState(4096 + 7 * s + imv)
            ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
            n = xs.size
            amvp = T.make_amvp(n, 2, 0, s_, rs)
            amvp['mvp_idx'] = rs.randint(0, 2, size=n)
            pus = T.tz_pus(s, s, n, rs, amvp, PW, PH)
            pus['x'] = xs.ravel(); pus['y'] = ys.ravel()
            pus['start_hor'] = rs.randint(-48 * 16, 48 * 16 + 1, size=n); pus['start_ver'] = rs.randint(-32 * 16, 32 * 16 + 1, size=n)
            bits = rs.randint(0, 40, size=n).astype(np.uint32)
            d_pus, d_amvp, d_bits = T._dev(pus), T._dev(amvp), T._dev(bits)
            d_mv = torch.zeros(n * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
            d_out = torch.zeros(n * V.AMVR_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
            torch.cuda.synchronize()

            def run_tz():
                assert eng.lib.vvb_tz_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), n, s, s, ctypes.byref(me), ctypes.byref(tz), None, 0, vp(d_mv.data_ptr())) == 0

            def run_refine():
                assert eng.lib.vvb_amvr_refine_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), vp(d_mv.data_ptr()), vp(d_amvp.data_ptr()), vp(d_bits.data_ptr()), n, s, s,
                                                   ctypes.byref(par), vp(d_out.data_ptr())) == 0
            row['tz_ms'][s] = round(timed(eng, stream, run_tz, a.reps), 3)
            row['refine_ms'][s] = round(timed(eng, stream, run_refine, a.reps), 3)
            row['refine_over_tz'][s] = round(row['refine_ms'][s] / row['tz_ms'][s], 3)
            eng.synchronize()
            mv, dev = T._host(d_mv, V.TZ_BEST_DT), T._host(d_out, V.AMVR_BEST_DT)
            row['mismatches_uni'][s] = sum(T.got(dev[i]) != T.restate(R, org, cur, S, 10, int(pus['x'][i]), int(pus['y'][i]), s, s,
                                                                       (int(mv['mv_hor'][i]), int(mv['mv_ver'][i])), amvp[i], int(bits[i]), V.DF_HAD, imv, (1, 1), LAM,
                                                                       1.0, PW, PH, 0, count=False) for i in range(n))
            # the bi branch, started from the uni result
            bi = np.zeros(n, dtype=V.BI_PU_DT)
            for f in ('x', 'y', 'pred_hor', 'pred_ver'):
                bi[f] = pus[f]
            bi['start_hor'] = mv['mv_hor'] * 16; bi['start_ver'] = mv['mv_ver'] * 16
            bi['bits'] = bits; bi['bcw_idx'] = np.arange(n) % 5
            pred = np.stack([oth[MARGIN + y:MARGIN + y + s, MARGIN + x:MARGIN + x + s] for x, y in zip(bi['x'], bi['y'])]).astype(np.int16)
            d_bi, d_pred = T._dev(bi), torch.from_numpy(pred).cuda()
            d_io = torch.zeros(n * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
            d_bo = torch.zeros(n * V.AMVR_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
            torch.cuda.synchronize()

            def run_bi():
                assert eng.lib.vvb_bipred_amvr_search_dev(eng.h, 0, 1, vp(d_bi.data_ptr()), vp(d_amvp.data_ptr()), n, s, s, ctypes.byref(bpar), mb.ctypes.data_as(vp),
                                                          None, 0, vp(d_pred.data_ptr()), vp(d_io.data_ptr()), vp(d_bo.data_ptr())) == 0
            row['bi_ms'][s] = round(timed(eng, stream, run_bi, a.reps), 3)
            eng.synchronize()
            io, bo = T._host(d_io, V.TZ_BEST_DT), T._host(d_bo, V.AMVR_BEST_DT)
            row['mismatches_bi'][s] = len(T.check_bi(R, eng, org, cur, S, 10, bi, amvp, np.zeros((0, 2), np.int32), pred, s, s, bpar, (1, 1), io, bo,
                                                     bcw_stats=False))
            row['pus'] += n
            print('imv %d: %dx%d done' % (imv, s, s), file=sys.stderr, flush=True)
        res['imv'].append(row)
    torch.cuda.synchronize()
    eng.close()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
