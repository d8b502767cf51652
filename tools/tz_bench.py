"""TZ integer motion search of a whole 3840x2160 10-bit picture: vvb_tz_search against the reference's own InterSearch::xTZSearch and the dense-table binding.

Every 8x8, 16x16, 32x32 and 64x64 PU of the picture, start vectors and predictors from a seeded field, fast settings (DIAMOND_FAST, first-search stop)
with SearchRange 128 and with SearchRange 384 (the medium preset).  Per setting:
  device_ms   vvb_tz_search, one call per shape, CUDA events around the calls of one picture after a warm-up picture
  member_ms   refshim_tz_search_member (oracle/_ref) over the same PUs, split over all usable host threads, wall clock
  table_ms    refshim_tz_search_rows_b200 (one dense vvb_sad_search launch per shape, then the member walking the tables on the host) on a sample of PUs per
              shape, scaled to the picture's PU count; SearchRange 128 only (TABLE_NOT_MEASURED)
Prints one JSON line with the card name and power limit read in the same run.  Needs oracle/_ref (built by build() where the reference sources exist)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from me_bench_common import PW, PH, card, pictures, timed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))

MARGIN, CTU, LAM = 144, 128, 57.0
# The dense-table binding cannot run SearchRange 384 here: the window of a 64x64 PU (the range clamped to the binding's reach, 145 x 145 positions) needs
# 233 920 bytes of shared memory in vvb_sad_search, above its 220 KB limit, so the call answers VVB_ERR_UNSUPPORTED; B200RowSearch::runTables turns that into a
# THROW, and composing that exception's message faults inside the reference probe library (vvenc::Exception::operator<< -> std::ostream::_M_insert<long>).
TABLE_NOT_MEASURED = {384: 'the 64x64 table window exceeds vvb_sad_search shared memory; the binding error path faults in the probe library (DESIGN §5)'}


def pu_lists():
    rs = np.random.RandomState(4096)
    out = {}
    for s in (8, 16, 32, 64):
        ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
        blk = np.zeros((xs.size, 6), dtype=np.int32)
        blk[:, 0] = xs.ravel(); blk[:, 1] = ys.ravel(); blk[:, 2] = s; blk[:, 3] = s
        blk[:, 4] = rs.randint(-48 * 16, 48 * 16 + 1, size=xs.size); blk[:, 5] = rs.randint(-32 * 16, 32 * 16 + 1, size=xs.size)
        out[s] = blk
    return out


def quarter(v):
    return np.where(v >= 0, (v + 1) >> 2, (v + 2) >> 2)


def table_leg(rng, sample):
    """refshim_tz_search_rows_b200 bound to the real library on `sample` PUs per shape, scaled to the picture; prints {"table_ms_scaled": ...}"""
    import vvenc_b200 as V
    from _libs import refshim, P, PO
    org, cur, S = pictures(MARGIN)
    R = refshim()
    R.refshim_tz_search_rows_b200.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double] + [ctypes.c_int] * 7 + [ctypes.c_void_p]
    R.refshim_b200_error.restype = ctypes.c_char_p
    assert R.refshim_install_b200_search(V.LIB_PATH.encode()) == 0, R.refshim_b200_error()
    base = MARGIN * S + MARGIN
    table_ms = 0.0
    for s, blk in pu_lists().items():
        sub = np.ascontiguousarray(blk[np.linspace(0, len(blk) - 1, min(sample, len(blk))).astype(int)])
        o = np.zeros((len(sub), 8), dtype=np.int64)
        t = time.perf_counter()
        # refReach is how far the binding may read around every block, the block included: the margin less the widest block and a guard
        rc = R.refshim_tz_search_rows_b200(1, PO(org, base), S, PO(cur, base), S, PW, PH, MARGIN - 72, P(sub), len(sub), 10, 1, LAM, rng, CTU, 0, 1, 0, 1, 0, P(o))
        table_ms += (time.perf_counter() - t) * 1e3 * len(blk) / len(sub)
        assert rc == 0, R.refshim_b200_error()
        print('table leg: %dx%d done' % (s, s), file=sys.stderr, flush=True)
    print(json.dumps({'table_ms_scaled': round(table_ms, 1)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--table-sample', type=int, default=128, help='PUs per shape timed on the dense-table path')
    ap.add_argument('--table-leg', type=int, default=0, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.table_leg:
        return table_leg(a.table_leg, a.table_sample)
    import torch
    import vvenc_b200 as V
    from _libs import refshim, P, PO
    name, plim = card()
    org, cur, S = pictures(MARGIN)
    lists = pu_lists()
    eng = V.CostEngine(0)
    eng.upload_plane(0, org, PW, PH, MARGIN, bit_depth=10); eng.upload_plane(1, cur, PW, PH, MARGIN, bit_depth=10)
    me = eng.me_par(LAM, 2, 0)
    R = refshim()
    tz_args = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
               ctypes.c_int, ctypes.c_int, ctypes.c_double] + [ctypes.c_int] * 7 + [ctypes.c_void_p]
    R.refshim_tz_search_member.argtypes = tz_args
    R.refshim_tz_search_seconds.restype = ctypes.c_double
    base = MARGIN * S + MARGIN
    threads = len(os.sched_getaffinity(0))
    res = {'metric': 'tz_search_picture', 'picture': '%dx%d 10-bit' % (PW, PH), 'pus': int(sum(len(b) for b in lists.values())), 'card': name, 'power_limit': plim,
           'host_threads': threads, 'settings': []}
    for rng in (128, 384):
        flags = (0, 1, 0, 1)                  # xTZSearch( ..., bExtendedSettings = false, bFastSettings = true ), first-search stop
        tz = eng.tz_par(rng, PW, PH, CTU, extended=0, fast=1, integer_et=0, first_search_stop=1, sub_shift_mode=1)
        d_pus, d_out = {}, {}
        for s, blk in lists.items():
            p = np.zeros(len(blk), dtype=V.TZ_PU_DT)
            p['x'] = blk[:, 0]; p['y'] = blk[:, 1]; p['start_hor'] = blk[:, 4]; p['start_ver'] = blk[:, 5]
            p['pred_hor'] = quarter(blk[:, 4]); p['pred_ver'] = quarter(blk[:, 5])
            d_pus[s] = torch.from_numpy(p.view(np.uint8).copy()).cuda()
            d_out[s] = torch.zeros(len(blk) * 32, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        stream = torch.cuda.ExternalStream(eng.stream)

        def picture():
            for s, blk in lists.items():
                rc = eng.lib.vvb_tz_search_dev(eng.h, 0, 1, d_pus[s].data_ptr(), len(blk), s, s, ctypes.byref(me), ctypes.byref(tz), None, 0, d_out[s].data_ptr())
                assert rc == 0, eng.lib.vvb_last_error(eng.h)
        dev_ms = timed(eng, stream, picture, a.reps)
        print('device: range %d %.3f ms' % (rng, dev_ms), file=sys.stderr, flush=True)
        # the member on all host threads; its results check the device's
        member_ms = 0.0; mismatched = 0
        for s, blk in lists.items():
            out = np.zeros((len(blk), 8), dtype=np.int64)
            chunks = np.array_split(np.arange(len(blk)), threads)

            def run(idx, blk=blk, out=out):
                if len(idx) == 0:
                    return 0
                sub = np.ascontiguousarray(blk[idx[0]:idx[-1] + 1]); o = np.zeros((len(sub), 8), dtype=np.int64)
                rc = R.refshim_tz_search_member(1, PO(org, base), S, PO(cur, base), S, PW, PH, MARGIN, P(sub), len(sub), 10, 1, LAM, rng, CTU, *flags, 0, P(o))
                out[idx[0]:idx[-1] + 1] = o
                return rc
            t = time.perf_counter()
            with ThreadPoolExecutor(threads) as ex:
                assert not any(ex.map(run, chunks))
            member_ms += (time.perf_counter() - t) * 1e3
            got = np.frombuffer(d_out[s].cpu().numpy().tobytes(), dtype=V.TZ_BEST_DT)
            same = (got['mv_hor'] == out[:, 0]) & (got['mv_ver'] == out[:, 1]) & (got['sad'].astype(np.int64) == out[:, 2]) & \
                   (got['cost'].astype(np.int64) == out[:, 4]) & (got['best_distance'].astype(np.int64) == out[:, 5])
            mismatched += int((~same).sum())
            print('member: %dx%d done' % (s, s), file=sys.stderr, flush=True)
        member_walk_s = R.refshim_tz_search_seconds()       # time inside xTZSearch summed over the threads, as the probe counts it
        # the dense-table path in a process of its own: the reference probe binds one C-ABI library per process
        if rng in TABLE_NOT_MEASURED:
            table = {'table_ms_scaled': 'not measured', 'table_reason': TABLE_NOT_MEASURED[rng]}
        else:
            leg = subprocess.run([sys.executable, os.path.abspath(__file__), '--table-leg', str(rng), '--table-sample', str(a.table_sample)], capture_output=True, text=True)
            table = json.loads(leg.stdout.strip().splitlines()[-1]) if leg.returncode == 0 else {'table_ms_scaled': None, 'table_error': leg.stderr[-400:]}
        res['settings'].append({'search_range': rng, 'fast': 1, 'device_ms': round(dev_ms, 3), 'member_ms': round(member_ms, 1), 'member_walk_cpu_s': round(member_walk_s, 2), 'device_vs_member_mismatches': mismatched, 'table_sample_per_shape': a.table_sample, **table})
    eng.close()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
