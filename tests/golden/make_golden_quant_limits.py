#!/usr/bin/env python3
"""Regenerates tests/golden/golden_v9_quant_limits.npz from the UNMODIFIED reference (oracle/_ref): the rate-distortion quantisers at the ends of their QP, lambda
and value range (the rows of test_gpu_quant_limits.rq_cases / ts_cases / rt_cases):
  rq_*  QuantRDOQ2::xRateDistOptQuant -- levels, (absSum, lastPos), the fractional bits it read (190), the per-call constants (7);
  dq_*  DepQuant::xQuantDQ -- levels of the scalar members (dq_q0_i) and of the x86 ones (dq_q1_i), meta = (absSum, lastPos) of each, rates (266), constants (9);
  ts_* / bd_*  QuantRDOQ::rateDistOptQuantTS and forwardRDPCM -- levels, absSum, the transform-skip rates (44);
  rt_*  the TU candidate round trip of tu_rdo_cases.ref_roundtrip_rdo (the first TU of tu_rdo_cases.inputs( row, 4 )): levels, reco - pred, the five results and
        need_rdoq, the rates the quantiser read.
The scalar and the AVX2 builds of RDOQ, transform skip, BDPCM and the round trip are required to agree at generation time.  Inputs are not stored: they are
regenerated from each row's seed (rq_crc, dq_crc, ts_crc hold their CRC-32, checked by the tests).
Run in the build container only:  python tests/golden/make_golden_quant_limits.py  (--check: compare with the file instead of writing it)"""
import os, sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import test_gpu_quant_limits as Q
import tu_rdo_cases as T


def main(check=False):
    out = {}
    rows = Q.rq_cases()
    out['rq_cases'] = rows; out['rq_crc'] = np.array([Q.crc(Q.rq_inputs(r)) for r in rows], np.uint32)
    meta = np.zeros((len(rows), 2), np.int64); rates = np.zeros((len(rows), 190), np.int32); consts = np.zeros((len(rows), 7), np.int32)
    for i, row in enumerate(rows):
        a, b = Q.ref_rdoq(row, 0), Q.ref_rdoq(row, 1)
        assert np.array_equal(a[0], b[0]) and a[1:3] == b[1:3] and np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4]), i
        out['rq_q_%d' % i] = b[0]; meta[i] = b[1:3]; rates[i] = b[3]; consts[i] = b[4]
    out['rq_meta'] = meta; out['rq_rates'] = rates; out['rq_consts'] = consts

    rows = Q.rq_cases(dq=True)
    out['dq_cases'] = rows; out['dq_crc'] = np.array([Q.crc(Q.rq_inputs(r)) for r in rows], np.uint32)
    meta = np.zeros((len(rows), 4), np.int64); rates = np.zeros((len(rows), 266), np.int32); consts = np.zeros((len(rows), 9), np.int64)
    for i, row in enumerate(rows):
        for opt in (0, 1):
            q, s, l, r, k = Q.ref_dep_quant(row, opt)
            out['dq_q%d_%d' % (opt, i)] = q; meta[i, 2 * opt:2 * opt + 2] = (s, l)
            assert opt == 0 or (np.array_equal(rates[i], r) and np.array_equal(consts[i], k)), i
            rates[i] = r; consts[i] = k
    out['dq_meta'] = meta; out['dq_rates'] = rates; out['dq_consts'] = consts

    rows = Q.ts_cases()
    out['ts_cases'] = rows; out['ts_crc'] = np.array([Q.crc(Q.ts_inputs(r)) for r in rows], np.uint32)
    rates = np.zeros((len(rows), 44), np.int32); ts_sum = np.zeros(len(rows), np.int64); bd_sum = np.zeros(len(rows), np.int64)
    for i, row in enumerate(rows):
        a, b = Q.ref_ts(row, 0, False), Q.ref_ts(row, 1, False)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2]), i
        out['ts_q_%d' % i] = b[0]; ts_sum[i] = b[1]; rates[i] = b[2]
        a, b = Q.ref_ts(row, 0, True), Q.ref_ts(row, 1, True)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], i
        out['bd_q_%d' % i] = b[0]; bd_sum[i] = b[1]
    out['ts_rates'] = rates; out['ts_abs_sum'] = ts_sum; out['bd_abs_sum'] = bd_sum

    rows = Q.rt_cases()
    out['rt_cases'] = rows
    meta = np.zeros((len(rows), 6), np.int64)
    for i, row in enumerate(rows):
        org, pred = T.inputs(row, 4)
        res = [T.ref_roundtrip_rdo(row, org[0], pred[0], simd) for simd in (b'SCALAR', b'AVX2')]
        (q0, r0, m0, n0, rt0, _), (q, reco, m, need, r, _) = res
        assert np.array_equal(q0, q) and np.array_equal(r0, reco) and m0 == m and n0 == need and np.array_equal(rt0, r), i
        meta[i] = m + [need]
        out['rt_q_%d' % i] = q; out['rt_dreco_%d' % i] = (reco - pred[0]).astype(np.int16); out['rt_rates_%d' % i] = r
    out['rt_meta'] = meta

    path = os.path.join(HERE, 'golden_v9_quant_limits.npz')
    if check:
        g = np.load(path)
        bad = sorted(k for k in set(out) | set(g.files) if k not in out or k not in g.files or not np.array_equal(out[k], g[k]))
        print('CHECK', 'OK' if not bad else 'MISMATCH %s' % bad[:20])
        return not bad
    np.savez_compressed(path, **out)
    print('wrote', path, {k: len(out[k + '_cases']) for k in ('rq', 'dq', 'ts', 'rt')}, os.path.getsize(path), 'bytes')
    return True


if __name__ == '__main__':
    sys.exit(0 if main(check='--check' in sys.argv[1:]) else 1)
