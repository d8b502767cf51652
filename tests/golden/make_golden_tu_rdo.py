#!/usr/bin/env python3
"""Regenerates tests/golden/golden_v8_tu_rdo.npz from the UNMODIFIED reference (oracle/_ref): for every row of tu_rdo_cases.cases() the TU candidate body of
xIntraCodingTUBlock / xEstimateInterResidualQT with the slice's quantiser -- the forward transform (+ LFNST) and xNeedRDOQ, QuantRDOQ2::xRateDistOptQuantFast or
DepQuant::xQuantDQ with the rates the reference read from its CABAC contexts, the matching dequantiser and invTransformNxN when uiAbsSum > 0, reconstruct, SSE.
The scalar and the AVX2 build of the members are required to agree at generation time.  org / pred are not stored: tu_rdo_cases.inputs() regenerates them
from each row's seed (inputs_crc holds their CRC-32, checked by the tests), and the reconstruction is stored as reco - pred (dreco_i).
Run in the build container only:  python tests/golden/make_golden_tu_rdo.py"""
import os, sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import tu_rdo_cases as T


def main():
    rows = T.cases()
    out = {'cases': rows}
    meta = np.zeros((len(rows), 6), dtype=np.int64)                  # dist_reco, dist_resi, dist_zero, abs_sum, last_pos, need_rdoq
    lfnst = np.zeros((len(rows), 2), dtype=np.int32)                 # the LFNST set and transpose flag the reference derived from the intra mode
    crc = np.zeros(len(rows), dtype=np.uint32)                       # CRC-32 of the regenerated org / pred
    for i, row in enumerate(rows):
        org, pred = T.inputs(row)
        res = [T.ref_roundtrip_rdo(row, org[0], pred[0], simd) for simd in (b'SCALAR', b'AVX2')]
        (q0, r0, m0, n0, rt0, st0), (q, reco, m, need, rates, st) = res
        assert np.array_equal(q0, q) and np.array_equal(r0, reco) and m0 == m and n0 == need and np.array_equal(rt0, rates) and st0 == st, i
        meta[i] = m + [need]; lfnst[i] = st; crc[i] = T.inputs_crc(org[0], pred[0])
        out['rates_%d' % i] = rates; out['q_%d' % i] = q; out['dreco_%d' % i] = (reco - pred[0]).astype(np.int16)
    out['meta'] = meta; out['lfnst'] = lfnst; out['inputs_crc'] = crc
    path = os.path.join(HERE, 'golden_v8_tu_rdo.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, len(rows), 'cases,', int((meta[:, 3] > 0).sum()), 'with an inverse,', int(meta[:, 5].sum()), 'with need_rdoq,', os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
