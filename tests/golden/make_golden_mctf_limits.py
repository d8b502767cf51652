#!/usr/bin/env python3
"""Regenerates tests/golden/golden_v7_mctf_limits.npz from the UNMODIFIED reference (oracle/_ref): the unit-32 motion field of MCTF::motionEstimationMCTF on the
in-range pyramid picture of tests/test_gpu_mctf_limits.py, and the apply-stage pictures (xFinalizeBlkLine per block) of its APPLY_CASES.  Run where
oracle/_ref is built:  python tests/golden/make_golden_mctf_limits.py
Every result comes from the scalar kernels and is cross-checked against the AVX2 ones wherever those are defined: the AVX2 apply kernels work on 4-pel
column groups and write past a block of width 2 or 6, so the trailing-unit pictures of those widths come from the scalar build alone."""
import os, sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import impls
import test_gpu_mctf_limits as T
from _libs import refshim, P


def main():
    R = refshim()
    out = {}
    org, ref = T.pyramid_case('smooth')
    H, W = org.shape
    res = []
    for opt, simd in ((0, b'SCALAR'), (1, b'AVX2')):
        R.refshim_set_simd(simd)
        f = np.zeros(((H + 31) // 32, (W + 31) // 32, 4), dtype=np.int32)
        R.refshim_mctf_estimate_pyramid(opt, P(org), P(ref), W, H, 10, 32, 0, 0, 0, P(f))
        res.append(f)
    assert np.array_equal(res[0], res[1]), 'scalar != AVX2 (pyramid)'
    out['pyramid_smooth'] = res[1]
    for k in range(len(T.APPLY_CASES)):
        case, tap4, planar = T.apply_case(k)
        res = []
        for opt, simd in ((0, b'SCALAR'), (1, b'AVX2'))[:2 if case['W'] % 4 == 0 else 1]:
            R.refshim_set_simd(simd)
            res.append(impls.mctf_apply_expected(R, 'refshim', case, tap4, planar, opt))
        assert all(np.array_equal(res[0], r) for r in res), ('scalar != AVX2', T.APPLY_CASES[k][0])
        out['apply_%d' % k] = res[0]
    path = os.path.join(HERE, 'golden_v7_mctf_limits.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, {k: v.shape for k, v in out.items()}, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
