"""Body of tests/test_shared_text_sanitizers.py, run in a process of its own with libasan / libubsan preloaded: the host / device shared texts (both RDOQ engines, the
transform-skip and BDPCM quantisers, the DepQuant trellis) compiled with -fsanitize=address,undefined, on the golden inputs and on random batches with extreme coefficients,
QPs and lambdas.  An out-of-bounds read that the CPU tolerates silently would be a fault (or garbage) on the device.  usage: _sanitizer_run.py <lib.so> rdoq|dq"""
import sys, ctypes, numpy as np
import os
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases as C
L = ctypes.CDLL(sys.argv[1])
WHAT = sys.argv[2]
I = ctypes.c_int; D = ctypes.c_double; V = ctypes.c_void_p
def P(a): return a.ctypes.data_as(V)
L.orc_rdoq.argtypes = [I]*8 + [D, I, V, V, I, V, V, V]; L.orc_rdoq_v2.argtypes = L.orc_rdoq.argtypes
L.orc_rdoq_ts.argtypes = [I]*5 + [D, V, V, I, V, V]
L.orc_rdoq_bdpcm.argtypes = [I]*6 + [D, V, V, I, V, V]
L.orc_dep_quant.argtypes = [I]*4 + [D] + [I]*4 + [V, V, I, V, V, V]
g = np.load(os.path.join(HERE, 'golden', 'golden_v6_rdoq.npz')); g5 = np.load(os.path.join(HERE, 'golden', 'golden_v5_depquant.npz'))
n = 0
for i, row in enumerate(C.rdoq_cases() if WHAT == 'rdoq' else []):
    w, h, bd, qp, lam1000, scale, decay10, comp, lf, sbt, intra, sh, cb, thr, init_id, seed = [int(v) for v in row]
    coef = C.rdoq_inputs(row); rates = np.ascontiguousarray(g['rates'][i])
    for f in (L.orc_rdoq, L.orc_rdoq_v2):
        q = np.zeros((h, w), np.int16); s = ctypes.c_int32(); l = ctypes.c_int32()
        assert f(w, h, bd, qp, int(comp > 0), lf, sbt, sh, lam1000 / 1000.0, thr, P(rates), P(coef), 1, P(q), ctypes.byref(s), ctypes.byref(l)) == 0
        assert np.array_equal(q, g['q_%d' % i]); n += 1
for i, row in enumerate(C.rdoq_ts_cases() if WHAT == 'rdoq' else []):
    w, h, bd, qp, lam1000, amp, kind, comp, intra, delta, init_id, seed = [int(v) for v in row]
    coef = C.rdoq_ts_inputs(row); rates = np.ascontiguousarray(g['ts_rates'][i])
    q = np.zeros((h, w), np.int16); s = ctypes.c_int32()
    assert L.orc_rdoq_ts(w, h, bd, qp, delta, lam1000 / 1000.0, P(rates), P(coef), 1, P(q), ctypes.byref(s)) == 0 and np.array_equal(q, g['tsq_%d' % i])
    assert L.orc_rdoq_bdpcm(w, h, bd, qp, delta, 1 + (seed & 1), lam1000 / 1000.0, P(rates), P(coef), 1, P(q), ctypes.byref(s)) == 0 and np.array_equal(q, g['bdq_%d' % i]); n += 2
for i, row in enumerate(C.dq_cases() if WHAT == 'dq' else []):
    w, h, bd, qp, lam1000, scale, decay10, mts, lf, sbt, intra, init_id, seed = [int(v) for v in row]
    coef = C.dq_inputs(row); rates = np.ascontiguousarray(g5['rates'][i])
    q = np.zeros((h, w), np.int16); s = ctypes.c_int32(); l = ctypes.c_int32()
    assert L.orc_dep_quant(w, h, bd, qp, lam1000 / 1000.0, 8, C.dq_zero_out(row), lf, 0, P(rates), P(coef), 1, P(q), ctypes.byref(s), ctypes.byref(l)) == 0; n += 1
# random batches incl. extreme coefficients
rs = np.random.RandomState(5)
for (w, h) in ([(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (4, 32), (64, 4), (16, 64), (32, 8)] if WHAT == 'rdoq' else []):
    for amp in (3, 300, 32767):
        cnt = 60
        coef = rs.randint(-amp, amp + 1, size=(cnt, h, w)).astype(np.int32); coef[:, :, 32:] = 0; coef[:, 32:, :] = 0
        for sh in (0, 1):
            for lf in (0, 1):
                rates = np.ascontiguousarray(g['rates'][int(rs.randint(len(g['rates'])))])
                for f in (L.orc_rdoq, L.orc_rdoq_v2):
                    q = np.zeros((cnt, h, w), np.int16); s = np.zeros(cnt, np.int32); l = np.zeros(cnt, np.int32)
                    assert f(w, h, 10, int(rs.choice([0, 17, 32, 51, 63])), int(rs.randint(2)), lf, 0, sh, float(rs.choice([0.5, 57.3, 20000.0])), 8, P(rates), P(coef), cnt, P(q), P(s), P(l)) == 0; n += cnt
        if w <= 32 and h <= 32:
            tr = np.ascontiguousarray(g['ts_rates'][int(rs.randint(len(g['ts_rates'])))])
            q = np.zeros((cnt, h, w), np.int16); s = np.zeros(cnt, np.int32)
            assert L.orc_rdoq_ts(w, h, 10, int(rs.choice([0, 17, 32, 51, 63])), 0, 57.3, P(tr), P(coef), cnt, P(q), P(s)) == 0
            assert L.orc_rdoq_bdpcm(w, h, 10, int(rs.choice([0, 17, 32, 51, 63])), 0, 1 + int(rs.randint(2)), 57.3, P(tr), P(coef), cnt, P(q), P(s)) == 0; n += 2 * cnt
# DepQuant at the ends of the QP range, below the floor -6 * (bd - 8) and above 63 included (the clip of the internal QP keeps the scale index in range), both
# member flavours, the lambdas the encoder derives there (only where the reference's uint32_t conversion is defined)
from test_gpu_quant_limits import qp_ends, lambdas, dq_defined
for (w, h) in ([(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (8, 4), (4, 32), (64, 16)] if WHAT == 'dq' else []):
    for bd in (8, 10):
        for qp in qp_ends(bd):
            for lam in lambdas(qp, bd):
                if not dq_defined(w, h, bd, qp, lam): continue
                cnt = 4
                coef = rs.choice([-32768, -3000, -1, 0, 0, 1, 400, 32767], size=(cnt, h, w)).astype(np.int32); coef[:, :, 32:] = 0; coef[:, 32:, :] = 0
                rates = np.ascontiguousarray(g5['rates'][int(rs.randint(len(g5['rates'])))])
                for scalar in (0, 1):
                    q = np.zeros((cnt, h, w), np.int16); s = np.zeros(cnt, np.int32); l = np.zeros(cnt, np.int32)
                    assert L.orc_dep_quant(w, h, bd, qp, lam, 8, 0, 0, scalar, P(rates), P(coef), cnt, P(q), P(s), P(l)) == 0; n += cnt
print('SANITIZER CLEAN', n)
