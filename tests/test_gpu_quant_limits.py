"""The rate-distortion quantisers -- vvb_rdoq (engines 1 and 2), vvb_rdoq_ts, vvb_rdoq_bdpcm, vvb_dep_quant (engines 0 and 1) and the one-call TU candidate
vvb_tu_roundtrip_rdo that chains them -- at the ends of their QP, lambda and TU-count range:
  * QP -o-2, -o-1, -o, 0, 63 and 64 with o = 6 * (bd - 8), at 8 and 10 bits, so that the clip of the base QP (QpParam, Quant.cpp:109) is crossed on both sides;
    for transform skip and BDPCM also the floor 4 + 6 * internalMinusInputBitDepth crossed from both sides with delta 0 and 2.  CABAC contexts initialised at
    slice QP 0, 32 and 63;
  * the lambda the encoder derives at each QP (EncSlice::xCalculateLambda: 0.57 * 2^((qp + o - 12) / 3)), and that lambda times and divided by 256;
  * coefficients at +32767 / -32768 (flat and sparse), the forward's worst-case outputs, dense large levels (sign hiding in groups of large levels, the budget of
    context-coded bins exhausted so that the Golomb-Rice branch runs with long escape codes), fast RDOQ levels beyond int16 (stored as the member stores them
    into TCoeffSig, QuantRDOQ2.cpp:942), DepQuant's maxQIdx, transform-skip levels at 32767, BDPCM reconstruction chains at +-pelMax;
  * TU counts 0, 1, 63, 64, 65 and above the resident grid, need_rdoq all 0 / all 1 / null, the nullable outputs null, a large BDPCM call after a small one.
The member outputs for the limit cases are in tests/golden/golden_v9_quant_limits.npz (tests/golden/make_golden_quant_limits.py); the inputs are regenerated from
each row's seed and checked by CRC-32.  The CPU tests pin the oracle (the shared text compiled for the CPU) to that file everywhere and to the reference members
where oracle/_ref is built (scalar and AVX2 builds); the GPU tests compare the device with the file and with the oracle bit for bit.

Excluded on purpose: DepQuant rows where the reference itself is undefined -- Quantizer::initQuantBlock converts nomDistFactor * qScale2 = 2^nomDShift / lambda to
uint32_t (DepQuant.cpp:566); dq_defined() keeps only rows where that product stays below 2^31."""
import ctypes
import os
import zlib
import numpy as np
import pytest
from _libs import dq_oracle, have_ref, refshim, P

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'golden_v9_quant_limits.npz')
needs_ref = pytest.mark.skipif(not have_ref(), reason="oracle/_ref (the reference probe) is not built here")
I32 = ctypes.c_int32
LAM_FACTOR = 256.0
CTX_QPS = (0, 32, 63)
RQ_SHAPES = [(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (8, 4), (4, 32), (64, 16), (16, 64)]
TS_SHAPES = [(4, 4), (8, 8), (16, 16), (32, 32), (8, 4), (4, 32), (32, 8), (16, 4)]
RQ_PATTERNS = 6          # flat +32767, flat -32768, sparse extremes, forward worst case, dense laplacian (large), dense uniform (moderate)
TS_PATTERNS = 6          # flat +32767, flat -32768, sparse extremes, +-pelMax checkerboard, random +-pelMax, dense scaled residual


def qp_ends(bd):
    o = 6 * (bd - 8)
    return (-o - 2, -o - 1, -o, 0, 63, 64)


def ts_floor_qps(bd, delta):
    """CU QPs whose internal QP is one below, at and one above the transform-skip floor 4 + 6 * delta"""
    f = 4 + 6 * delta - 6 * (bd - 8)
    return (f - 1, f, f + 1)


def enc_lambda(qp, bd):
    """EncSlice::xCalculateLambda for an intra slice at this QP (the encoder clips the QP to -o..63 first)"""
    o = 6 * (bd - 8)
    qc = max(-o, min(63, qp))
    return 0.57 * 2.0 ** ((qc + o - 12) / 3.0)


def lambdas(qp, bd):
    lam = enc_lambda(qp, bd)
    return (lam / LAM_FACTOR, lam, lam * LAM_FACTOR)


def internal_qp(qp, bd):
    o = 6 * (bd - 8)
    return max(0, min(63 + o, qp + o))


def dq_defined(w, h, bd, qp, lam):
    """the reference's (uint32_t)( nomDistFactor * qScale2 ) (DepQuant.cpp:566) is defined: 2^nomDShift / lambda stays below 2^31 (margin for rounding)"""
    lw, lh = w.bit_length() - 1, h.bit_length() - 1
    q = internal_qp(qp, bd) + 1
    nom = 15 - bd - ((lw + lh) >> 1)
    sqrt2 = (lw + lh) & 1
    qshift = 13 + q // 6 + nom - sqrt2
    nom_dshift = 15 - 2 * nom + qshift + sqrt2
    return 2.0 ** nom_dshift / lam < 2.0 ** 31


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a, dtype=np.int32).tobytes())


# ---------------------------------------------------------------------------------------------------- cases
# fast RDOQ / DepQuant row: w, h, bd, qp, lam_idx, pattern, comp, sign_hiding, ctx_qp, init_id, seed (lambda = lambdas(qp, bd)[lam_idx])
RQ_COLS = ('w', 'h', 'bd', 'qp', 'lam_idx', 'pattern', 'comp', 'sh', 'ctx_qp', 'init_id', 'seed')
# transform-skip / BDPCM row: w, h, bd, qp, delta, lam_idx, pattern, comp, dir_mode, ctx_qp, init_id, seed
TS_COLS = ('w', 'h', 'bd', 'qp', 'delta', 'lam_idx', 'pattern', 'comp', 'dir_mode', 'ctx_qp', 'init_id', 'seed')


def rd(row, cols):
    return dict(zip(cols, [int(v) for v in row]))


# fast-RDOQ rows beyond the grid, seeds picked by searching the seed space: pattern 6 rows, where a Rice parameter reads a level from 32768 to 65535 (templateAbsSum
# counts abs() of its negative TCoeffSig) and the decision it prices flips with it; pattern 7 rows, where the Rice update of a level >= 4 runs with exactly four
# context-coded bins left (remRegBins >= 4, QuantRDOQ2.cpp:777), in each engine
RQ_EXTRA = [[32, 32, 10, -12, 2, 6, 0, 0, 0, 2, 20029], [32, 32, 10, -14, 2, 6, 1, 1, 32, 1, 20058], [32, 32, 10, -13, 2, 6, 1, 0, 0, 0, 20096],
            [32, 32, 10, -13, 2, 6, 1, 1, 63, 0, 20140], [64, 64, 10, -14, 2, 6, 1, 1, 32, 2, 20165], [32, 32, 10, -13, 2, 6, 0, 1, 32, 2, 20213],
            [4, 4, 10, -14, 2, 7, 0, 1, 63, 0, 20808], [4, 32, 8, -1, 1, 7, 0, 0, 63, 0, 20989], [16, 64, 8, 0, 1, 7, 1, 1, 63, 2, 21546],
            [64, 64, 10, -13, 2, 7, 1, 0, 32, 2, 22830], [16, 64, 8, 0, 2, 7, 1, 1, 0, 2, 23762], [16, 64, 10, -12, 2, 7, 0, 1, 63, 1, 24857]]


def rq_cases(dq=False):
    """every (bit depth, end QP, lambda, pattern); the 64 x 64 shape for the forward's worst case at the encoder's lambda, the other shapes cycled; DepQuant rows
    (dq=True, luma only, no sign hiding) where the reference is undefined are left out"""
    rows = []
    k = 0
    for bd in (8, 10):
        for qi, qp in enumerate(qp_ends(bd)):
            for li in range(3):
                for pat in range(RQ_PATTERNS):
                    w, h = (64, 64) if (pat == 3 and li == 1) else RQ_SHAPES[k % len(RQ_SHAPES)]
                    k += 1
                    if dq and not dq_defined(w, h, bd, qp, lambdas(qp, bd)[li]):
                        continue
                    comp = 0 if dq else k % 2
                    sh = 0 if dq else (k // 2) % 2
                    rows.append([w, h, bd, qp, li, pat, comp, sh, CTX_QPS[k % 3], k % 3, (7100 if dq else 6100) + k])
    return np.array(rows + ([] if dq else RQ_EXTRA), dtype=np.int64)


def ts_cases():
    """every (bit depth, end QP or transform-skip floor QP with delta 0 / 2, lambda, pattern), shapes up to 32 cycled"""
    rows = []
    k = 0
    for bd in (8, 10):
        qps = [(qp, 0) for qp in qp_ends(bd)] + [(qp, 0) for qp in ts_floor_qps(bd, 0)] + ([(qp, 2) for qp in ts_floor_qps(bd, 2)] if bd == 10 else [])
        for qp, delta in qps:
            for li in range(3):
                for pat in range(TS_PATTERNS):
                    w, h = TS_SHAPES[k % len(TS_SHAPES)]
                    k += 1
                    rows.append([w, h, bd, qp, delta, li, pat, k % 2, 1 + (k // 2) % 2, CTX_QPS[k % 3], k % 3, 8100 + k])
    return np.array(rows, dtype=np.int64)


def _zero_out(c, w, h):
    c[:, 32:] = 0
    c[32:, :] = 0
    return c


def rq_inputs(row):
    """the transform coefficients [h][w] (int32) of a fast-RDOQ / DepQuant row: only the 32 x 32 region the quantisers scan is non-zero"""
    c = rd(row, RQ_COLS)
    w, h, pat = c['w'], c['h'], c['pattern']
    rs = np.random.RandomState(c['seed'])
    if pat == 0:
        x = np.full((h, w), 32767)
    elif pat == 1:
        x = np.full((h, w), -32768)
    elif pat == 2:
        x = np.where(rs.rand(h, w) < 0.5, 32767, -32768) * (rs.rand(h, w) < 0.15)
    elif pat == 3:
        from test_gpu_tu_limits import worst_residuals, fwd_oracle
        resi = worst_residuals(w, h, 0, 0, c['bd'], c['seed'])
        x = fwd_oracle(w, h, 0, 0, c['bd'], 0, 0, 0, resi[c['seed'] % len(resi)][None])['coef'][0]
    elif pat == 4:
        x = rs.laplace(0, 4000.0, size=(h, w)) + np.sign(rs.rand(h, w) - 0.5) * 3000
    elif pat == 5:
        x = rs.randint(-400, 401, size=(h, w))
    elif pat == 6:                       # moderate coefficients whose right / lower neighbours are near full scale: their Rice parameter reads levels above 32767
        x = np.zeros((h, w), np.int64)
        for _ in range(rs.randint(4, 16)):
            py, px = rs.randint(min(h, 32) - 1), rs.randint(min(w, 32) - 1)
            x[py, px] = rs.randint(3, 401) * rs.choice([-1, 1])
            x[py, px + 1] = rs.randint(21000, 32768) * rs.choice([-1, 1]); x[py + 1, px] = rs.randint(21000, 32768) * rs.choice([-1, 1])
    else:                                # dense moderate levels of a seed-chosen spread: the bin budget runs out at varying positions
        x = rs.randint(-1, 2, size=(h, w)) * rs.randint(0, 10 ** rs.uniform(1, 3.5), size=(h, w))
    return _zero_out(np.clip(x, -32768, 32767).astype(np.int32), w, h)


def ts_inputs(row):
    """the coefficients [h][w] (int32) of a transform-skip / BDPCM row: xTransformSkip copies the residual unscaled; patterns 0-2 drive the level to the int16
    ends, 3-4 the residual (and the BDPCM reconstruction chain) to +-pelMax, 5 large dense levels for the bin budget"""
    c = rd(row, TS_COLS)
    w, h, pat, m = c['w'], c['h'], c['pattern'], (1 << c['bd']) - 1
    rs = np.random.RandomState(c['seed'])
    yy, xx = np.mgrid[0:h, 0:w]
    if pat == 0:
        x = np.full((h, w), 32767)
    elif pat == 1:
        x = np.full((h, w), -32768)
    elif pat == 2:
        x = np.where(rs.rand(h, w) < 0.5, 32767, -32768) * (rs.rand(h, w) < 0.15)
    elif pat == 3:
        x = np.where((yy + xx) & 1, -m, m)
    elif pat == 4:
        x = np.where(rs.rand(h, w) < 0.5, -m, m)
    else:
        x = rs.randint(-m, m + 1, size=(h, w)) << 5
    return np.clip(x, -32768, 32767).astype(np.int32)


# ---------------------------------------------------------------------------------------------------- the members and the oracle on one row
LAST_GROUPS = {4: 4, 8: 6, 16: 8, 32: 10, 64: 10}        # g_uiGroupIdx[ min( n, 32 ) - 1 ] + 1: last-position groups of a side


def used_rates(rates, w, h):
    """the rate tables with the last-position entries a TU of this shape never reads set to 0.  The probe copies whole tables out of the member objects,
    and entries beyond the TU's own last-position range keep whatever an earlier TU of another shape left there."""
    r = np.array(rates, copy=True)
    if len(r) == 266:                                      # vvb_dq_rates: last_bits_x[32], last_bits_y[32] by position
        r[min(w, 32):32] = 0; r[32 + min(h, 32):64] = 0
    else:                                                  # vvb_rdoq_rates: last_bits_x[16], last_bits_y[16] by group, from entry 154
        r[154 + LAST_GROUPS[w]:170] = 0; r[170 + LAST_GROUPS[h]:186] = 0
    return r


def ref_rdoq(row, opt):
    """QuantRDOQ2::xRateDistOptQuant on the probe's rig -> q, abs_sum, last_pos, rates (190), constants (7)"""
    R = refshim(); R.refshim_set_simd(b'AVX2' if opt else b'SCALAR')
    c = rd(row, RQ_COLS); w, h = c['w'], c['h']
    lam = lambdas(c['qp'], c['bd'])[c['lam_idx']]
    q = np.zeros((h, w), np.int16); s = I32(); l = I32(); rates = np.zeros(190, np.int32); k = np.zeros(7, np.int32)
    assert R.refshim_rdoq(c['comp'], P(rq_inputs(row)), w, h, c['bd'], c['qp'], 1, 0, 0, c['sh'], 0, lam, 8, c['ctx_qp'], c['init_id'], P(q), ctypes.byref(s),
                          ctypes.byref(l), P(rates), P(k)) == 0
    R.refshim_set_simd(b'AVX2')
    return q, s.value, l.value, used_rates(rates, w, h), k


def ref_dep_quant(row, opt):
    """DepQuant::xQuantDQ on the probe's rig (opt 0 scalar members, 1 the x86 ones) -> q, abs_sum, last_pos, rates (266), constants (9)"""
    R = refshim()
    c = rd(row, RQ_COLS); w, h = c['w'], c['h']
    lam = lambdas(c['qp'], c['bd'])[c['lam_idx']]
    q = np.zeros((h, w), np.int16); s = I32(); l = I32(); rates = np.zeros(266, np.int32); k = np.zeros(9, np.int64)
    assert R.refshim_dep_quant(P(rq_inputs(row)), w, h, c['bd'], c['qp'], 0, 1, 0, 0, lam, 8, opt, c['ctx_qp'], c['init_id'], P(q), ctypes.byref(s), ctypes.byref(l),
                               P(rates), P(k)) == 0
    return q, s.value, l.value, used_rates(rates, w, h), k


def ref_ts(row, opt, bdpcm):
    """QuantRDOQ::rateDistOptQuantTS or forwardRDPCM on the probe's rig -> q, abs_sum, rates (44), constants (3) of rateDistOptQuantTS"""
    R = refshim(); R.refshim_set_simd(b'AVX2' if opt else b'SCALAR')
    c = rd(row, TS_COLS); w, h = c['w'], c['h']
    lam = lambdas(c['qp'], c['bd'])[c['lam_idx']]
    q = np.zeros((h, w), np.int16); s = I32(); rates = np.zeros(44, np.int32); k = np.zeros(3, np.int32); e = ctypes.c_double()
    if bdpcm:
        assert R.refshim_rdoq_bdpcm(c['comp'], P(ts_inputs(row)), w, h, c['bd'], c['qp'], c['delta'], 1, c['dir_mode'], lam, c['ctx_qp'], c['init_id'], P(q),
                                    ctypes.byref(s), P(rates)) == 0
    else:
        assert R.refshim_rdoq_ts(c['comp'], P(ts_inputs(row)), w, h, c['bd'], c['qp'], c['delta'], 1, lam, c['ctx_qp'], c['init_id'], P(q), ctypes.byref(s), P(rates),
                                 P(k), ctypes.byref(e)) == 0
    R.refshim_set_simd(b'AVX2')
    return q, s.value, rates, k


def orc_rdoq(row, rates, coef=None, v2=False):
    O = dq_oracle()
    c = rd(row, RQ_COLS); w, h = c['w'], c['h']
    coef = rq_inputs(row)[None] if coef is None else coef
    n = len(coef)
    q = np.zeros((n, h, w), np.int16); s = np.zeros(n, np.int32); l = np.zeros(n, np.int32)
    f = O.orc_rdoq_v2 if v2 else O.orc_rdoq
    assert f(w, h, c['bd'], c['qp'], c['comp'], 0, 0, c['sh'], lambdas(c['qp'], c['bd'])[c['lam_idx']], 8, P(np.ascontiguousarray(rates)), P(coef), n, P(q), P(s), P(l)) == 0
    return q, s, l


def orc_dep_quant(row, rates, scalar, coef=None):
    O = dq_oracle()
    c = rd(row, RQ_COLS); w, h = c['w'], c['h']
    coef = rq_inputs(row)[None] if coef is None else coef
    n = len(coef)
    q = np.zeros((n, h, w), np.int16); s = np.zeros(n, np.int32); l = np.zeros(n, np.int32)
    assert O.orc_dep_quant(w, h, c['bd'], c['qp'], lambdas(c['qp'], c['bd'])[c['lam_idx']], 8, 0, 0, scalar, P(np.ascontiguousarray(rates)), P(coef), n, P(q), P(s), P(l)) == 0
    return q, s, l


def orc_ts(row, rates, bdpcm, coef=None):
    O = dq_oracle()
    c = rd(row, TS_COLS); w, h = c['w'], c['h']
    coef = ts_inputs(row)[None] if coef is None else coef
    n = len(coef)
    q = np.zeros((n, h, w), np.int16); s = np.zeros(n, np.int32)
    lam = lambdas(c['qp'], c['bd'])[c['lam_idx']]
    r = np.ascontiguousarray(rates)
    if bdpcm:
        assert O.orc_rdoq_bdpcm(w, h, c['bd'], c['qp'], c['delta'], c['dir_mode'], lam, P(r), P(coef), n, P(q), P(s)) == 0
    else:
        assert O.orc_rdoq_ts(w, h, c['bd'], c['qp'], c['delta'], lam, P(r), P(coef), n, P(q), P(s)) == 0
    return q, s


def orc_dq_constants(row):
    c = rd(row, RQ_COLS)
    k = np.zeros(9, np.int64)
    assert dq_oracle().orc_dep_quant_constants(c['w'], c['h'], c['bd'], c['qp'], lambdas(c['qp'], c['bd'])[c['lam_idx']], 8, P(k)) == 0
    return k


def orc_rq_constants(row):
    c = rd(row, RQ_COLS)
    k = np.zeros(7, np.int32)
    assert dq_oracle().orc_rdoq_constants(c['w'], c['h'], c['bd'], c['qp'], c['comp'], 0, 0, 8, P(k)) == 0
    return k


# ---------------------------------------------------------------------------------------------------- which limit cases a row reaches
def budget_exhausted(q, area, per_level):
    """the context-coded-bin budget ((area * 28) >> 4) certainly ran out: even the fewest bins the non-zero levels take (per_level(|l|)) exceed it"""
    a = np.abs(q[q != 0].astype(np.int64))
    return int(per_level(a).sum()) > ((area * 28) >> 4) + 8


def rq_level_beyond_int16(row, consts):
    """a coefficient of the row quantises to a level above 32768: the member stores it into TCoeffSig as it is"""
    coef = np.abs(rq_inputs(row).astype(np.int64))
    return int(((coef * int(consts[0])) >> int(consts[2])).max()) > 32768


def rq_wrapped_template(row, consts):
    """a position with a moderate level has a template neighbour (right, right + 1, diagonal, below, below + 1) whose level lies in 32769..65534: its Rice
    parameter reads that level's negative TCoeffSig"""
    c = rd(row, RQ_COLS)
    lv = (np.abs(rq_inputs(row).astype(np.int64))[:min(c['h'], 32), :min(c['w'], 32)] * int(consts[0])) >> int(consts[2])
    wrapped = np.pad((lv >= 32769) & (lv <= 65534), ((0, 2), (0, 2)))
    nb = wrapped[:-2, 1:-1] | wrapped[:-2, 2:] | wrapped[1:-1, 1:-1] | wrapped[1:-1, :-2] | wrapped[2:, :-2]
    return bool((nb & (lv >= 1) & (lv < 1000)).any())


def dq_max_qidx_hit(row, consts):
    """( |c| * qScale + qAdd ) >> qShift exceeds maxQIdx for a coefficient of the row (depquant_core.h: the index is clipped there)"""
    coef = np.abs(rq_inputs(row).astype(np.int64))
    return int(((coef * int(consts[5]) + int(consts[4])) >> int(consts[0])).max()) > int(consts[1])


def rq_tally(rows, q_of, consts_of, dq):
    t = dict(beyond_int16=0, wrapped_template=0, budget=0, max_qidx=0, below_floor=0, above_ceiling=0, sign_hidden_large=0)
    for i, row in enumerate(rows):
        c = rd(row, RQ_COLS); q = q_of(i)
        area = min(c['w'], 32) * min(c['h'], 32)
        t['budget'] += budget_exhausted(q, area, lambda a: np.where(a >= 2, 4, 2))
        t['below_floor'] += c['qp'] + 6 * (c['bd'] - 8) < 0
        t['above_ceiling'] += c['qp'] > 63
        if dq:
            t['max_qidx'] += dq_max_qidx_hit(row, consts_of(i))
        else:
            t['beyond_int16'] += rq_level_beyond_int16(row, consts_of(i))
            t['wrapped_template'] += rq_wrapped_template(row, consts_of(i))
            t['sign_hidden_large'] += bool(c['sh'] and np.abs(q.astype(np.int32)).max() > 1000)
    return t


def ts_tally(rows, q_of):
    t = dict(at_32767=0, budget=0, below_ts_floor=0, above_ts_floor=0, pel_max=0)
    for i, row in enumerate(rows):
        c = rd(row, TS_COLS); q = q_of(i)
        t['at_32767'] += int(np.abs(q.astype(np.int32)).max() >= 32767)
        t['budget'] += budget_exhausted(q, c['w'] * c['h'], lambda a: np.full(a.shape, 3))
        f = 4 + 6 * c['delta']; iq = internal_qp(c['qp'], c['bd'])
        t['below_ts_floor'] += iq < f
        t['above_ts_floor'] += iq > f
        t['pel_max'] += c['pattern'] in (3, 4)
    return t


# ---------------------------------------------------------------------------------------------------- CPU: the oracle against the golden file and the members
@pytest.fixture(scope='module')
def golden_v9():
    return np.load(GOLDEN)


def test_golden_v9_inputs_and_coverage(golden_v9):
    """the rows and the regenerated inputs are the ones the file was made from, and every limit axis occurs in the members' own results"""
    g = golden_v9
    for key, rows, inputs in (('rq', rq_cases(), rq_inputs), ('dq', rq_cases(dq=True), rq_inputs), ('ts', ts_cases(), ts_inputs)):
        assert np.array_equal(g[key + '_cases'], rows), key
        assert [crc(inputs(r)) for r in rows] == [int(v) for v in g[key + '_crc']], key
    rq = rq_tally(g['rq_cases'], lambda i: g['rq_q_%d' % i], lambda i: g['rq_consts'][i], False)
    dq = rq_tally(g['dq_cases'], lambda i: g['dq_q1_%d' % i], lambda i: g['dq_consts'][i], True)
    ts = ts_tally(g['ts_cases'], lambda i: g['ts_q_%d' % i])
    bd = ts_tally(g['ts_cases'], lambda i: g['bd_q_%d' % i])
    print('fast RDOQ', rq, 'DepQuant', dq, 'transform skip', ts, 'BDPCM', bd)
    assert rq['beyond_int16'] >= 10 and rq['wrapped_template'] >= 6 and rq['budget'] >= 10 and rq['sign_hidden_large'] >= 5 and rq['below_floor'] >= 36 and rq['above_ceiling'] >= 36, rq
    assert dq['max_qidx'] >= 10 and dq['budget'] >= 10 and dq['below_floor'] >= 20 and dq['above_ceiling'] >= 20, dq
    for t in (ts, bd):
        assert t['at_32767'] >= 10 and t['budget'] >= 10 and t['below_ts_floor'] >= 30 and t['above_ts_floor'] >= 30 and t['pel_max'] >= 30, t
    assert len(g['dq_cases']) >= 150 and int((g['dq_meta'][:, 1] >= 0).sum()) > 60


def test_oracle_equals_golden_v9(golden_v9):
    """the shared texts compiled for the CPU give the members' levels, sums, last positions and constants at every limit row"""
    g = golden_v9
    bad = []
    for i, row in enumerate(g['rq_cases']):
        for v2 in (False, True):
            q, s, l = orc_rdoq(row, g['rq_rates'][i], v2=v2)
            if not (np.array_equal(q[0], g['rq_q_%d' % i]) and [int(s[0]), int(l[0])] == [int(v) for v in g['rq_meta'][i]]):
                bad.append(('rdoq', 'engine 2' if v2 else 'engine 1', i))
        if not np.array_equal(orc_rq_constants(row), g['rq_consts'][i]):
            bad.append(('rdoq constants', i))
    for i, row in enumerate(g['dq_cases']):
        for scalar in (0, 1):
            q, s, l = orc_dep_quant(row, g['dq_rates'][i], scalar)
            key = 'dq_q%d_%d' % (1 - scalar, i)                        # dq_q0: the scalar members, dq_q1: the x86 ones
            if not (np.array_equal(q[0], g[key]) and [int(s[0]), int(l[0])] == [int(v) for v in g['dq_meta'][i, 2 * (1 - scalar):2 * (1 - scalar) + 2]]):
                bad.append(('dep_quant', scalar, i))
        if not np.array_equal(orc_dq_constants(row), g['dq_consts'][i]):
            bad.append(('dep_quant constants', i))
    for i, row in enumerate(g['ts_cases']):
        for bdpcm, key in ((False, 'ts'), (True, 'bd')):
            q, s = orc_ts(row, g['ts_rates'][i], bdpcm)
            if not (np.array_equal(q[0], g['%s_q_%d' % (key, i)]) and int(s[0]) == int(g[key + '_abs_sum'][i])):
                bad.append((key, i))
    assert bad == [], (len(bad), bad[:10])


@needs_ref
def test_members_equal_golden_v9(golden_v9):
    """the reference's members (scalar and AVX2 / x86 builds) still produce the file's results, rates and constants on the regenerated inputs"""
    g = golden_v9
    bad = []
    for i, row in enumerate(g['rq_cases']):
        for opt in (0, 1):
            q, s, l, rates, k = ref_rdoq(row, opt)
            if not (np.array_equal(q, g['rq_q_%d' % i]) and [s, l] == [int(v) for v in g['rq_meta'][i]] and np.array_equal(rates, g['rq_rates'][i])
                    and np.array_equal(k, g['rq_consts'][i])):
                bad.append(('rdoq', opt, i))
    for i, row in enumerate(g['dq_cases']):
        for opt in (0, 1):
            q, s, l, rates, k = ref_dep_quant(row, opt)
            if not (np.array_equal(q, g['dq_q%d_%d' % (opt, i)]) and [s, l] == [int(v) for v in g['dq_meta'][i, 2 * opt:2 * opt + 2]]
                    and np.array_equal(rates, g['dq_rates'][i]) and np.array_equal(k, g['dq_consts'][i])):
                bad.append(('dep_quant', opt, i))
    for i, row in enumerate(g['ts_cases']):
        for opt in (0, 1):
            q, s, rates, k = ref_ts(row, opt, False)
            if not (np.array_equal(q, g['ts_q_%d' % i]) and s == int(g['ts_abs_sum'][i]) and np.array_equal(rates, g['ts_rates'][i])):
                bad.append(('ts', opt, i))
            q, s, _, _ = ref_ts(row, opt, True)
            if not (np.array_equal(q, g['bd_q_%d' % i]) and s == int(g['bd_abs_sum'][i])):
                bad.append(('bdpcm', opt, i))
    assert bad == [], (len(bad), bad[:10])


def test_dep_quant_qp_is_clipped_like_qp_param():
    """below the floor and above the ceiling the DepQuant constants are those of the clipped QP, as QpParam (Quant.cpp:109) makes them for the reference; the
    library's constants call agrees with the oracle"""
    import vvenc_b200._lib as L
    lib = L.load()
    D = dq_oracle()
    for bd in (8, 10):
        o = 6 * (bd - 8)
        for (w, h) in ((4, 4), (8, 4), (64, 64), (32, 16)):
            lam = 1.0
            ref = {}
            for qp in qp_ends(bd):
                k = np.zeros(9, np.int64)
                assert D.orc_dep_quant_constants(w, h, bd, qp, lam, 8, P(k)) == 0
                par = L.vvb_tu_par(w, h, 0, 0, bd, qp, 0, 1, 0, 0, 0, 0, 0, 0, 0)
                dq = L.vvb_dq_par(lam, 8, 0, 0, 0)
                kl = np.zeros(9, np.int64)
                assert lib.vvb_dep_quant_constants(ctypes.byref(par), ctypes.byref(dq), P(kl)) == 0
                assert np.array_equal(k, kl), (w, h, bd, qp)
                assert int(k[5]) > 0, (w, h, bd, qp)                      # a scale from the table, not from before its start
                ref[qp] = k
            assert np.array_equal(ref[-o - 2], ref[-o]) and np.array_equal(ref[-o - 1], ref[-o]) and np.array_equal(ref[64], ref[63]), (w, h, bd)
            assert not np.array_equal(ref[-o], ref[0]) or o == 0


def test_library_constants_equal_golden_v9(golden_v9):
    """vvb_rdoq_constants and vvb_dep_quant_constants (host calls of the library, no device) at the QP ends against the members' constants"""
    import vvenc_b200._lib as L
    lib = L.load()
    g = golden_v9
    for i, row in enumerate(g['rq_cases']):
        c = rd(row, RQ_COLS)
        par = L.vvb_tu_par(c['w'], c['h'], 0, 0, c['bd'], c['qp'], 0, 0, c['sh'], 0, 0, 0, 0, 0, c['comp'])
        rq = L.vvb_rdoq_par(lambdas(c['qp'], c['bd'])[c['lam_idx']], 8, 0)
        k = np.zeros(7, np.int32)
        assert lib.vvb_rdoq_constants(ctypes.byref(par), ctypes.byref(rq), P(k)) == 0 and np.array_equal(k, g['rq_consts'][i]), (i, c)
    for i, row in enumerate(g['dq_cases']):
        c = rd(row, RQ_COLS)
        par = L.vvb_tu_par(c['w'], c['h'], 0, 0, c['bd'], c['qp'], 0, 1, 0, 0, 0, 0, 0, 0, 0)
        dq = L.vvb_dq_par(lambdas(c['qp'], c['bd'])[c['lam_idx']], 8, 0, 0, 0)
        k = np.zeros(9, np.int64)
        assert lib.vvb_dep_quant_constants(ctypes.byref(par), ctypes.byref(dq), P(k)) == 0 and np.array_equal(k, g['dq_consts'][i]), (i, c)


# ---------------------------------------------------------------------------------------------------- the one-call round trip at the QP ends
def rt_cases():
    """tu_rdo_cases rows at the QP ends: both quantisers, 8 and 10 bits, full-scale and mid-range residuals, a few shapes (64 x 64 included)"""
    import tu_rdo_cases as T
    rows = []
    k = 0
    for quantiser in (1, 2):
        for bd in (8, 10):
            for qp in qp_ends(bd):
                for (w, h) in ((64, 64), (8, 8), (16, 4)):
                    k += 1
                    lam = enc_lambda(qp, bd)
                    if quantiser == 2 and not dq_defined(w, h, bd, qp, lam):
                        continue
                    amp = (1 << bd) - 1 if k % 2 else 40
                    rows.append([quantiser, w, h, 0, 0, 0, 0, 0, bd, qp, k % 2, int(quantiser == 1 and k % 3 == 0), k % 2, int(lam * 1000) or 1, amp, k % 3, 9100 + k])
    return np.array(rows, dtype=np.int64)


@needs_ref
def test_oracle_round_trip_equals_the_members_at_qp_ends(golden_v9):
    """the oracle composition of tu_rdo_cases (forward, quantiser, the matching dequantiser and inverse) against the members one after the other at the QP ends:
    with dependent quantisation the quantiser and the dequantiser must use the same clipped QP"""
    import tu_rdo_cases as T
    bad = []
    for i, row in enumerate(rt_cases()):
        org, pred = T.inputs(row)
        q, reco, m, need, rates, _ = T.ref_roundtrip_rdo(row, org[0], pred[0])
        oq, oreco, om, oneed = T.oracle_roundtrip_rdo(row, org[0], pred[0], rates)
        if not (np.array_equal(q, oq) and np.array_equal(reco, oreco) and m == om and need == oneed):
            bad.append((i, T.row_dict(row)))
    assert bad == [], (len(bad), bad[:3])


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope='module')
def eng():
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def rq_par(eng, c, dq=False):
    return eng.tu_par(c['w'], c['h'], 0, 0, c['bd'], c['qp'], dep_quant=dq, sign_hiding=bool(c.get('sh', 0)), is_chroma=bool(c['comp']))


def ts_par(eng, c):
    return eng.tu_par(c['w'], c['h'], 0, 0, c['bd'], c['qp'], transform_skip=True, input_bit_depth_delta=c['delta'], is_chroma=bool(c['comp']))


def resident(kind):
    """TUs one launch holds before its threads stride over the list (grid caps of capi.cu: 64-thread CTAs, 16 / 8 CTAs per SM; DepQuant engine 1: 32 TUs per CTA)"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {'rdoq': sms * 16 * 64, 'ts': sms * 16 * 64, 'bdpcm': sms * 8 * 64, 'dq0': sms * 8 * 64, 'dq1': sms * 16 * 32}[kind]


@pytest.mark.gpu
def test_gpu_rdoq_limits_equal_golden_v9(eng, golden_v9):
    g = golden_v9
    bad = []
    for engine in (1, 2):
        eng.set_rdoq_engine(engine)
        try:
            for i, row in enumerate(g['rq_cases']):
                c = rd(row, RQ_COLS)
                r = eng.rdoq(rq_par(eng, c), eng.rdoq_rates(g['rq_rates'][i]), rq_inputs(row)[None], lambdas(c['qp'], c['bd'])[c['lam_idx']])
                if not (np.array_equal(r['q'][0], g['rq_q_%d' % i]) and [int(r['abs_sum'][0]), int(r['last_pos'][0])] == [int(v) for v in g['rq_meta'][i]]):
                    bad.append((engine, i, c))
        finally:
            eng.set_rdoq_engine(1)
    assert bad == [], (len(bad), bad[:5])


@pytest.mark.gpu
def test_gpu_dep_quant_limits_equal_golden_v9(eng, golden_v9):
    g = golden_v9
    bad = []
    for engine in (0, 1):
        eng.set_depquant_engine(engine)
        try:
            for i, row in enumerate(g['dq_cases']):
                c = rd(row, RQ_COLS)
                for scalar in (0, 1):
                    r = eng.dep_quant(rq_par(eng, c, True), eng.dq_rates(g['dq_rates'][i]), rq_inputs(row)[None], lambdas(c['qp'], c['bd'])[c['lam_idx']],
                                      scalar_members=bool(scalar))
                    j = 1 - scalar
                    if not (np.array_equal(r['q'][0], g['dq_q%d_%d' % (j, i)]) and [int(r['abs_sum'][0]), int(r['last_pos'][0])] == [int(v) for v in g['dq_meta'][i, 2 * j:2 * j + 2]]):
                        bad.append((engine, scalar, i, c))
        finally:
            eng.set_depquant_engine(1)
    assert bad == [], (len(bad), bad[:5])


@pytest.mark.gpu
def test_gpu_ts_and_bdpcm_limits_equal_golden_v9(eng, golden_v9):
    g = golden_v9
    bad = []
    for i, row in enumerate(g['ts_cases']):
        c = rd(row, TS_COLS)
        lam = lambdas(c['qp'], c['bd'])[c['lam_idx']]
        rates = eng.rdoq_ts_rates(g['ts_rates'][i])
        r = eng.rdoq_ts(ts_par(eng, c), rates, ts_inputs(row)[None], lam)
        if not (np.array_equal(r['q'][0], g['ts_q_%d' % i]) and int(r['abs_sum'][0]) == int(g['ts_abs_sum'][i])):
            bad.append(('ts', i, c))
        r = eng.rdoq_bdpcm(ts_par(eng, c), rates, ts_inputs(row)[None], lam, c['dir_mode'])
        if not (np.array_equal(r['q'][0], g['bd_q_%d' % i]) and int(r['abs_sum'][0]) == int(g['bd_abs_sum'][i])):
            bad.append(('bdpcm', i, c))
    assert bad == [], (len(bad), bad[:5])


def _batch(rows, inputs, n, seed):
    """n TUs drawn from the limit rows of one shape (their inputs, with random sign flips and zeroed positions so that TUs differ)"""
    rs = np.random.RandomState(seed)
    base = np.stack([inputs(r) for r in rows])
    x = base[rs.randint(len(base), size=n)].astype(np.int64)
    x *= np.where(rs.rand(*x.shape) < 0.5, -1, 1)
    x[rs.rand(*x.shape) < 0.3] = 0
    return np.clip(x, -32768, 32767).astype(np.int32)


def _call(eng, kind, c, rates, coef, n, need, with_sums=True, sentinel=0x5A5A):
    """the C ABI call of one kernel with raw buffers (nullable outputs null when with_sums is False); returns rc, q, abs_sum, last_pos"""
    import vvenc_b200._lib as L
    h, w = c['h'], c['w']
    q = np.full((max(n, 1), h, w), sentinel, np.int16); s = np.full(max(n, 1), sentinel, np.int32); l = np.full(max(n, 1), sentinel, np.int32)
    nr = None if need is None else np.ascontiguousarray(need, np.uint8)
    ps, pl = (P(s), P(l)) if with_sums else (None, None)
    lam = lambdas(c['qp'], c['bd'])[c['lam_idx']]
    if kind == 'rdoq':
        rq = L.vvb_rdoq_par(lam, 8, 0)
        rc = eng.lib.vvb_rdoq(eng.h, ctypes.byref(rq_par(eng, c)), ctypes.byref(rq), ctypes.byref(eng.rdoq_rates(rates)), P(coef), P(nr) if nr is not None else None, n, P(q), ps, pl)
    elif kind in ('dq0', 'dq1'):
        dq = L.vvb_dq_par(lam, 8, 0, 0, 0)
        rc = eng.lib.vvb_dep_quant(eng.h, ctypes.byref(rq_par(eng, c, True)), ctypes.byref(dq), ctypes.byref(eng.dq_rates(rates)), P(coef), P(nr) if nr is not None else None, n,
                                   P(q), ps, pl)
    elif kind == 'ts':
        rc = eng.lib.vvb_rdoq_ts(eng.h, ctypes.byref(ts_par(eng, c)), ctypes.c_double(lam), ctypes.byref(eng.rdoq_ts_rates(rates)), P(coef), P(nr) if nr is not None else None,
                                 n, P(q), ps)
    else:
        rc = eng.lib.vvb_rdoq_bdpcm(eng.h, ctypes.byref(ts_par(eng, c)), ctypes.c_double(lam), c['dir_mode'], ctypes.byref(eng.rdoq_ts_rates(rates)), P(coef),
                                    P(nr) if nr is not None else None, n, P(q), ps)
    return rc, q[:n], s[:n], l[:n]


def _expect(kind, row, rates, coef, need):
    """the oracle's results for a batch, with the need_rdoq mask applied as the kernels apply it (all-zero levels, abs_sum 0, last_pos -1)"""
    if kind == 'rdoq':
        q, s, l = orc_rdoq(row, rates, coef)
    elif kind in ('dq0', 'dq1'):
        q, s, l = orc_dep_quant(row, rates, 0, coef)
    else:
        q, s = orc_ts(row, rates, kind == 'bdpcm', coef)
        l = np.full(len(q), -1, np.int32)
    if need is not None:
        off = np.asarray(need) == 0
        q[off] = 0; s[off] = 0; l[off] = -1
    return q, s, l


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['rdoq', 'rdoq2', 'dq0', 'dq1', 'ts', 'bdpcm'])
def test_gpu_tu_counts_masks_and_null_outputs(eng, golden_v9, kind):
    """n = 0 (returns OK, sentinel outputs untouched), 1, 63, 64, 65 and above the resident grid (threads stride over the list and reuse their arena slots);
    need_rdoq all 0, all 1, null and mixed; abs_sum / last_pos null -- each against the oracle on the same inputs, at the lowest QP of 10 bits"""
    g = golden_v9
    base = 'rdoq' if kind == 'rdoq2' else kind
    ts = base in ('ts', 'bdpcm')
    key = 'ts' if ts else ('dq' if base.startswith('dq') else 'rq')
    pick = [i for i, r in enumerate(g[key + '_cases']) if int(r[0]) == 4 and int(r[1]) == 4 and int(r[2]) == 10]
    rows = [g[key + '_cases'][i] for i in pick]
    row = rows[0]
    c = rd(row, TS_COLS if ts else RQ_COLS)
    rates = g[key + '_rates'][pick[0]]
    inputs = ts_inputs if ts else rq_inputs
    if kind == 'rdoq2':
        eng.set_rdoq_engine(2)
    if base.startswith('dq'):
        eng.set_depquant_engine(int(base[2]))
    try:
        rc, q, s, l = _call(eng, base, c, rates, np.zeros((1, 4, 4), np.int32), 0, None)
        assert rc == 0 and (q == 0x5A5A).all() and (s == 0x5A5A).all()
        big = resident(base) + 65
        rs = np.random.RandomState(len(kind))
        for n, need in ((1, None), (63, None), (64, 'ones'), (65, 'mixed'), (65, 'zeros'), (big, 'mixed')):
            coef = _batch(rows, inputs, n, n)
            nr = None if need is None else np.ones(n, np.uint8) if need == 'ones' else np.zeros(n, np.uint8) if need == 'zeros' else (rs.rand(n) < 0.8).astype(np.uint8)
            eq, es, el = _expect(base, row, rates, coef, nr)
            for with_sums in (True, False):
                rc, q, s, l = _call(eng, base, c, rates, coef, n, nr, with_sums)
                assert rc == 0 and np.array_equal(q, eq), (kind, n, need, with_sums, int((q != eq).any(axis=(1, 2)).sum()))
                if with_sums:
                    assert np.array_equal(s, es), (kind, n, need)
                    if not ts:
                        assert np.array_equal(l, el), (kind, n, need)
                else:
                    assert (s == 0x5A5A).all() and (l == 0x5A5A).all()
            if need == 'zeros':
                assert not eq.any()
            elif n >= 64:
                assert (es > 0).sum() > n // 4, (kind, n)
    finally:
        eng.set_rdoq_engine(1); eng.set_depquant_engine(1)


@pytest.mark.gpu
def test_gpu_large_bdpcm_batch_after_small_one(golden_v9):
    """the BDPCM reconstruction arena grows (and is reallocated) between two calls of one context: the second call equals the oracle"""
    import vvenc_b200 as V
    g = golden_v9
    pick = [i for i, r in enumerate(g['ts_cases']) if int(r[0]) == 32 and int(r[1]) == 32 and int(r[2]) == 10]
    rows = [g['ts_cases'][i] for i in pick]
    c = rd(rows[0], TS_COLS); rates = g['ts_rates'][pick[0]]
    e = V.CostEngine(0)
    try:
        small = _batch(rows, ts_inputs, 1, 1)
        rc, q, s, _ = _call(e, 'bdpcm', c, rates, small, 1, None)
        assert rc == 0 and np.array_equal(q, _expect('bdpcm', rows[0], rates, small, None)[0])
        n = 8000
        big = _batch(rows, ts_inputs, n, 2)
        rc, q, s, _ = _call(e, 'bdpcm', c, rates, big, n, None)
        eq, es, _ = _expect('bdpcm', rows[0], rates, big, None)
        assert rc == 0 and np.array_equal(q, eq) and np.array_equal(s, es), int((q != eq).any(axis=(1, 2)).sum())
    finally:
        e.close()


@pytest.mark.gpu
def test_gpu_round_trip_rdo_at_qp_ends(eng, golden_v9):
    """vvb_tu_roundtrip_rdo at the QP ends against the members' round trip (the file), the three-call device chain and the oracle composition"""
    import tu_rdo_cases as T
    from test_gpu_tu_rdo_roundtrip import call, chain, res_rows, same
    g = golden_v9
    rows = rt_cases()
    assert np.array_equal(rows, g['rt_cases'])
    bad = []
    for i, row in enumerate(rows):
        c = T.row_dict(row)
        org, pred = T.inputs(row, 4)
        rates = g['rt_rates_%d' % i]
        r = call(eng, c, org, pred, rates)
        m = [int(v) for v in g['rt_meta'][i]]
        if not (np.array_equal(r['q'][0], g['rt_q_%d' % i]) and np.array_equal(r['reco'][0], pred[0] + g['rt_dreco_%d' % i])
                and res_rows(r['res'])[0].tolist() == m[:5] and int(r['need_rdoq'][0]) == m[5]):
            bad.append(('golden', i, c))
        if not same((r['q'], r['reco'], res_rows(r['res']), r['need_rdoq']), chain(eng, c, org, pred, rates)):
            bad.append(('chain', i, c))
        for k in range(4):
            oq, oreco, om, oneed = T.oracle_roundtrip_rdo(row, org[k], pred[k], rates)
            if not same((r['q'][k], r['reco'][k], res_rows(r['res'])[k], r['need_rdoq'][k]), (oq, oreco, om, oneed)):
                bad.append(('oracle', i, k, c))
    assert bad == [], (len(bad), bad[:3])
