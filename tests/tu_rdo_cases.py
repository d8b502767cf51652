"""The TU round trip with the slice's quantiser (vvb_tu_roundtrip_rdo*): seeded cases and two compositions that compute what it must return.

  oracle_roundtrip_rdo -- the CPU oracle: oracle.c forward (+ LFNST) and xNeedRDOQ -> rdoq_oracle / depquant_oracle -> oracle.c dequantiser (plain or
                          DepQuant's) and inverse -> reconstruct -> SSE
  ref_roundtrip_rdo    -- the unmodified reference's members through oracle/_ref, one step after the other in the order DepQuant::quant /
                          QuantRDOQ2::quant and xIntraCodingTUBlock call them; the quantiser step also returns the rate tables it read from its CABAC state.
                          Quant::xNeedRDOQ reads the coefficients, the TU size, the QP, the component and the transform-skip flag only, so for MTS and
                          LFNST TUs it runs on the coefficients the transform left (refshim_need_rdoq, with the slice's dependent-quantisation flag)

A case row: quantiser (1 fast RDOQ, 2 dependent quantisation), w, h, tr_hor, tr_ver, lfnst_idx, intra_mode, comp (0 luma, 1 Cb), bit_depth, qp, is_irap,
sign_hiding, selective, lambda * 1000, amplitude (of the residual, in pels), ctx_init_id, seed.  Transform types use the vvb_tu_par numbering (0 DCT-II,
1 DCT-VIII, 2 DST-VII).  Dependent quantisation's zero_out is the condition the encoder evaluates for a luma TU with an MTS pair (mtsIdx > MTS_SKIP)."""
import ctypes
import numpy as np
from _libs import oracle, dq_oracle, refshim, P

COLS = ('quantiser', 'w', 'h', 'th', 'tv', 'lfnst', 'mode', 'comp', 'bd', 'qp', 'irap', 'sh', 'sel', 'lam1000', 'amp', 'init_id', 'seed')
SHAPES = [(w, h) for w in (4, 8, 16, 32, 64) for h in (4, 8, 16, 32, 64)]
MTS_IDX = {(0, 0): 0, (2, 2): 2, (1, 2): 3, (2, 1): 4, (1, 1): 5}          # (tr_hor, tr_ver) -> tu.mtsIdx (MTS_DST7_DST7 = 2 ... MTS_DCT8_DCT8 = 5)
LFNST_MODES = (0, 1, 2, 18, 34, 50, 66)


def row_dict(row):
    return dict(zip(COLS, [int(v) for v in row]))


def zero_out(c):
    return int(c['quantiser'] == 2 and c['comp'] == 0 and MTS_IDX[(c['th'], c['tv'])] > 1)


def cases(n=300, seed=8101):
    """about n rows over both quantisers, luma and Cb, 8 and 10 bits, QP 17..51, the 25 shapes, MTS pairs, LFNST 1/2 on 4x4 / 8x8 / 16x16, sign hiding on and
    off (fast RDOQ), selective on and off, and residuals from flat to full scale"""
    rs = np.random.RandomState(seed)
    rows = []
    k = 0
    while len(rows) < n:
        w, h = SHAPES[k % 25]
        quantiser = 1 + (k // 25) % 2
        k += 1
        comp = int(rs.randint(2))
        th = tv = 0; lf = 0; mode = 0
        if comp == 0 and w <= 32 and h <= 32 and rs.rand() < 0.35:
            th, tv = [(2, 2), (1, 2), (2, 1), (1, 1)][rs.randint(4)]
        elif comp == 0 and (w, h) in ((4, 4), (8, 8), (16, 16)) and rs.rand() < 0.5:
            lf = 1 + int(rs.randint(2)); mode = int(rs.choice(LFNST_MODES))
        bd = 8 if rs.rand() < 0.4 else 10
        qp = int(rs.choice([17, 22, 27, 32, 37, 42, 47, 51]))
        sh = int(quantiser == 1 and rs.rand() < 0.5)
        sel = int(rs.rand() < 0.6)
        lam = float(rs.choice([3.0, 11.7, 30.0, 57.3, 120.0, 800.0]))
        amp = int(rs.choice([0, 2, 8, 40, 200, (1 << bd) - 1]))
        rows.append([quantiser, w, h, th, tv, lf, mode, comp, bd, qp, int(rs.randint(2)), sh, sel, int(lam * 1000), amp, int(rs.randint(3)), seed * 1000 + k])
    return np.array(rows, dtype=np.int64)


def inputs_crc(org, pred):
    """CRC-32 of a case's inputs, which the golden file stores so that a change of inputs() cannot go unnoticed"""
    import zlib
    return zlib.crc32(np.ascontiguousarray(pred, dtype=np.int16).tobytes(), zlib.crc32(np.ascontiguousarray(org, dtype=np.int16).tobytes()))


def inputs(row, count=1):
    """org, pred int16 [count][h][w] of a case: a prediction inside the bit depth and an original within +-amp of it (clipped), smoother in the low frequencies"""
    c = row_dict(row)
    rs = np.random.RandomState(c['seed'] & 0x7fffffff)
    w, h, mx = c['w'], c['h'], (1 << c['bd']) - 1
    pred = rs.randint(0, mx + 1, size=(count, h, w))
    if c['amp'] >= mx:                                             # full scale: the sign of each TU's residual chosen per pel
        org = np.where(rs.rand(count, h, w) < 0.5, 0, mx)
    else:
        org = pred + rs.randint(-c['amp'], c['amp'] + 1, size=(count, h, w))
    return np.clip(org, 0, mx).astype(np.int16), pred.astype(np.int16)


def _sse(a, b):
    d = a.astype(np.int64) - b.astype(np.int64)
    return int((d * d).sum())


def _finish(org, pred, rec, bd):
    reco = np.clip(pred.astype(np.int32) + rec, 0, (1 << bd) - 1).astype(np.int16)
    resi = org.astype(np.int32) - pred.astype(np.int32)
    return reco, [_sse(org, reco), _sse(resi, rec), _sse(resi, np.zeros_like(resi))]


def oracle_roundtrip_rdo(row, org, pred, rates, lfnst_st=(0, 0)):
    """one TU through the CPU oracle -> (q [h][w], reco [h][w], [dist_reco, dist_resi, dist_zero, abs_sum, last_pos], need_rdoq)"""
    O, D = oracle(), dq_oracle()
    c = row_dict(row)
    w, h, bd, qp = c['w'], c['h'], c['bd'], c['qp']
    dq = c['quantiser'] == 2
    resi = np.ascontiguousarray(org.astype(np.int32) - pred.astype(np.int32)).astype(np.int16)
    coef = np.zeros((h, w), dtype=np.int32); qf = np.zeros((h, w), dtype=np.int16); s = ctypes.c_int32(); lp = ctypes.c_int32()
    st, tr = lfnst_st
    if c['lfnst']:
        assert O.orc_transform_quant_lfnst(P(resi), w, w, h, bd, qp, c['irap'], 0, st, c['lfnst'], tr, P(coef), P(qf), ctypes.byref(s), ctypes.byref(lp)) == 0
    else:
        assert O.orc_transform_quant_ex(c['th'], c['tv'], P(resi), w, w, h, bd, qp, c['irap'], 0, P(coef), P(qf), ctypes.byref(s), ctypes.byref(lp)) == 0
    need = int(O.orc_need_rdoq_ex(P(coef), w, h, bd, qp, int(dq), 0, 0, c['comp']))
    q = np.zeros((h, w), dtype=np.int16); s = np.zeros(1, dtype=np.int32); lp = np.full(1, -1, dtype=np.int32)
    if not (c['sel'] and not need):
        r = np.ascontiguousarray(rates, dtype=np.int32)
        if dq and c['comp']:
            assert D.orc_dep_quant_chroma(w, h, bd, qp, c['lam1000'] / 1000.0, 8, int(c['lfnst'] > 0), 0, P(r), P(coef), 1, P(q), P(s), P(lp)) == 0
        elif dq:
            assert D.orc_dep_quant(w, h, bd, qp, c['lam1000'] / 1000.0, 8, zero_out(c), int(c['lfnst'] > 0), 0, P(r), P(coef), 1, P(q), P(s), P(lp)) == 0
        else:
            assert D.orc_rdoq(w, h, bd, qp, c['comp'], int(c['lfnst'] > 0), 0, c['sh'], c['lam1000'] / 1000.0, 8, P(r), P(coef), 1, P(q), P(s), P(lp)) == 0
    rec = np.zeros((h, w), dtype=np.int32)
    if s[0] > 0:
        cO = np.zeros((h, w), dtype=np.int32); rO = np.zeros((h, w), dtype=np.int16)
        if c['lfnst']:
            assert O.orc_inv_transform_quant_lfnst(P(q), w, h, bd, qp, int(dq), st, c['lfnst'], tr, P(cO), P(rO), w) == 0
        elif dq:
            assert O.orc_inv_transform_quant_dq(c['th'], c['tv'], P(q), w, h, bd, qp, P(cO), P(rO), w) == 0
        else:
            assert O.orc_inv_transform_quant(c['th'], c['tv'], P(q), w, h, bd, qp, P(cO), P(rO), w) == 0
        rec = rO.astype(np.int32)
    reco, d = _finish(org, pred, rec, bd)
    return q, reco, d + [int(s[0]), int(lp[0])], need


def ref_roundtrip_rdo(row, org, pred, simd=b'AVX2'):
    """one TU through the reference's members (oracle/_ref) -> (q, reco, [dist_reco, dist_resi, dist_zero, abs_sum, last_pos], need_rdoq, rates, (lfnst set,
    transpose)).  The rates are the tables the quantiser read from the CABAC contexts of slice QP = qp, init type init_id."""
    R = refshim()
    R.refshim_set_simd(simd)
    c = row_dict(row)
    w, h, bd, qp, comp = c['w'], c['h'], c['bd'], c['qp'], c['comp']
    dq = c['quantiser'] == 2
    lam = c['lam1000'] / 1000.0
    intra = 1 if c['lfnst'] else int(c['seed'] & 1)
    resi = np.ascontiguousarray(org.astype(np.int32) - pred.astype(np.int32)).astype(np.int16)
    coef = np.zeros((h, w), dtype=np.int32); qf = np.zeros((h, w), dtype=np.int16); s = ctypes.c_int32(); lp = ctypes.c_int32(); nr = ctypes.c_int32()
    st = np.zeros(2, dtype=np.int32)
    if c['lfnst']:
        assert R.refshim_transform_quant_lfnst(P(resi), w, w, h, bd, qp, c['irap'], 0, c['mode'], c['lfnst'], P(coef), P(qf), ctypes.byref(s), ctypes.byref(lp),
                                               ctypes.byref(nr), P(st)) == 0
        need = int(R.refshim_need_rdoq(P(coef), w, h, bd, qp, int(dq)))
        assert dq or need == nr.value                             # the LFNST rig's own xNeedRDOQ (its slice has no dependent quantisation)
    elif (c['th'], c['tv']) != (0, 0):
        assert R.refshim_transform_quant(c['th'], c['tv'], P(resi), w, w, h, bd, qp, c['irap'], P(coef), P(qf), ctypes.byref(s), ctypes.byref(lp)) == 0
        need = int(R.refshim_need_rdoq(P(coef), w, h, bd, qp, int(dq)))
    else:
        assert R.refshim_transform_quant_ts(P(resi), w, w, h, bd, qp, c['irap'], 0, int(dq), 0, 0, comp, P(coef), P(qf), ctypes.byref(s), ctypes.byref(lp),
                                            ctypes.byref(nr)) == 0
        need = int(nr.value)
    q = np.zeros((h, w), dtype=np.int16); s = ctypes.c_int32(0); lp = ctypes.c_int32(-1)
    if dq:
        rates = np.zeros(266, dtype=np.int32)
        assert R.refshim_dep_quant_comp(comp, P(coef), w, h, bd, qp, MTS_IDX[(c['th'], c['tv'])], intra, c['lfnst'], 0, lam, 8, 1, qp, c['init_id'],
                                        P(q), ctypes.byref(s), ctypes.byref(lp), P(rates), None) == 0
    else:
        rates = np.zeros(190, dtype=np.int32)
        assert R.refshim_rdoq(comp, P(coef), w, h, bd, qp, intra, c['lfnst'], 0, c['sh'], 0, lam, 8, qp, c['init_id'], P(q), ctypes.byref(s), ctypes.byref(lp),
                              P(rates), None) == 0
    if c['sel'] and not need:                                     # DepQuant::quant :1464-1468, QuantRDOQ2::quant :291-295: no levels
        q[:] = 0; s = ctypes.c_int32(0); lp = ctypes.c_int32(-1)
    rec = np.zeros((h, w), dtype=np.int32)
    if s.value > 0:
        cO = np.zeros((h, w), dtype=np.int32); rO = np.zeros((h, w), dtype=np.int16); st2 = np.zeros(2, dtype=np.int32)
        if c['lfnst']:
            assert R.refshim_inv_transform_quant_lfnst(P(q), w, h, bd, qp, int(dq), lp.value, c['mode'], c['lfnst'], P(cO), P(rO), w, P(st2)) == 0
        elif dq:
            assert R.refshim_inv_transform_quant_dq(c['th'], c['tv'], P(q), lp.value, w, h, bd, qp, P(cO), P(rO), w) == 0
        else:
            assert R.refshim_inv_transform_quant(c['th'], c['tv'], P(q), w, h, bd, qp, P(cO), P(rO), w) == 0
        rec = rO.astype(np.int32)
    reco, d = _finish(org, pred, rec, bd)
    return q, reco, d + [int(s.value), int(lp.value)], need, rates, (int(st[0]), int(st[1]))
