"""The TU path -- vvb_fwd_trquant*, vvb_inv_trquant*, vvb_tu_roundtrip* and the TU stage of vvb_search_refine_tu -- at the limits of its number formats and
geometry, bit for bit against the CPU oracle:
  * worst-case residuals built here (residual = org - pred lies in [-pelMax, pelMax]): constant +-pelMax, pelMax * sign( T_v[k][y] * T_h[l][x] ) for DCT-II,
    DST-VII and DCT-VIII bases (the transform matrices are read from oracle/vvc_tables.h), checkerboards, stripes and random +-pelMax;
  * 8, 10, 11 and 12 bits at QP -6 * (bd - 8) - 1, -6 * (bd - 8), 0, 63 and 64, so that the clip of the base QP is crossed on both sides;
  * every admitted shape (sides 4..64, MTS pairs at 32 with their 16-wide zero-out), forward levels at the +-32767 / -32768 entropy-coding clip, abs_sum where the
    clipped and unclipped sums differ, need_rdoq on both sides of its threshold, sign-bit hiding that meets a clipped level, the inverse on levels at the int16
    extremes, round-trip distortions above 2^32, partial tiles and grid-stride launches, odd and 8-aligned plane positions;
  * the bit-depth and shape admission of the TU entries, and which kernels the limit cases launch.
The CPU tests pin the oracle to the reference (oracle/_ref, scalar and AVX2 members) on the same inputs; they are skipped where the reference was not built.
Every GPU case runs with vvb_set_tensor_transform(1) and (0): the raw-byte wgmma engines where they apply, the CUDA-core kernels everywhere.

The dequantiser's input clip (Quant.cpp:606, targetInputBitDepth) is 16 bits throughout the admitted domain: its shift is 6 - transformShift - per >= -9, so
32 + shift - 7 >= 16 (test_dequantiser_input_clip_is_16_bits restates this); it only clips what int16 levels cannot exceed anyway."""
import ctypes
import os
import re
import numpy as np
import pytest
from _libs import oracle, have_ref, refshim, P

I32 = ctypes.c_int32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWO32 = 1 << 32
SIDES = (4, 8, 16, 32, 64)
# every admitted (w, h) with DCT-II, and MTS pairs (DCT-VIII = 1, DST-VII = 2) up to 32, 32 with the 16-wide zero-out included
SHAPES = [(w, h, 0, 0) for w in SIDES for h in SIDES] + [(32, 32, 1, 2), (32, 32, 2, 1), (32, 16, 2, 2), (16, 32, 1, 1), (4, 4, 2, 2), (8, 4, 1, 2),
                                                         (32, 4, 2, 1), (4, 32, 1, 2)]
needs_ref = pytest.mark.skipif(not have_ref(), reason="oracle/_ref (the reference probe) is not built here")


def pel_max(bd):
    return (1 << bd) - 1


def qp_ends(bd):
    o = 6 * (bd - 8)
    return (-o - 1, -o, 0, 63, 64)


# ---------------------------------------------------------------------------------------------------- transform matrices, worst-case inputs
_MATS = {}


def tr_matrix(t, n):
    """forward matrix of type t (0 DCT-II, 1 DCT-VIII, 2 DST-VII) and size n, row k = basis k, from the table the oracle and the library compile"""
    if not _MATS:
        src = open(os.path.join(ROOT, 'oracle', 'vvc_tables.h')).read()
        body = re.search(r'vvc_tr_table_host\[VVC_TR_TABLE_SIZE\] = \{(.*?)\};', src, re.S).group(1)
        _MATS['table'] = np.array([int(v) for v in re.findall(r'-?\d+', body)], dtype=np.int64)
        offs = re.search(r'vvc_tr_offset_host\[3\]\[7\] = \{(.*?)\};', src, re.S).group(1)
        _MATS['off'] = np.array([int(v) for v in re.findall(r'-?\d+', re.sub(r'//[^\n]*', '', offs))]).reshape(3, 7)
    off = int(_MATS['off'][t][n.bit_length() - 1])
    assert off >= 0, (t, n)
    return _MATS['table'][off:off + n * n].reshape(n, n)


def kept(n, t):
    """coefficients kept along a side of n with transform t (TrQuant.cpp:496-497)"""
    return 16 if (t and n == 32) else min(n, 32)


def basis_pattern(w, h, th, tv, k, l, m):
    """m * sign( T_v[k][y] * T_h[l][x] ) (sign 0 -> +): the residual of amplitude m that maximises coefficient (k, l)"""
    s = np.outer(tr_matrix(tv, h)[k], tr_matrix(th, w)[l])
    return np.where(s >= 0, m, -m).astype(np.int16)


def worst_residuals(w, h, th, tv, bd, seed):
    m = pel_max(bd)
    kw, kh = kept(w, th), kept(h, tv)
    out = [np.full((h, w), m, np.int16), np.full((h, w), -m, np.int16)]
    for (k, l) in sorted({(0, 0), (1, 0), (0, 1), (kh - 1, kw - 1), (kh // 2, kw // 3)}):
        out.append(basis_pattern(w, h, th, tv, k, l, m))
        out.append(-out[-1])
    yy, xx = np.mgrid[0:h, 0:w]
    out.append(np.where((yy + xx) & 1, -m, m).astype(np.int16))
    out.append(np.where(xx & 2, -m, m).astype(np.int16))
    rs = np.random.RandomState(seed & 0x7fffffff)
    out += [rs.choice([-m, m], size=(h, w)).astype(np.int16) for _ in range(2)]
    return np.stack(out)


def org_pred_from(resi, bd):
    """org, pred in [0, pelMax] with org - pred = resi for residuals of +-pelMax: full contrast, the reconstruction clips at 0 and at pelMax"""
    m = pel_max(bd)
    org = np.where(resi > 0, m, 0).astype(np.int16)
    return org, (org.astype(np.int32) - resi).astype(np.int16)


# ---------------------------------------------------------------------------------------------------- oracle expectations
def fwd_oracle(w, h, th, tv, bd, qp, irap, dq, resi, sh=0, chroma=0, ts=0, delta=0, lf=(0, 0, 0)):
    """dict(coef, q, abs_sum, last_pos, need_rdoq) of a batch of residuals [n][h][w], TU by TU; lf = (lfnst_idx, set, transpose)"""
    O = oracle()
    n = len(resi)
    r = dict(coef=np.zeros((n, h, w), np.int32), q=np.zeros((n, h, w), np.int16), abs_sum=np.zeros(n, np.int32), last_pos=np.zeros(n, np.int32),
             need_rdoq=np.zeros(n, np.uint8))
    for i in range(n):
        x = np.ascontiguousarray(resi[i], dtype=np.int16); c = r['coef'][i]; q = r['q'][i]; s = I32(); lp = I32()
        if ts:
            rc = O.orc_transform_quant_ts(P(x), w, w, h, bd, qp, irap, sh, delta, P(c), P(q), ctypes.byref(s), ctypes.byref(lp))
        elif lf[0]:
            rc = O.orc_transform_quant_lfnst(P(x), w, w, h, bd, qp, irap, sh, lf[1], lf[0], lf[2], P(c), P(q), ctypes.byref(s), ctypes.byref(lp))
        else:
            rc = O.orc_transform_quant_ex(th, tv, P(x), w, w, h, bd, qp, irap, sh, P(c), P(q), ctypes.byref(s), ctypes.byref(lp))
        assert rc == 0
        r['abs_sum'][i] = s.value; r['last_pos'][i] = lp.value
        r['need_rdoq'][i] = O.orc_need_rdoq_ex(P(c), w, h, bd, qp, dq, ts, delta, chroma)
    return r


def inv_oracle(w, h, th, tv, bd, qp, dq, q):
    """(dequantised coefficients, residual) of a batch of level blocks"""
    O = oracle()
    co = np.zeros(q.shape, np.int32); re_ = np.zeros(q.shape, np.int16)
    for i in range(len(q)):
        x = np.ascontiguousarray(q[i])
        f = O.orc_inv_transform_quant_dq if dq else O.orc_inv_transform_quant
        assert f(th, tv, P(x), w, h, bd, qp, P(co[i]), P(re_[i]), w) == 0
    return co, re_


def rt_oracle(w, h, th, tv, bd, qp, irap, org, pred, sh=0):
    """dict(q, reco, dist_reco, dist_resi, dist_zero, abs_sum, last_pos, need_rdoq) of the fused round trip"""
    O = oracle()
    n = len(org)
    r = dict(q=np.zeros((n, h, w), np.int16), reco=np.zeros((n, h, w), np.int16), dist_reco=np.zeros(n, np.uint64), dist_resi=np.zeros(n, np.uint64),
             dist_zero=np.zeros(n, np.uint64), abs_sum=np.zeros(n, np.int32), last_pos=np.zeros(n, np.int32))
    o4 = np.zeros(4, np.uint64)
    for i in range(n):
        assert O.orc_tu_roundtrip_ex(th, tv, P(np.ascontiguousarray(org[i])), w, P(np.ascontiguousarray(pred[i])), w, w, h, bd, qp, irap, sh,
                                     P(r['q'][i]), P(r['reco'][i]), w, P(o4)) == 0
        r['dist_reco'][i], r['dist_resi'][i], r['dist_zero'][i] = o4[0], o4[1], o4[2]
        r['abs_sum'][i] = np.int32(np.uint32(int(o4[3]) & 0xffffffff)); r['last_pos'][i] = np.int32(np.uint32(int(o4[3]) >> 32))
    f = fwd_oracle(w, h, th, tv, bd, qp, irap, 0, (org.astype(np.int32) - pred).astype(np.int16), sh=sh)
    r['need_rdoq'] = f['need_rdoq']
    return r


FWD_KEYS = ('coef', 'q', 'abs_sum', 'last_pos', 'need_rdoq')


def assert_fwd(got, exp, what, keys=FWD_KEYS):
    for k in keys:
        assert np.array_equal(got[k], exp[k]), (what, k, np.argwhere(got[k] != exp[k])[:4].tolist(), got[k][got[k] != exp[k]][:4], exp[k][got[k] != exp[k]][:4])


def assert_rt(got, exp, what):
    for k in ('q', 'reco', 'need_rdoq'):
        assert np.array_equal(got[k], exp[k]), (what, k, np.argwhere(got[k] != exp[k])[:4].tolist())
    for k in ('dist_reco', 'dist_resi', 'dist_zero', 'abs_sum', 'last_pos'):
        assert np.array_equal(got['res'][k], exp[k]), (what, k, got['res'][k][:6], exp[k][:6])


def both_engines(eng, fn):
    """fn() with the raw-byte wgmma engines on (1) and with the CUDA-core kernels (0)"""
    out = []
    try:
        for t in (1, 0):
            eng.set_tensor_transform(t)
            out.append(fn())
    finally:
        eng.set_tensor_transform(1)
    return out


def need_rdoq_flip(w, h, th, tv, bd, qp, dq, chroma, ts=0, delta=0):
    """the smallest constant residual a with need_rdoq(a) = 1 (then need_rdoq(a - 1) = 0, by bisection on the oracle), None if pelMax stays below"""
    f = lambda a: int(fwd_oracle(w, h, th, tv, bd, qp, 0, dq, np.full((1, h, w), a, np.int16), chroma=chroma, ts=ts, delta=delta)['need_rdoq'][0])
    lo, hi = 0, pel_max(bd)
    if f(lo) or not f(hi):
        return None
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if f(mid): hi = mid
        else: lo = mid
    return hi


_SBH = {}


def sbh_clip_cases():
    """(w, h, bd, qp, residuals): TUs where sign-bit hiding changes a level that QuantCore left at the entropy-coding clip (Quant.cpp:486-489), found on the oracle
    among residuals of +-pelMax whose energy sits in coefficient group 0"""
    if not _SBH:
        O = oracle()
        for (w, h, bd) in ((8, 8, 12), (16, 16, 12), (16, 8, 12), (32, 32, 11)):
            qp = -6 * (bd - 8); m = pel_max(bd)
            Tv, Th = tr_matrix(0, h), tr_matrix(0, w)
            rs = np.random.RandomState(w * 100 + h + bd)
            found = []
            for trial in range(400):
                acc = np.zeros((h, w))
                for _ in range(int(rs.randint(2, 9))):
                    k, l = int(rs.randint(0, 4)), int(rs.randint(0, 4))
                    acc += rs.choice([-1.0, 1.0]) * rs.rand() * np.outer(Tv[k], Th[l])
                resi = np.ascontiguousarray(np.where(acc >= 0, m, -m).astype(np.int16))
                q0 = np.zeros((h, w), np.int16); q1 = np.zeros((h, w), np.int16); c = np.zeros((h, w), np.int32); s = I32(); lp = I32()
                O.orc_transform_quant_ex(0, 0, P(resi), w, w, h, bd, qp, 0, 0, P(c), P(q0), ctypes.byref(s), ctypes.byref(lp))
                O.orc_transform_quant_ex(0, 0, P(resi), w, w, h, bd, qp, 0, 1, P(c), P(q1), ctypes.byref(s), ctypes.byref(lp))
                d = q0 != q1
                if d.any() and ((q0[d] == 32767) | (q0[d] == -32768)).any():
                    found.append(resi)
                if len(found) == 6:
                    break
            _SBH[(w, h, bd)] = (qp, np.stack(found) if found else np.zeros((0, h, w), np.int16))
    return _SBH


# ---------------------------------------------------------------------------------------------------- host rules, restated
def test_dequantiser_input_clip_is_16_bits():
    """Quant::dequant's input clip (targetInputBitDepth = min(16, 32 + rightShift - 7), Quant.cpp:561, 606) over every admitted shape, bit depth and QP:
    rightShift = 6 - (transformShift + per) never drops below -9, so the clip is the int16 range the levels already have (plain and transform-skip QPs)"""
    lo = 99
    for bd in range(8, 13):
        for lw in range(2, 7):
            for lh in range(2, 7):
                for qp in range(-6 * (bd - 8) - 1, 65):
                    base = max(0, min(63 + 6 * (bd - 8), qp + 6 * (bd - 8)))
                    sqrt2 = (lw + lh) & 1
                    tr_shift = 15 - bd - ((lw + lh) >> 1) - sqrt2
                    lo = min(lo, 6 - (tr_shift + base // 6))
                    for delta in (0, 8):
                        if lw <= 5 and lh <= 5:
                            lo = min(lo, 6 - max(base, 4 + 6 * delta) // 6)
    assert lo == -9 and min(16, 32 + lo - 7) == 16


# ---------------------------------------------------------------------------------------------------- the oracle against the reference (CPU)
CPU_SHAPES = [(4, 4, 0, 0), (8, 8, 2, 1), (16, 16, 0, 0), (32, 32, 1, 2), (64, 64, 0, 0), (4, 64, 0, 0), (64, 4, 0, 0), (32, 8, 2, 2), (8, 32, 0, 0)]


@needs_ref
@pytest.mark.parametrize("opt", [0, 1])
def test_oracle_forward_equals_the_reference_at_the_limits(opt):
    """TrQuant::transformNxN + Quant::quant + xNeedRDOQ on the worst-case residuals, 8 / 10 / 12 bits, QP at both sides of the base-QP clip, I and non-I slices:
    coefficients, levels, absSum, lastPos and need_rdoq with dependent quantisation off and on (luma, every transform pair) and for a chroma component (DCT-II).
    The inputs reach the level clip and sums where absSum exceeds the sum of the clipped levels."""
    O = oracle(); R = refshim()
    R.refshim_set_simd(b'AVX2' if opt else b'SCALAR')
    n = 0; clip_hi = clip_lo = wide_sum = 0; nr = set()
    try:
        for (w, h, th, tv) in CPU_SHAPES:
            for bd in (8, 10, 12):
                for i, qp in enumerate(qp_ends(bd)):
                    irap = i & 1
                    for resi in worst_residuals(w, h, th, tv, bd, 7 * w + h + bd)[:: 1 if opt else 2]:
                        resi = np.ascontiguousarray(resi)
                        cR = np.zeros((h, w), np.int32); qR = np.zeros((h, w), np.int16); sR = I32(); lR = I32(); nR = I32()
                        assert R.refshim_transform_quant(th, tv, P(resi), w, w, h, bd, qp, irap, P(cR), P(qR), ctypes.byref(sR), ctypes.byref(lR)) == 0
                        e = fwd_oracle(w, h, th, tv, bd, qp, irap, 0, resi[None])
                        what = (w, h, th, tv, bd, qp, irap)
                        assert np.array_equal(e['coef'][0], cR) and np.array_equal(e['q'][0], qR), (what, np.argwhere(e['q'][0] != qR)[:4].tolist())
                        assert (int(e['abs_sum'][0]), int(e['last_pos'][0])) == (sR.value, lR.value), (what, int(e['abs_sum'][0]), sR.value, int(e['last_pos'][0]), lR.value)
                        for dq in (0, 1):
                            assert O.orc_need_rdoq_ex(P(cR), w, h, bd, qp, dq, 0, 0, 0) == R.refshim_need_rdoq(P(cR), w, h, bd, qp, dq), (what, dq)
                            nr.add(R.refshim_need_rdoq(P(cR), w, h, bd, qp, dq))
                        if th == 0 and tv == 0:
                            for dq in (0, 1):
                                assert R.refshim_transform_quant_ts(P(resi), w, w, h, bd, qp, irap, 0, dq, 0, 0, 1, P(cR), P(qR), ctypes.byref(sR), ctypes.byref(lR),
                                                                    ctypes.byref(nR)) == 0
                                assert np.array_equal(e['q'][0], qR) and O.orc_need_rdoq_ex(P(cR), w, h, bd, qp, dq, 0, 0, 1) == nR.value, (what, 'chroma', dq)
                        clip_hi += int((qR == 32767).any()); clip_lo += int((qR == -32768).any())
                        wide_sum += int(sR.value > int(np.abs(qR.astype(np.int64)).sum()))
                        n += 1
    finally:
        R.refshim_set_simd(b'AVX2')
    assert clip_hi > 20 and clip_lo > 20 and wide_sum > 20 and nr == {0, 1}, (n, clip_hi, clip_lo, wide_sum, nr)


@needs_ref
@pytest.mark.parametrize("opt", [0, 1])
def test_oracle_sign_hiding_transform_skip_and_lfnst_equal_the_reference_at_the_limits(opt):
    """xSignBitHidingHDQ where it meets a level at the clip (the change turns towards zero, Quant.cpp:486); transform skip at 8 / 10 / 12 bits with
    internalMinusInputBitDepth 0 and 8 (luma and chroma, dependent quantisation off and on for need_rdoq); LFNST with both indices, transposed and not, at the QP ends"""
    O = oracle(); R = refshim()
    R.refshim_set_simd(b'AVX2' if opt else b'SCALAR')
    try:
        nsbh = 0
        for (w, h, bd), (qp, cases) in sbh_clip_cases().items():
            for resi in cases:
                resi = np.ascontiguousarray(resi)
                cR = np.zeros((h, w), np.int32); qR = np.zeros((h, w), np.int16); sR = I32(); lR = I32()
                assert R.refshim_transform_quant_sdh(0, 0, P(resi), w, w, h, bd, qp, 0, 1, P(cR), P(qR), ctypes.byref(sR), ctypes.byref(lR)) == 0
                e = fwd_oracle(w, h, 0, 0, bd, qp, 0, 0, resi[None], sh=1)
                assert np.array_equal(e['q'][0], qR) and (int(e['abs_sum'][0]), int(e['last_pos'][0])) == (sR.value, lR.value), (w, h, bd)
                nsbh += 1
        assert nsbh >= 12, nsbh
        nts = 0
        for (w, h) in ((4, 4), (8, 8), (32, 32), (4, 32), (16, 8)):
            for bd in (8, 10, 12):
                for qp in qp_ends(bd):
                    for delta in (0, 8):
                        for k, resi in enumerate(worst_residuals(w, h, 0, 0, bd, bd + qp)[::3]):
                            resi = np.ascontiguousarray(resi); comp = k & 1; dq = (k >> 1) & 1
                            cR = np.zeros((h, w), np.int32); qR = np.zeros((h, w), np.int16); sR = I32(); lR = I32(); nR = I32()
                            assert R.refshim_transform_quant_ts(P(resi), w, w, h, bd, qp, 0, 1, dq, 1, delta, comp, P(cR), P(qR), ctypes.byref(sR), ctypes.byref(lR),
                                                                ctypes.byref(nR)) == 0
                            e = fwd_oracle(w, h, 0, 0, bd, qp, 0, dq, resi[None], sh=1, chroma=comp, ts=1, delta=delta)
                            assert np.array_equal(e['coef'][0], cR) and np.array_equal(e['q'][0], qR), (w, h, bd, qp, delta)
                            assert (int(e['abs_sum'][0]), int(e['last_pos'][0]), int(e['need_rdoq'][0])) == (sR.value, lR.value, nR.value), (w, h, bd, qp, delta, comp, dq)
                            if sR.value:
                                dR = np.zeros((h, w), np.int32); rR = np.zeros((h, w), np.int16); dO = np.zeros((h, w), np.int32); rO = np.zeros((h, w), np.int16)
                                assert R.refshim_inv_transform_quant_ts(P(qR), w, h, bd, qp, delta, P(dR), P(rR), w) == 0
                                assert O.orc_inv_transform_quant_ts(P(qR), w, h, bd, qp, delta, P(dO), P(rO), w) == 0
                                assert np.array_equal(dR, dO) and np.array_equal(rR, rO), (w, h, bd, qp, delta)
                            nts += 1
        sets = set()
        for (w, h) in ((4, 4), (8, 8), (16, 16), (64, 64), (4, 16), (32, 8)):
            for bd in (8, 10, 12):
                for j, qp in enumerate(qp_ends(bd)):
                    for mode, idx in ((0, 1), (18, 2), (34, 1), (50, 2), (66, 1), (2, 2)):
                        resi = np.ascontiguousarray(worst_residuals(w, h, 0, 0, bd, mode)[(mode + j) % 16])
                        cR = np.zeros((h, w), np.int32); qR = np.zeros((h, w), np.int16); sR = I32(); lR = I32(); nR = I32(); st = np.zeros(2, np.int32)
                        assert R.refshim_transform_quant_lfnst(P(resi), w, w, h, bd, qp, j & 1, j >> 2, mode, idx, P(cR), P(qR), ctypes.byref(sR), ctypes.byref(lR),
                                                               ctypes.byref(nR), P(st)) == 0
                        e = fwd_oracle(w, h, 0, 0, bd, qp, j & 1, 0, resi[None], sh=j >> 2, lf=(idx, int(st[0]), int(st[1])))
                        assert np.array_equal(e['coef'][0], cR) and np.array_equal(e['q'][0], qR), (w, h, bd, qp, mode, idx)
                        assert (int(e['abs_sum'][0]), int(e['last_pos'][0]), int(e['need_rdoq'][0])) == (sR.value, lR.value, nR.value), (w, h, bd, qp, mode, idx)
                        sets.add((int(st[0]), int(st[1])))
        assert {t for _, t in sets} == {0, 1}, sets
    finally:
        R.refshim_set_simd(b'AVX2')


def extreme_levels(w, h, seed):
    """level blocks at the int16 extremes: all 32767, all -32768, a checkerboard of both, random {32767, -32768, 0}, and a block with a single extreme DC"""
    rs = np.random.RandomState(seed & 0x7fffffff)
    yy, xx = np.mgrid[0:h, 0:w]
    q = [np.full((h, w), 32767, np.int16), np.full((h, w), -32768, np.int16), np.where((yy + xx) & 1, -32768, 32767).astype(np.int16),
         rs.choice([32767, -32768, 0], size=(h, w)).astype(np.int16), np.zeros((h, w), np.int16)]
    q[-1][0, 0] = -32768
    return np.stack(q)


def last_scan_pos(q, w, h):
    """scan position of the last non-zero level (-1: none), what tu.lastPos carries into DepQuant::dequant"""
    so = np.zeros(1024, np.int32); n = oracle().orc_scan_order(w, h, P(so))
    nz = np.flatnonzero(q.ravel()[so[:n]])
    return int(nz[-1]) if len(nz) else -1


@needs_ref
@pytest.mark.parametrize("opt", [0, 1])
def test_oracle_inverse_and_round_trip_equal_the_reference_at_the_limits(opt):
    """Quant::dequant (and DepQuant::dequant) + TrQuant::invTransformNxN on levels at the int16 extremes, and the whole round trip on full-contrast org / pred,
    8 / 10 / 12 bits at the QP ends: dequantised coefficients, residuals, levels, reconstructions and the three distortions (above 2^32 at 64 x 64, 12 bits)"""
    O = oracle(); R = refshim()
    R.refshim_set_simd(b'AVX2' if opt else b'SCALAR')
    big = 0
    try:
        for (w, h, th, tv) in CPU_SHAPES:
            for bd in (8, 10, 12):
                for qp in qp_ends(bd):
                    for dq in (0, 1):
                        for q in extreme_levels(w, h, w + h + qp)[:: 1 if opt else 2]:
                            q = np.ascontiguousarray(q)
                            cR = np.zeros((h, w), np.int32); rR = np.zeros((h, w), np.int16)
                            if dq:
                                assert R.refshim_inv_transform_quant_dq(th, tv, P(q), last_scan_pos(q, w, h), w, h, bd, qp, P(cR), P(rR), w) == 0
                            else:
                                assert R.refshim_inv_transform_quant(th, tv, P(q), w, h, bd, qp, P(cR), P(rR), w) == 0
                            cO, rO = inv_oracle(w, h, th, tv, bd, qp, dq, q[None])
                            assert np.array_equal(cO[0], cR) and np.array_equal(rO[0], rR), (w, h, th, tv, bd, qp, dq)
                    resi = worst_residuals(w, h, th, tv, bd, qp + 50)[:: 2 if opt else 4]
                    org, pred = org_pred_from(resi, bd)
                    e = rt_oracle(w, h, th, tv, bd, qp, 0, org, pred)
                    for i in range(len(org)):
                        qR = np.zeros((h, w), np.int16); rc = np.zeros((h, w), np.int16); o4 = np.zeros(4, np.uint64)
                        assert R.refshim_tu_roundtrip(opt, th, tv, P(np.ascontiguousarray(org[i])), w, P(np.ascontiguousarray(pred[i])), w, w, h, bd, qp, 0,
                                                      P(qR), P(rc), w, P(o4)) == 0
                        assert np.array_equal(qR, e['q'][i]) and np.array_equal(rc, e['reco'][i]), (w, h, th, tv, bd, qp, i)
                        assert [int(v) for v in o4[:3]] == [int(e['dist_reco'][i]), int(e['dist_resi'][i]), int(e['dist_zero'][i])], (w, h, bd, qp, i, o4)
                        big += int(o4[2]) >= TWO32
    finally:
        R.refshim_set_simd(b'AVX2')
    assert big > 0


# ---------------------------------------------------------------------------------------------------- GPU cases
@pytest.fixture(scope="module")
def eng():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


@pytest.mark.gpu
def test_forward_worst_cases_every_shape(eng):
    """every admitted shape, 8 / 10 / 11 / 12 bits, the QP ends, worst-case residuals: coef, levels, abs_sum, last_pos, need_rdoq (dependent quantisation off / on,
    luma / chroma) equal the oracle with both engines.  The levels reach +32767 and -32768, abs_sum exceeds the sum of the clipped levels, need_rdoq takes both values."""
    seen = dict(hi=0, lo=0, wide=0, nr0=0, nr1=0); top = 0
    for (w, h, th, tv) in SHAPES:
        for bd in (8, 10, 11, 12):
            for i, qp in enumerate(qp_ends(bd)):
                irap, dq, chroma = i & 1, (i >> 1) & 1, int(i in (2, 4))
                resi = worst_residuals(w, h, th, tv, bd, w * 3 + h + bd + i)
                exp = fwd_oracle(w, h, th, tv, bd, qp, irap, dq, resi, chroma=chroma)
                par = eng.tu_par(w, h, th, tv, bd, qp, bool(irap), bool(dq), is_chroma=bool(chroma))
                for t, got in zip((1, 0), both_engines(eng, lambda: eng.fwd_trquant(par, resi))):
                    assert_fwd(got, exp, (w, h, th, tv, bd, qp, t))
                seen['hi'] += int((exp['q'] == 32767).sum()); seen['lo'] += int((exp['q'] == -32768).sum())
                seen['wide'] += int((exp['abs_sum'] > np.abs(exp['q'].astype(np.int64)).sum(axis=(1, 2))).sum())
                seen['nr0'] += int((exp['need_rdoq'] == 0).sum()); seen['nr1'] += int((exp['need_rdoq'] == 1).sum())
                top = max(top, int(exp['abs_sum'].max()))
    assert all(v > 0 for v in seen.values()) and top < 1 << 24, (seen, top)      # the header's bound on abs_sum for in-range residuals


@pytest.mark.gpu
def test_need_rdoq_on_both_sides_of_its_threshold(eng):
    """constant residuals a - 1 and a where the oracle's need_rdoq turns from 0 to 1 (found by bisection): the device's integer threshold (rdoqThr) gives the same
    answer for plain and dependent quantisation (QP + 1), luma (171) and chroma (256) rounding, transforms and transform skip"""
    found = 0
    for (w, h, th, tv, ts) in ((4, 4, 0, 0, 0), (8, 8, 0, 0, 0), (16, 16, 2, 1, 0), (32, 32, 0, 0, 0), (64, 64, 0, 0, 0), (4, 64, 0, 0, 0), (8, 8, 0, 0, 1), (32, 4, 0, 0, 1)):
        for bd in (8, 10, 12):
            for qp in (qp_ends(bd)[1], 22, 40, 51, 63):
                for dq in (0, 1):
                    for chroma in (0, 1):
                        a = need_rdoq_flip(w, h, th, tv, bd, qp, dq, chroma, ts=ts)
                        if a is None:
                            continue
                        resi = np.stack([np.full((h, w), a - 1, np.int16), np.full((h, w), a, np.int16), np.full((h, w), -a, np.int16)])
                        par = eng.tu_par(w, h, th, tv, bd, qp, False, bool(dq), transform_skip=bool(ts), is_chroma=bool(chroma))
                        for t, got in zip((1, 0), both_engines(eng, lambda: eng.fwd_trquant(par, resi))):
                            assert got['need_rdoq'].tolist() == [0, 1, 1], (w, h, th, tv, ts, bd, qp, dq, chroma, a, t)
                        found += 1
    assert found > 150, found


@pytest.mark.gpu
def test_sign_hiding_meets_a_clipped_level(eng):
    """sign-bit hiding where the position chosen in a group holds a level at the clip: forward call and fused round trip against the oracle, both engine settings"""
    n = 0
    for (w, h, bd), (qp, resi) in sbh_clip_cases().items():
        assert len(resi) >= 2, (w, h, bd)
        exp = fwd_oracle(w, h, 0, 0, bd, qp, 0, 0, resi, sh=1)
        par = eng.tu_par(w, h, 0, 0, bd, qp, False, False, True)
        for t, got in zip((1, 0), both_engines(eng, lambda: eng.fwd_trquant(par, resi))):
            assert_fwd(got, exp, (w, h, bd, qp, t))
        org, pred = org_pred_from(resi, bd)
        e = rt_oracle(w, h, 0, 0, bd, qp, 0, org, pred, sh=1)
        for t, got in zip((1, 0), both_engines(eng, lambda: eng.tu_roundtrip(par, org, pred))):
            assert_rt(got, e, (w, h, bd, qp, t))
        n += len(resi)
    assert n >= 12


@pytest.mark.gpu
def test_inverse_on_extreme_levels(eng):
    """levels at +32767 / -32768 at the QP ends, plain and DepQuant dequantiser: the dequantised coefficients reach the 16-bit transform clip and the first inverse
    stage's 16-bit clip engages (checked in int64 from the matrices); residuals equal the oracle with both engines"""
    stage1_clipped = dq_clipped = 0
    for (w, h, th, tv) in SHAPES[::2] + SHAPES[25:]:
        for bd in (8, 10, 12):
            for qp in (qp_ends(bd)[0], 0, 63):
                for dq in (0, 1):
                    q = extreme_levels(w, h, w * h + qp + dq)
                    co, exp = inv_oracle(w, h, th, tv, bd, qp, dq, q)
                    par = eng.tu_par(w, h, th, tv, bd, qp, False, bool(dq))
                    for t, got in zip((1, 0), both_engines(eng, lambda: eng.inv_trquant(par, q))):
                        assert np.array_equal(got, exp), (w, h, th, tv, bd, qp, dq, t, np.argwhere(got != exp)[:4].tolist())
                    dq_clipped += int((co == 32767).any() or (co == -32768).any())
                    kh, kw = kept(h, tv), kept(w, th)
                    s1 = np.einsum('ky,nkx->nyx', tr_matrix(tv, h)[:kh], co[:, :kh, :kw].astype(np.int64))        # xIT: the vertical pass first
                    stage1_clipped += int((np.abs((s1 + 64) >> 7) > 32767).any())
    assert dq_clipped > 50 and stage1_clipped > 50, (dq_clipped, stage1_clipped)


@pytest.mark.gpu
def test_round_trip_full_contrast_every_shape(eng):
    """org / pred at 0 and pelMax (both ways round, basis patterns, checkerboards), every shape, 8 / 10 / 11 / 12 bits, QP ends: levels, reconstructions (clipped at 0
    and at pelMax), the three 64-bit distortions, abs_sum, last_pos and need_rdoq equal the oracle with both engines; at 64 x 64 and 12 bits dist_zero is
    4096 * 4095^2 > 2^32"""
    big = clip0 = clipm = 0
    for (w, h, th, tv) in SHAPES:
        for bd in (8, 10, 11, 12):
            for i, qp in enumerate(qp_ends(bd)):
                org, pred = org_pred_from(worst_residuals(w, h, th, tv, bd, w + 5 * h + i), bd)
                exp = rt_oracle(w, h, th, tv, bd, qp, i & 1, org, pred)
                par = eng.tu_par(w, h, th, tv, bd, qp, bool(i & 1))
                for t, got in zip((1, 0), both_engines(eng, lambda: eng.tu_roundtrip(par, org, pred))):
                    assert_rt(got, exp, (w, h, th, tv, bd, qp, t))
                big += int((exp['dist_zero'] >= TWO32).sum()) + int((exp['dist_reco'] >= TWO32).sum())
                clip0 += int((exp['reco'] == 0).any()); clipm += int((exp['reco'] == pel_max(bd)).any())
                if (w, h, bd) == (64, 64, 12):
                    assert int(exp['dist_zero'][0]) == 4096 * 4095 ** 2 > TWO32
    assert big > 0 and clip0 > 0 and clipm > 0, (big, clip0, clipm)


def _tiled(base, n):
    return np.ascontiguousarray(np.resize(base, (n,) + base.shape[1:]))


@pytest.mark.gpu
def test_partial_tiles_and_grid_stride(eng):
    """TU counts that leave a partial tile / team (1, 3, 37) and counts above what one wave of CTAs holds on this device (the kernels then stride over the list):
    forward, inverse and round trip against the oracle's results of the distinct TUs, both engines"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for (w, h, th, tv, bd, qp) in ((4, 4, 0, 0, 12, -24), (8, 8, 2, 1, 10, 0), (16, 16, 0, 0, 12, 63), (32, 32, 0, 0, 11, -18), (64, 64, 0, 0, 12, -25), (64, 4, 0, 0, 8, 3)):
        t_core = min(128, max(4, w * h // 4))
        one_wave = max(sms * 16 * (128 // t_core), sms * 8 * (128 // min(w, 32)))      # CUDA-core teams, raw-byte tiles
        base_r = worst_residuals(w, h, th, tv, bd, w + h)
        ef = fwd_oracle(w, h, th, tv, bd, qp, 1, 1, base_r)
        base_q = np.concatenate([extreme_levels(w, h, 3), ef['q']])
        _, ei = inv_oracle(w, h, th, tv, bd, qp, 0, base_q)
        org, pred = org_pred_from(base_r, bd)
        er = rt_oracle(w, h, th, tv, bd, qp, 1, org, pred)
        par = eng.tu_par(w, h, th, tv, bd, qp, True, True)
        for n in (1, 3, 37, one_wave + 37):
            r = _tiled(base_r, n)
            for t, got in zip((1, 0), both_engines(eng, lambda: eng.fwd_trquant(par, r))):
                assert_fwd(got, {k: _tiled(v, n) for k, v in ef.items()}, (w, h, n, t))
            qq = _tiled(base_q, n)
            par_i = eng.tu_par(w, h, th, tv, bd, qp, True, False)
            for t, got in zip((1, 0), both_engines(eng, lambda: eng.inv_trquant(par_i, qq))):
                assert np.array_equal(got, _tiled(ei, n)), (w, h, n, t)
            o, p = _tiled(org, n), _tiled(pred, n)
            for t, got in zip((1, 0), both_engines(eng, lambda: eng.tu_roundtrip(par_i, o, p))):
                assert_rt(got, {k: _tiled(v, n) for k, v in er.items()}, (w, h, n, t))


def _planes(bd, W, H, m, seed):
    """org and pred planes of full contrast: random blocks of 0 / pelMax, pred the complement of org with a few flipped pels"""
    rs = np.random.RandomState(seed)
    mx = pel_max(bd)
    org = (rs.randint(0, 2, size=(H + 2 * m, W + 2 * m)) * mx).astype(np.int16)
    org[: (H + 2 * m) // 2, : (W + 2 * m) // 2] = mx                                   # a quarter of flat pelMax: the constant residual of maximum DC
    pred = (mx - org).astype(np.int16)
    pred[rs.rand(*pred.shape) < 0.05] = 0
    return np.ascontiguousarray(org), np.ascontiguousarray(pred)


@pytest.mark.gpu
def test_plane_forms_at_odd_and_aligned_positions(eng):
    """vvb_fwd_trquant_planes and vvb_tu_roundtrip_planes(_dev) on full-contrast 12- and 10-bit planes (org = pelMax / pred = 0 and the other way round), TUs at odd
    and at 8-pel-aligned positions with odd and even prediction displacements: against the oracle on the pels the blocks address, both engines"""
    import vvenc_b200 as V
    W, H, m = 192, 128, 16
    for bd in (12, 10):
        org, pred = _planes(bd, W, H, m, bd)
        eng.upload_plane(0, org, W, H, m, bd); eng.upload_plane(1, pred, W, H, m, bd)
        rs = np.random.RandomState(bd)
        for (w, h, th, tv) in ((64, 64, 0, 0), (8, 8, 0, 0), (32, 32, 1, 2), (4, 64, 0, 0), (64, 4, 0, 0), (16, 8, 2, 2), (4, 4, 0, 0)):
            n = 41
            B = np.zeros(n, dtype=V.BLOCK_DT)
            B['x'] = rs.randint(0, W - w + 1, n); B['y'] = rs.randint(0, H - h + 1, n)
            B['x'][: n // 2] &= ~7; B['x'][n // 2:] |= 1; B['x'] = np.minimum(B['x'], W - w)
            B['x'][0] = B['y'][0] = 0
            B['start_x'] = rs.randint(-m, m + 1, n); B['start_y'] = rs.randint(-m, m + 1, n); B['start_x'][0] = B['start_y'][0] = 0
            o = np.stack([org[m + b['y']:m + b['y'] + h, m + b['x']:m + b['x'] + w] for b in B])
            p = np.stack([pred[m + b['y'] + b['start_y']:m + b['y'] + b['start_y'] + h, m + b['x'] + b['start_x']:m + b['x'] + b['start_x'] + w] for b in B])
            assert (B['x'] & 1).any() and not (B['x'][: n // 2] & 7).any()
            for qp in (qp_ends(bd)[0], 63):
                par = eng.tu_par(w, h, th, tv, bd, qp, False, False)
                ef = fwd_oracle(w, h, th, tv, bd, qp, 0, 0, (o.astype(np.int32) - p).astype(np.int16))
                for t, got in zip((1, 0), both_engines(eng, lambda: eng.fwd_trquant_planes(par, 0, 1, B, want_coef=True))):
                    assert_fwd(got, ef, (bd, w, h, th, tv, qp, t))
                er = rt_oracle(w, h, th, tv, bd, qp, 0, o, p)
                for t, got in zip((1, 0), both_engines(eng, lambda: eng.tu_roundtrip_planes(par, 0, 1, B))):
                    assert_rt(got, er, (bd, w, h, th, tv, qp, t))
                if (w, h, bd) == (64, 64, 12):
                    assert int(er['dist_zero'][0]) == 4096 * 4095 ** 2 and (er['q'] == 32767).any() == (qp < 0)


@pytest.mark.gpu
def test_search_refine_tu_at_12_bits(eng):
    """vvb_search_refine_tu on 12-bit full-contrast planes with a TU stage at the lowest QP: the levels, abs_sum, last_pos and need_rdoq of the chain equal the
    separate calls (search, then vvb_fwd_trquant_planes at the best vectors) and the oracle on the residuals of those vectors"""
    import vvenc_b200 as V
    import vvenc_b200._lib as VL
    W, H, m, bd = 128, 64, 32, 12
    org, pred = _planes(bd, W, H, m, 99)
    eng.upload_plane(8, org, W, H, m, bd); eng.upload_plane(9, pred, W, H, m, bd)
    lists = V.candidates.pyramid_lists(8, 2, W, H)
    blks = []
    for xs, ys in lists:
        bl = np.zeros(len(xs), dtype=V.BLOCK_DT)
        bl['x'] = xs; bl['y'] = ys; bl['left'] = -4; bl['right'] = 4; bl['top'] = -4; bl['bottom'] = 4
        blks.append(bl)
    me = eng.me_par(10.0, 2, 0, 0)
    qp = qp_ends(bd)[0]
    best = eng.sad_search_pyramid(8, 9, blks, 8, me, 9, 9)
    io = (VL.vvb_level_io * 2)(); keep = []
    for l, bl in enumerate(blks):
        n = 8 << l; cnt = len(bl)
        o = dict(best=np.zeros(cnt, dtype=V.BEST_DT), q=np.zeros((cnt, n, n), dtype=np.int16), s=np.zeros(cnt, dtype=np.int32), lp=np.zeros(cnt, dtype=np.int32),
                 nr=np.zeros(cnt, dtype=np.uint8), blk=np.ascontiguousarray(bl))
        keep.append(o)
        io[l].blocks = o['blk'].ctypes.data; io[l].count = cnt; io[l].best = o['best'].ctypes.data
        io[l].q = o['q'].ctypes.data; io[l].abs_sum = o['s'].ctypes.data; io[l].last_pos = o['lp'].ctypes.data; io[l].need_rdoq = o['nr'].ctypes.data
        io[l].tu = eng.tu_par(n, n, V.DCT2, V.DCT2, bd, qp + l, bool(l), bool(l))
    rc = eng.lib.vvb_search_refine_tu(eng.h, 8, 9, 2, io, 8, ctypes.byref(me), 9, 9, V.DF_SAD, None, 0)
    assert rc == 0, eng.lib.vvb_last_error(eng.h)
    clipped = 0
    for l, bl in enumerate(blks):
        n = 8 << l; o = keep[l]
        assert np.array_equal(o['best'], best[l]), l
        b2 = bl.copy(); b2['start_x'] = best[l]['dx']; b2['start_y'] = best[l]['dy']
        r = eng.fwd_trquant_planes(io[l].tu, 8, 9, b2)
        assert np.array_equal(o['q'], r['q']) and np.array_equal(o['s'], r['abs_sum']) and np.array_equal(o['lp'], r['last_pos']) and np.array_equal(o['nr'], r['need_rdoq']), l
        ov = np.stack([org[m + b['y']:m + b['y'] + n, m + b['x']:m + b['x'] + n] for b in b2])
        pv = np.stack([pred[m + b['y'] + b['start_y']:m + b['y'] + b['start_y'] + n, m + b['x'] + b['start_x']:m + b['x'] + b['start_x'] + n] for b in b2])
        e = fwd_oracle(n, n, 0, 0, bd, qp + l, l, l, (ov.astype(np.int32) - pv).astype(np.int16))
        assert_fwd(dict(q=o['q'], abs_sum=o['s'], last_pos=o['lp'], need_rdoq=o['nr']), e, ('chain', l), keys=FWD_KEYS[1:])
        clipped += int((np.abs(o['q'].astype(np.int32)) >= 32767).sum())
    assert clipped > 0


# ---------------------------------------------------------------------------------------------------- _dev buffers 8- but not 16-byte aligned
DEV_ENTRIES = ('fwd', 'fwd_planes', 'inv', 'rt')


def dev_case(eng, w, entry, off):
    """(call, expected) of one _dev entry on square w x w TUs at 10 bits and the lowest QP, with every pool and output `off` bytes into its own torch allocation
    (the block list stays at the start of its own).  call() returns the outputs as numpy arrays; the plane form reads org / pred from planes 30 / 31."""
    import torch
    import vvenc_b200 as V
    import vvenc_b200._lib as L
    bd = 10; qp = qp_ends(bd)[0]
    par = eng.tu_par(w, w, 0, 0, bd, qp, True, False)
    resi = worst_residuals(w, w, 0, 0, bd, w)
    n = len(resi)
    keep, outs = [], {}

    def dev_in(a):
        raw = torch.from_numpy(np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8).copy())
        t = torch.zeros(raw.numel() + 16, dtype=torch.uint8, device='cuda')
        t[off:off + raw.numel()] = raw.cuda()
        keep.append(t)
        return ctypes.c_void_p(t.data_ptr() + off)

    def dev_out(name, dt, shape):
        nb = int(np.prod(shape)) * np.dtype(dt).itemsize
        t = torch.zeros(nb + 16, dtype=torch.uint8, device='cuda')
        outs[name] = (t, dt, shape, nb)
        return ctypes.c_void_p(t.data_ptr() + off)

    def fwd_outs():
        return (dev_out('coef', np.int32, (n, w, w)), dev_out('q', np.int16, (n, w, w)), dev_out('abs_sum', np.int32, (n,)), dev_out('last_pos', np.int32, (n,)),
                dev_out('need_rdoq', np.uint8, (n,)))

    lib, h, pp = eng.lib, eng.h, ctypes.byref(par)
    if entry == 'fwd':
        args = (pp, dev_in(resi), n) + fwd_outs()
        fn, exp = lib.vvb_fwd_trquant_dev, fwd_oracle(w, w, 0, 0, bd, qp, 1, 0, resi)
    elif entry == 'fwd_planes':
        W, H, m = 192, 128, 16
        org, pred = _planes(bd, W, H, m, w)
        eng.upload_plane(30, org, W, H, m, bd); eng.upload_plane(31, pred, W, H, m, bd)
        rs = np.random.RandomState(w)
        B = np.zeros(n, dtype=V.BLOCK_DT)
        B['x'] = rs.randint(0, W - w + 1, n); B['y'] = rs.randint(0, H - w + 1, n); B['start_x'] = rs.randint(-m, m + 1, n); B['start_y'] = rs.randint(-m, m + 1, n)
        o = np.stack([org[m + b['y']:m + b['y'] + w, m + b['x']:m + b['x'] + w] for b in B])
        p = np.stack([pred[m + b['y'] + b['start_y']:m + b['y'] + b['start_y'] + w, m + b['x'] + b['start_x']:m + b['x'] + b['start_x'] + w] for b in B])
        d_blk = torch.from_numpy(np.frombuffer(B.tobytes(), np.uint8).copy()).cuda()
        keep.append(d_blk)
        args = (pp, 30, 31, ctypes.c_void_p(d_blk.data_ptr()), n) + fwd_outs()
        fn, exp = lib.vvb_fwd_trquant_planes_dev, fwd_oracle(w, w, 0, 0, bd, qp, 1, 0, (o.astype(np.int32) - p).astype(np.int16))
    elif entry == 'inv':
        q = extreme_levels(w, w, w)
        args = (pp, dev_in(q), len(q), dev_out('resi', np.int16, (len(q), w, w)))
        fn, exp = lib.vvb_inv_trquant_dev, dict(resi=inv_oracle(w, w, 0, 0, bd, qp, 0, q)[1])
    else:
        org, pred = org_pred_from(resi, bd)
        args = (pp, dev_in(org), dev_in(pred), n, dev_out('q', np.int16, (n, w, w)), dev_out('reco', np.int16, (n, w, w)), dev_out('res', L.TU_RESULT_DT, (n,)),
                dev_out('need_rdoq', np.uint8, (n,)))
        fn, exp = lib.vvb_tu_roundtrip_dev, rt_oracle(w, w, 0, 0, bd, qp, 1, org, pred)
    torch.cuda.synchronize()

    def call():
        assert fn(h, *args) == 0, lib.vvb_last_error(h)
        torch.cuda.synchronize()
        return {k: np.frombuffer(t[off:off + nb].cpu().numpy().tobytes(), dt).reshape(shape) for k, (t, dt, shape, nb) in outs.items()}
    return call, exp


@pytest.mark.gpu
def test_dev_buffers_8_byte_aligned(eng):
    """_dev calls on square 8 / 16 / 32 / 64 TUs with the tensor engines switched on, every pool and output 8 bytes into its torch allocation (8- but not 16-byte
    aligned): forward from a pool and from planes, inverse and round trip equal the same calls on 16-byte aligned buffers and the oracle.  The misaligned calls
    run on the CUDA-core kernels, the aligned ones on the raw-byte engines (test_kernel_selection)."""
    eng.set_tensor_transform(1)
    for w in (8, 16, 32, 64):
        for entry in DEV_ENTRIES:
            got = {}
            for off in (8, 0):
                call, exp = dev_case(eng, w, entry, off)
                got[off] = g = call()
                what = (w, entry, off)
                if entry == 'inv':
                    assert np.array_equal(g['resi'], exp['resi']), what
                elif entry == 'rt':
                    assert_rt(g, exp, what)
                else:
                    assert_fwd(g, exp, what)
            assert got[8].keys() == got[0].keys()
            for k in got[0]:
                assert np.array_equal(got[8][k], got[0][k]), (w, entry, k)


# ---------------------------------------------------------------------------------------------------- admission
@pytest.mark.gpu
def test_admission(eng):
    """bit depths 8..12 and the documented shapes are admitted; 7 and 13 bits, sides outside 4..64 or not powers of two, DST-VII / DCT-VIII above 32, transform skip
    above 32, LFNST with a transform other than DCT-II or on a skipped transform return VVB_ERR_UNSUPPORTED; unknown transform types, LFNST indices / sets and
    input bit-depth deltas return VVB_ERR_ARG -- from every TU entry"""
    import vvenc_b200._lib as L
    import vvenc_b200 as V
    org = np.zeros((64 + 2 * 8, 64 + 2 * 8), np.int16)
    eng.upload_plane(20, org, 64, 64, 8, 10)
    blk = np.zeros(1, dtype=V.BLOCK_DT)

    def calls(par):
        w, h = max(4, min(par.w, 64)), max(4, min(par.h, 64))
        a = np.zeros((1, h, w), np.int16); q = np.zeros((1, 128, 128), np.int16); c = np.zeros((1, 128, 128), np.int32)
        s = np.zeros(1, np.int32); lp = np.zeros(1, np.int32); nr = np.zeros(1, np.uint8); res = np.zeros(1, dtype=L.TU_RESULT_DT)
        lib, hh, pp = eng.lib, eng.h, ctypes.byref(par)
        return dict(fwd=lib.vvb_fwd_trquant(hh, pp, P(a), 1, P(c), P(q), P(s), P(lp), P(nr)),
                    fwd_planes=lib.vvb_fwd_trquant_planes(hh, pp, 20, 20, P(blk), 1, P(c), P(q), P(s), P(lp), P(nr)),
                    inv=lib.vvb_inv_trquant(hh, pp, P(q), 1, P(q)),
                    rt=lib.vvb_tu_roundtrip(hh, pp, P(a), P(a), 1, P(q), P(q), P(res), P(nr)))

    T = eng.tu_par
    for bd in (8, 9, 10, 11, 12):
        assert set(calls(T(16, 8, 2, 1, bd, 30)).values()) == {L.VVB_OK}, bd
    unsupported = [T(16, 16, 0, 0, 7, 30), T(16, 16, 0, 0, 13, 30), T(4, 4, 0, 0, 0, 30), T(2, 8, 0, 0, 10, 30), T(128, 8, 0, 0, 10, 30), T(8, 128, 0, 0, 10, 30),
                   T(12, 8, 0, 0, 10, 30), T(8, 6, 0, 0, 10, 30), T(64, 8, 2, 0, 10, 30), T(8, 64, 0, 1, 10, 30), T(64, 32, 0, 0, 10, 30, transform_skip=True),
                   T(8, 8, 1, 0, 10, 30, lfnst_idx=1), T(8, 8, 0, 0, 10, 30, lfnst_idx=1, transform_skip=True)]
    for par in unsupported:
        rc = calls(par)
        assert set(rc.values()) == {L.VVB_ERR_UNSUPPORTED}, (par.w, par.h, par.tr_hor, par.tr_ver, par.bit_depth, par.transform_skip, par.lfnst_idx, rc)
    bad = [T(8, 8, 3, 0, 10, 30), T(8, 8, 0, -1, 10, 30), T(8, 8, 0, 0, 10, 30, lfnst_idx=3), T(8, 8, 0, 0, 10, 30, lfnst_idx=1, lfnst_set=4),
           T(8, 8, 0, 0, 10, 30, transform_skip=True, input_bit_depth_delta=9), T(8, 8, 0, 0, 10, 30, transform_skip=True, input_bit_depth_delta=-1)]
    for par in bad:
        rc = calls(par)
        assert set(rc.values()) == {L.VVB_ERR_ARG}, (par.tr_hor, par.tr_ver, par.lfnst_idx, par.lfnst_set, par.input_bit_depth_delta, rc)
    eng.free_plane(20)


# ---------------------------------------------------------------------------------------------------- which kernels run
def kernel_selection_cases():
    """[(label, setup)] for tests/_kernel_selection_run.py: the square 8..64 limit cases run the raw-byte engines (fwd_trquant_tc2_kernel, inv_trquant_tc_kernel)
    with vvb_set_tensor_transform on and the CUDA-core kernels with it off; 4 x 4, rectangular TUs and sign-bit hiding run the CUDA-core kernels either way; with
    the tensor engines on, the _dev calls of test_dev_buffers_8_byte_aligned run the raw-byte engines on 16-byte aligned buffers and the CUDA-core kernels on
    buffers 8 bytes off"""
    from test_gpu_format_limits import ran
    cases = []
    for (w, h, sh) in ((8, 8, 0), (16, 16, 0), (32, 32, 0), (64, 64, 0), (4, 4, 0), (64, 4, 0), (16, 16, 1)):
        for tensor in (1, 0):
            tc = tensor and w == h and w >= 8 and not sh
            for entry in ('fwd', 'inv', 'rt'):
                if entry == 'inv' and sh:
                    continue

                def setup(eng, w=w, h=h, sh=sh, tensor=tensor, tc=tc, entry=entry):
                    bd = 12; qp = qp_ends(bd)[0]
                    eng.set_tensor_transform(tensor)
                    par = eng.tu_par(w, h, 0, 0, bd, qp, False, False, bool(sh))
                    resi = worst_residuals(w, h, 0, 0, bd, 1)
                    org, pred = org_pred_from(resi, bd)
                    q = extreme_levels(w, h, 1)
                    call = {'fwd': lambda: eng.fwd_trquant(par, resi), 'inv': lambda: eng.inv_trquant(par, q), 'rt': lambda: eng.tu_roundtrip(par, org, pred)}[entry]
                    fwd_k, inv_k = ('fwd_trquant_tc2_kernel', 'inv_trquant_tc_kernel') if tc else ('fwd_trquant_kernel', 'inv_trquant_kernel')
                    want = {'fwd': [fwd_k], 'inv': [inv_k], 'rt': [fwd_k, inv_k] if tc else ['tu_roundtrip_kernel']}[entry]
                    other = {'fwd_trquant_tc2_kernel', 'inv_trquant_tc_kernel'} if not tc else set()
                    return call, (lambda names: all(ran(names, k) for k in want) and not any(ran(names, k) for k in other))
                cases.append(('%dx%d sh=%d tensor=%d %s: %s' % (w, h, sh, tensor, entry, 'raw-byte engines' if tc else 'CUDA-core kernels'), setup))
    for w in (8, 16, 32, 64):
        for entry in DEV_ENTRIES:
            for off in (0, 8):
                tc = off == 0

                def setup(eng, w=w, entry=entry, off=off, tc=tc):
                    eng.set_tensor_transform(1)
                    call, _ = dev_case(eng, w, entry, off)
                    fwd_k, inv_k = ('fwd_trquant_tc2_kernel', 'inv_trquant_tc_kernel') if tc else ('fwd_trquant_kernel', 'inv_trquant_kernel')
                    want = {'fwd': [fwd_k], 'fwd_planes': [fwd_k], 'inv': [inv_k], 'rt': [fwd_k, inv_k] if tc else ['tu_roundtrip_kernel']}[entry]
                    other = {'fwd_trquant_tc2_kernel', 'inv_trquant_tc_kernel'} if not tc else set()
                    return call, (lambda names: all(ran(names, k) for k in want) and not any(ran(names, k) for k in other))
                cases.append(('%dx%d _dev %s buffers +%d bytes: %s' % (w, w, entry, off, 'raw-byte engines' if tc else 'CUDA-core kernels'), setup))
    return cases


@pytest.mark.gpu
def test_kernel_selection():
    import json, subprocess, sys
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_kernel_selection_run.py')
    out = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [script, 'test_gpu_tu_limits'], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]
    assert [r['case'] for r in rows] == [label for label, _ in kernel_selection_cases()]
    assert [r for r in rows if not r['ok']] == [], rows
