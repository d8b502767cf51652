"""vvb_frac_search, InterSearch::xPatternSearchFracDIF with its selection on the device, against the reference (all but the coverage check need -m gpu).

  * the member (refshim_frac_search_member: xPatternSearchFracDIF called on the unmodified reference objects): dfunc x reduce_tap x alt_hpel x fast_sub_pel,
    fourteen PU shapes up to 128x128, bit depths 8, 10 and 12, integer vectors spread over the picture and beyond every edge within the margin.
  * coverage: the content (smooth, shifted by known quarter-pel vectors, plus noise) makes the member take every half-pel direction and every quarter-pel
    offset with fast_sub_pel 0 and 1, and end after the half-pel round (pattern 0) in fast mode.
  * chain: vvb_tz_search_dev -> vvb_frac_search_dev on device arrays for every PU of 8x8..128x128 on a 1920x1080 10-bit pair whose reference margin is the
    one the header states, against the TZ member followed by the fractional member.
  * the grid path: vvb_frac_cost_grid plus candidates.subpel_refinement(_fast) for the shapes it serves.
  * admission: every error code, the read box at the margin on each side, one pel beyond it (refused by the host call, the sentinel from _dev), n == 0.
  * format limits: 128x128 at 12 bits with the Hadamard sum and the MV rate near their tops.
"""
import ctypes
import itertools

import numpy as np
import pytest

from _libs import have_ref, refshim, oracle, P, PO

pytestmark = pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
gpu = pytest.mark.gpu

LAM = 57.25
SHAPES = [(8, 8), (16, 16), (32, 32), (64, 64), (128, 128), (128, 64), (64, 128), (16, 8), (8, 16), (32, 8), (8, 32), (64, 16), (4, 8), (8, 4)]
SETTINGS = list(itertools.product((1, 2, 3), (0, 1, 2), (0, 1), (0, 1)))     # dfunc, reduce_tap, alt_hpel, fast_sub_pel
W, H, M = 320, 256, 160
REFINE_HALF = ((0, 0), (0, -1), (0, 1), (-1, 0), (1, 0), (-1, -1), (1, -1), (-1, 1), (1, 1))


def content(W, H, M, bd, seed):
    """smooth content (a sum of sinusoids) as reference; the original samples it displaced by one quarter-pel vector per 16x16 region, both with noise.
    Returns org, ref (int16, (H + 2M) x (W + 2M), sample (0, 0) at [M, M]) and the vectors (quarter pel) per region."""
    rs = np.random.RandomState(seed)
    mx = (1 << bd) - 1
    ys, xs = np.mgrid[-M:H + M, -M:W + M].astype(np.float64)

    def f(x, y):
        v = np.full(x.shape, 0.5)
        for k in range(5):
            per = rs_f[k, 0]; ang = rs_f[k, 1]; ph = rs_f[k, 2]
            v += 0.09 * np.sin(2 * np.pi * (np.cos(ang) * x + np.sin(ang) * y) / per + ph)
        return v * mx
    rs_f = np.stack([rs.uniform(6, 40, 5), rs.uniform(0, np.pi, 5), rs.uniform(0, 2 * np.pi, 5)], axis=1)
    nb = max(1, 1 << (bd - 8))
    ref = np.clip(np.rint(f(xs, ys)) + rs.randint(-nb, nb + 1, size=xs.shape), 0, mx)
    gy, gx = (H + 2 * M + 15) // 16, (W + 2 * M + 15) // 16
    vec = rs.randint(-14, 15, size=(gy, gx, 2))
    dx = np.kron(vec[:, :, 0], np.ones((16, 16)))[:xs.shape[0], :xs.shape[1]] / 4.0
    dy = np.kron(vec[:, :, 1], np.ones((16, 16)))[:xs.shape[0], :xs.shape[1]] / 4.0
    org = np.clip(np.rint(f(xs + dx, ys + dy)) + rs.randint(-nb, nb + 1, size=xs.shape), 0, mx)
    return np.ascontiguousarray(org, dtype=np.int16), np.ascontiguousarray(ref, dtype=np.int16), vec


def _int_vectors(rs, vec, x, y, w, h, W, H, M, extreme):
    """the integer vector the TZ walk would roughly find (the region's vector rounded, +-1), or a vector that takes the read box to a random place in the margin"""
    if not extreme:
        v = vec[(y + M) // 16, (x + M) // 16]
        return int(np.round(v[0] / 4.0)) + int(rs.randint(-1, 2)), int(np.round(v[1] / 4.0)) + int(rs.randint(-1, 2))
    # columns x + mx - 5 .. x + mx + w + 4 and rows y + my - 4 .. y + my + h + 3 inside -M .. W + M - 1 / H + M - 1
    side = rs.randint(4)
    mx = int(rs.randint(-M + 5, W + M - w - 4)) - x
    my = int(rs.randint(-M + 4, H + M - h - 3)) - y
    if side == 0: mx = -M + 5 + int(rs.randint(0, 8)) - x
    if side == 1: mx = W + M - 1 - w - 4 - int(rs.randint(0, 8)) - x
    if side == 2: my = -M + 4 + int(rs.randint(0, 8)) - y
    if side == 3: my = H + M - 1 - h - 3 - int(rs.randint(0, 8)) - y
    return mx, my


def pus_for(w, h, k, seed, vec, W=W, H=H, M=M):
    """k PUs of one shape: positions spread over the picture, half of them with vectors beyond a picture edge.  Rows: x, y, w, h, mvx, mvy, pred_hor, pred_ver"""
    rs = np.random.RandomState(seed)
    blk = np.zeros((k, 8), dtype=np.int32)
    for i in range(k):
        x = int(rs.randint(0, (W - w) // 4 + 1)) * 4; y = int(rs.randint(0, (H - h) // 4 + 1)) * 4
        mx, my = _int_vectors(rs, vec, x, y, w, h, W, H, M, i % 2 == 1)
        blk[i] = (x, y, w, h, mx, my, int(rs.randint(-200, 201)), int(rs.randint(-200, 201)))
    return blk


@pytest.fixture(scope="module")
def ref():
    R = refshim()
    R.refshim_frac_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    R.refshim_tz_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double] + [ctypes.c_int] * 7 + [ctypes.c_void_p]
    R.refshim_set_simd(b'AVX2')
    return R


@pytest.fixture(scope="module")
def eng():
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def member(R, org, ref_, S, M, blk, bd, lam, dfunc, rt, alt, fast):
    """the member's rcMvHalf, rcMvQter and ruiCost: int64 [n][5]"""
    base = M * S + M
    out = np.zeros((len(blk), 6), dtype=np.int32)
    R.refshim_frac_search_member(1, PO(org, base), S, PO(ref_, base), S, P(np.ascontiguousarray(blk)), len(blk), bd, lam, rt, dfunc - 1, alt, fast, P(out))
    cost = (out[:, 4].astype(np.int64) & 0xffffffff) | (out[:, 5].astype(np.int64) << 32)
    return np.concatenate([out[:, :4].astype(np.int64), cost[:, None]], axis=1)


def tz_arrays(blk):
    import vvenc_b200 as V
    pus = np.zeros(len(blk), dtype=V.TZ_PU_DT); mv = np.zeros(len(blk), dtype=V.TZ_BEST_DT)
    pus['x'] = blk[:, 0]; pus['y'] = blk[:, 1]; pus['pred_hor'] = blk[:, 6]; pus['pred_ver'] = blk[:, 7]
    mv['mv_hor'] = blk[:, 4]; mv['mv_ver'] = blk[:, 5]
    return pus, mv


def as_rows(best):
    cost = best['cost'].astype(np.uint64)
    assert (cost < (1 << 63)).all()
    return np.stack([best['half_hor'], best['half_ver'], best['qter_hor'], best['qter_ver'], cost.astype(np.int64)], axis=1).astype(np.int64)


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_frac_search_equals_the_member(eng, ref, bd):
    org, cur, vec = content(W, H, M, bd, 300 + bd)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M, bit_depth=bd); eng.upload_plane(1, cur, W, H, M, bit_depth=bd)
    bad = []; n = 0
    for (w, h) in SHAPES:
        blk = pus_for(w, h, 6, 10 * w + h + bd, vec)
        pus, mv = tz_arrays(blk)
        for (dfunc, rt, alt, fast) in SETTINGS:
            mem = member(ref, org, cur, S, M, blk, bd, LAM, dfunc, rt, alt, fast)
            dev = as_rows(eng.frac_search(0, 1, pus, mv, w, h, eng.frac_par(LAM, dfunc, rt, alt, fast)))
            n += len(blk)
            if not np.array_equal(dev, mem):
                bad.append((w, h, dfunc, rt, alt, fast))
    assert n == len(SHAPES) * len(SETTINGS) * 6
    assert bad == [], bad[:10]


def test_content_exercises_the_selection(ref):
    """every half-pel direction and every quarter-pel offset with fast_sub_pel 0 and 1, and the pattern-0 end of fast mode (the member's quarter-pel round does
    not run: the replay of its pattern id on the oracle's table says so, and the replay's result is the member's)"""
    from vvenc_b200 import candidates as cand
    O = oracle()
    O.orc_mv_cost.restype = ctypes.c_uint64
    org, cur, vec = content(W, H, M, 10, 310)
    S = W + 2 * M; base = M * S + M
    for fast in (0, 1):
        halves, quarters, pattern0 = set(), set(), 0
        for (w, h) in SHAPES:
            if max(w, h) > 64:
                continue
            blk = pus_for(w, h, 64, 10 * w + h + 10, vec)
            for dfunc in (1, 2):
                mem = member(ref, org, cur, S, M, blk, 10, LAM, dfunc, 2, 0, fast)
                halves |= {REFINE_HALF.index((int(r[0]), int(r[1]))) for r in mem}
                quarters |= {(int(r[2]), int(r[3])) for r in mem}
                if fast:
                    tab = np.zeros((len(blk), 7, 7), dtype=np.uint32)
                    O.orc_frac_cost_grid(PO(org, base), S, PO(cur, base), S, P(np.ascontiguousarray(blk[:, :6])), len(blk), dfunc, 10, 2, 0, P(tab))
                    for k, r in enumerate(mem):
                        ph, pv = int(blk[k, 6]), int(blk[k, 7])
                        half, quarter, cost = cand.subpel_refinement_fast(tab[k], (int(blk[k, 4]), int(blk[k, 5])),
                                                                          lambda x, y, cs: int(O.orc_mv_cost(LAM, x, y, ph, pv, cs, 0)))
                        assert (half, quarter or (0, 0), cost) == ((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4]))
                        pattern0 += quarter is None
        assert halves == set(range(9)), (fast, halves)
        assert quarters == {(x, y) for x in (-1, 0, 1) for y in (-1, 0, 1)}, (fast, quarters)
        if fast:
            assert pattern0 > 0



@gpu
def test_chain_tz_then_frac_on_the_device(eng, ref):
    """every PU of 8x8..128x128 on a 1920x1080 10-bit pair: vvb_tz_search_dev -> vvb_frac_search_dev, one synchronise, against the two members"""
    import torch
    import vvenc_b200 as V
    PW, PH, CTU, RNG = 1920, 1080, 128, 64
    MG = CTU + 12                                            # the margin the header states for chained calls
    org, cur, vec = content(PW, PH, MG, 10, 77)
    S = PW + 2 * MG; base = MG * S + MG
    eng.upload_plane(0, org, PW, PH, MG); eng.upload_plane(1, cur, PW, PH, MG)
    me = eng.me_par(LAM, 2, 0)
    tz = eng.tz_par(RNG, PW, PH, CTU, extended=False, fast=True, integer_et=False, first_search_stop=True)
    fpar = eng.frac_par(LAM, V.DF_HAD, 2, False, 1)
    rs = np.random.RandomState(5)
    jobs = []
    for s in (8, 16, 32, 64, 128):
        ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
        pus = np.zeros(xs.size, dtype=V.TZ_PU_DT)
        pus['x'] = xs.ravel(); pus['y'] = ys.ravel()
        pus['start_hor'] = rs.randint(-40 * 16, 40 * 16 + 1, size=xs.size); pus['start_ver'] = rs.randint(-24 * 16, 24 * 16 + 1, size=xs.size)
        q = lambda v: np.where(v >= 0, (v + 1) >> 2, (v + 2) >> 2)
        pus['pred_hor'] = q(pus['start_hor'].astype(np.int64)); pus['pred_ver'] = q(pus['start_ver'].astype(np.int64))
        d_pus = torch.from_numpy(np.frombuffer(pus.tobytes(), dtype=np.uint8).copy()).cuda()
        d_mv = torch.zeros(len(pus) * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        d_out = torch.zeros(len(pus) * V.FRAC_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        jobs.append((s, pus, d_pus, d_mv, d_out))
    torch.cuda.synchronize()
    before = eng.launches
    for (s, pus, d_pus, d_mv, d_out) in jobs:
        vp = ctypes.c_void_p
        eng._chk(eng.lib.vvb_tz_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), len(pus), s, s, ctypes.byref(me), ctypes.byref(tz), None, 0, vp(d_mv.data_ptr())))
        eng._chk(eng.lib.vvb_frac_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), vp(d_mv.data_ptr()), len(pus), s, s, ctypes.byref(fpar), vp(d_out.data_ptr())))
    eng.synchronize()
    assert eng.launches - before == 2 * len(jobs)
    for (s, pus, d_pus, d_mv, d_out) in jobs:
        blk = np.zeros((len(pus), 6), dtype=np.int32)
        blk[:, 0] = pus['x']; blk[:, 1] = pus['y']; blk[:, 2] = s; blk[:, 3] = s; blk[:, 4] = pus['start_hor']; blk[:, 5] = pus['start_ver']
        tzm = np.zeros((len(pus), 8), dtype=np.int64)
        assert ref.refshim_tz_search_member(1, PO(org, base), S, PO(cur, base), S, PW, PH, MG, P(blk), len(blk), 10, 0, LAM, RNG, CTU, 0, 1, 0, 1, 0, P(tzm)) == 0
        fb = np.zeros((len(pus), 8), dtype=np.int32)
        fb[:, :4] = blk[:, :4]; fb[:, 4] = tzm[:, 0]; fb[:, 5] = tzm[:, 1]; fb[:, 6] = pus['pred_hor']; fb[:, 7] = pus['pred_ver']
        mem = member(ref, org, cur, S, MG, fb, 10, LAM, V.DF_HAD, 2, 0, 1)
        dev_mv = np.frombuffer(d_mv.cpu().numpy().tobytes(), dtype=V.TZ_BEST_DT)
        assert np.array_equal(dev_mv['mv_hor'], tzm[:, 0]) and np.array_equal(dev_mv['mv_ver'], tzm[:, 1]), s
        dev = as_rows(np.frombuffer(d_out.cpu().numpy().tobytes(), dtype=V.FRAC_BEST_DT))
        assert np.array_equal(dev, mem), (s, int((dev != mem).any(axis=1).sum()))


@gpu
@pytest.mark.parametrize("fast", [0, 1])
def test_frac_search_equals_the_grid_path(eng, ref, fast):
    import vvenc_b200 as V
    from vvenc_b200 import candidates as cand
    O = oracle()
    O.orc_mv_cost.restype = ctypes.c_uint64
    org, cur, vec = content(W, H, M, 10, 320)
    eng.upload_plane(0, org, W, H, M); eng.upload_plane(1, cur, W, H, M)
    n = 0
    for (w, h) in SHAPES:
        if max(w, h) > 64:
            continue
        blk = pus_for(w, h, 12, 7 * w + h, vec)
        pus, mv = tz_arrays(blk)
        for dfunc, alt in ((1, 0), (2, 0), (3, 0), (2, 1)):
            b = np.zeros(len(blk), dtype=V.BLOCK_DT)
            b['x'] = blk[:, 0]; b['y'] = blk[:, 1]; b['start_x'] = blk[:, 4]; b['start_y'] = blk[:, 5]
            tab = eng.frac_cost_grid(dfunc, 0, 1, b, w, h, 2, alt)
            dev = eng.frac_search(0, 1, pus, mv, w, h, eng.frac_par(LAM, dfunc, 2, alt, fast))
            replay = cand.subpel_refinement_fast if fast else cand.subpel_refinement
            for k in range(len(blk)):
                ph, pv = int(blk[k, 6]), int(blk[k, 7])
                half, quarter, cost = replay(tab[k], (int(blk[k, 4]), int(blk[k, 5])), lambda x, y, cs: int(O.orc_mv_cost(LAM, x, y, ph, pv, cs, 0)), quarter_round=not alt)
                d = dev[k]
                assert ((int(d['half_hor']), int(d['half_ver'])), (int(d['qter_hor']), int(d['qter_ver'])), int(d['cost'])) == (half, quarter or (0, 0), cost), (w, h, dfunc, alt, k)
                n += 1
    assert n == 11 * 12 * 4


@gpu
def test_frac_search_admission(eng, ref):
    import vvenc_b200 as V
    import vvenc_b200._lib as L
    org, cur, vec = content(W, H, M, 10, 330)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M); eng.upload_plane(1, cur, W, H, M)
    blk = pus_for(16, 16, 4, 3, vec)
    pus, mv = tz_arrays(blk)
    par = eng.frac_par(LAM, V.DF_HAD)
    out = np.zeros(len(pus), dtype=V.FRAC_BEST_DT)
    lib, h = eng.lib, eng.h

    def call(pu=pus, m=mv, n=len(pus), w=16, hh=16, p=par, o=out, org_plane=0, ref_plane=1):
        return lib.vvb_frac_search(h, org_plane, ref_plane, P(pu) if pu is not None else None, P(m) if m is not None else None, n, w, hh,
                                   ctypes.byref(p) if p is not None else None, P(o) if o is not None else None)
    assert call() == L.VVB_OK
    for kw in (dict(pu=None), dict(m=None), dict(p=None), dict(o=None), dict(n=-1), dict(org_plane=7), dict(ref_plane=-1)):
        assert call(**kw) == L.VVB_ERR_ARG, kw
    for p in (eng.frac_par(LAM, V.DF_HAD, fast_sub_pel=2), eng.frac_par(LAM, V.DF_HAD, fast_sub_pel=-1), eng.frac_par(LAM, V.DF_HAD, reduce_tap=3),
              eng.frac_par(LAM, V.DF_HAD, reduce_tap=-1), eng.frac_par(-1.0, V.DF_HAD), eng.frac_par(float('nan'), V.DF_HAD), eng.frac_par(float('inf'), V.DF_HAD)):
        assert call(p=p) == L.VVB_ERR_ARG
    for p in (eng.frac_par(LAM, V.DF_SSE), eng.frac_par(LAM, V.DF_HAD_2SAD)):
        assert call(p=p) == L.VVB_ERR_UNSUPPORTED
    for (w, hh) in ((4, 4), (256, 16), (16, 256), (2, 8), (12, 16), (16, 24)):
        assert call(w=w, hh=hh) == L.VVB_ERR_UNSUPPORTED, (w, hh)
    # a PU outside the picture: refused by the host call, the sentinel from _dev
    for (x, y) in ((-4, 0), (0, -4), (W - 12, 0), (0, H - 12)):
        p2 = pus.copy(); p2['x'][1] = x; p2['y'][1] = y
        m2 = mv.copy(); m2['mv_hor'][1] = 0; m2['mv_ver'][1] = 0
        assert call(pu=p2, m=m2) == L.VVB_ERR_ARG, (x, y)
    # n == 0: no launch
    before = eng.launches
    assert call(n=0) == L.VVB_OK and eng.launches == before
    # planes above 12 bits
    eng.upload_plane(2, cur, W, H, M, bit_depth=13)
    assert call(ref_plane=2) == L.VVB_ERR_UNSUPPORTED and call(org_plane=2) == L.VVB_ERR_UNSUPPORTED
    eng.free_plane(2)

    # the read box (columns x + mv - 5 .. x + mv + w + 4, rows y + mv - 4 .. y + mv + h + 3) at the margin on each side, then one pel beyond it
    import torch
    w = hh = 16
    x, y = 64, 48
    edges = [(-M + 5 - x, 0), (W + M - 1 - w - 4 - x, 0), (0, -M + 4 - y), (0, H + M - 1 - hh - 3 - y)]
    steps = [(-1, 0), (1, 0), (0, -1), (0, 1)]
    for (mx, my), (sx, sy) in zip(edges, steps):
        blk1 = np.array([[x, y, w, hh, mx, my, 3, -5], [x, y, w, hh, mx + sx, my + sy, 3, -5]], dtype=np.int32)
        pu1, mv1 = tz_arrays(blk1)
        for dfunc, rt, fast in ((2, 0, 0), (1, 2, 1)):
            par1 = eng.frac_par(LAM, dfunc, rt, False, fast)
            mem = member(ref, org, cur, S, M, blk1[:1], 10, LAM, dfunc, rt, 0, fast)
            assert np.array_equal(as_rows(eng.frac_search(0, 1, pu1[:1], mv1[:1], w, hh, par1)), mem), (mx, my)
            o1 = np.zeros(2, dtype=V.FRAC_BEST_DT)
            assert call(pu=pu1, m=mv1, n=2, p=par1, o=o1) == L.VVB_ERR_UNSUPPORTED
            d_pu = torch.from_numpy(np.frombuffer(pu1.tobytes(), dtype=np.uint8).copy()).cuda()
            d_mv = torch.from_numpy(np.frombuffer(mv1.tobytes(), dtype=np.uint8).copy()).cuda()
            d_o = torch.full((2 * V.FRAC_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
            torch.cuda.synchronize()
            vp = ctypes.c_void_p
            assert lib.vvb_frac_search_dev(h, 0, 1, vp(d_pu.data_ptr()), vp(d_mv.data_ptr()), 2, w, hh, ctypes.byref(par1), vp(d_o.data_ptr())) == L.VVB_OK
            eng.synchronize()
            dv = np.frombuffer(d_o.cpu().numpy().tobytes(), dtype=V.FRAC_BEST_DT)
            assert np.array_equal(as_rows(dv[:1]), mem)
            assert int(dv['cost'][1]) == (1 << 64) - 1 and int(dv['half_hor'][1]) == int(dv['half_ver'][1]) == int(dv['qter_hor'][1]) == int(dv['qter_ver'][1]) == 0


@gpu
@pytest.mark.parametrize("dfunc", [2, 3])
def test_frac_search_format_limits(eng, ref, dfunc):
    """128x128 at 12 bits: original 0 / 4095 at random, reference 0, so every difference is 0 or 4095 and the Hadamard sums are near their top; a predictor at the
    int16 end against a vector at the far margin and a lambda whose table top fills 32 bits, so the MV rate alone comes near 2^32 (the table's entries are 32-bit)"""
    bd, w, hh, MG = 12, 128, 128, 160
    rs = np.random.RandomState(61)
    org = np.ascontiguousarray((rs.randint(0, 2, size=(H + 2 * MG, W + 2 * MG)) * 4095).astype(np.int16))
    cur = np.zeros_like(org)
    S = W + 2 * MG
    eng.upload_plane(0, org, W, H, MG, bit_depth=bd); eng.upload_plane(1, cur, W, H, MG, bit_depth=bd)
    lam = (4294967295.0 / 79) ** 2 * 0.999
    x, y = W - w, H - hh
    mx, my = W + MG - 1 - w - 4 - x, H + MG - 1 - hh - 3 - y
    blk = np.array([[x, y, w, hh, mx, my, -32768, -32768], [0, 0, w, hh, -MG + 5, -MG + 4, 32767, 32767]], dtype=np.int32)
    pus, mv = tz_arrays(blk)
    for fast in (0, 1):
        mem = member(ref, org, cur, S, MG, blk, bd, lam, dfunc, 2, 0, fast)
        assert (mem[:, 4] > (1 << 31)).all()
        dev = as_rows(eng.frac_search(0, 1, pus, mv, w, hh, eng.frac_par(lam, dfunc, 2, False, fast)))
        assert np.array_equal(dev, mem), (dev, mem)
