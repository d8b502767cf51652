"""vvb_amvr_refine and vvb_bipred_amvr_search: InterSearch::xPatternSearchIntRefine on the device, against a restatement of the member on the probe's own
pieces (the compiler report runs on the CPU, the rest needs -m gpu).

No probe entry runs xPatternSearchIntRefine, so the member (InterSearch.cpp:2576-2676) is restated here as `restate`:
  * every distortion is refshim_dist (the AVX2 table; the scalar table agrees on these shapes and targets, test_gpu_bipred_search pins both);
  * the MV rate is refshim_mv_bits at cost scale 0 (getBitsOfVectorWithPredictor) and getCost is test_gpu_bipred_search.get_cost, cross-checked against
    refshim_mv_cost;
  * Mv::changePrecision's rounding (Mv.h:189-203), roundTransPrecInternal2Amvr, xClipMvToFppLine with CU::isMvInRangeFPP (InterSearch.cpp:2154-2163,
    UnitTools.cpp:3526-3535), roundTransPrecInternal2AmvrVertical (Mv.h:227-234) and clipMv (Mv.cpp:68-80, test_gpu_tz_search.Replay.clip with search False).
The bi branch's integer stage is checked against refshim_pattern_search_member over test_gpu_bipred_search's replayed start (BiReplay), with imvShift 2 / 4.
"""
import ctypes
import itertools

import numpy as np
import pytest

from _libs import have_ref, refshim, P, PO
from test_gpu_tz_search import Replay, _rshift
import test_gpu_bipred_search as B

pytestmark = pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
gpu = pytest.mark.gpu

LAM = 57.25
SHAPES = B.SHAPES + [(4, 8), (8, 4)]
W, H, CTU, M = B.W, B.H, B.CTU, B.M
POS = ((0, 0), (-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1))     # testPos (:2595), (hor, ver)
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
# dfunc, imv, ifp_lines, num_cand, mvp_idx, equal mvp_bits
SETTINGS = [s for s in itertools.product((1, 2, 3), (1, 2), (0, 1, 2), (1, 2), (0, 1), (0, 1)) if s[4] < s[3]]
STATS = dict(equal=0, fpp_moved=0, clip_moved=0, mvp_changed=0, off_centre=0, bcw_changed=0)


@pytest.fixture(scope="module")
def ref():
    return B.ref_setup(refshim())


@pytest.fixture(scope="module")
def eng():
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def fpp(y, h, ver, ifp, ph, ctu):
    """CU::isMvInRangeFPP (UnitTools.cpp:3526-3535) and xClipMvToFppLine (InterSearch.cpp:2154-2163); the vertical component, unrounded"""
    l2 = ctu.bit_length() - 1
    y_bmax = ((ph + ctu - 1) // ctu - 1 - ifp) << l2
    y_refmax = (((y >> l2) + ifp + 1) << l2) - 1
    y_refmv = y + h + 4 + (ver >> 4) - 1
    if ifp and y < y_bmax and y_refmv > y_refmax:
        return ver - ((y_refmv - y_refmax) << 4)
    return ver


def restate(R, key, ref_pl, S, bd, x, y, w, h, mv, amvp, bits, fam, imv, mvp_bits, lam, weight, pw, ph, ifp, count=True):
    """xPatternSearchIntRefine (InterSearch.cpp:2576-2676) for one PU whose key block is at key[M + y, M + x] and whose reference is ref_pl (both with margin
    M).  Returns (mv_hor, mv_ver, mvp_idx, bits, dist, cost), or None where the member throws."""
    s = 4 if imv == 1 else 6
    cand = [(int(amvp['cand_hor'][c]), int(amvp['cand_ver'][c])) for c in (0, 1)]
    nc, idx = int(amvp['num_cand']), int(amvp['mvp_idx'])
    rc = (16 * mv[0], 16 * mv[1])                                   # :2128 changePrecision( INT, INTERNAL )
    bits = (bits - mvp_bits[idx]) & M32                             # :2587
    bmvd = [(rc[0] - cand[c][0], rc[1] - cand[c][1]) for c in (0, 1)]
    if any((v & 3) for b in bmvd for v in b):                       # :2601-2602
        return None
    base = [(_rshift(b[0], s) << s, _rshift(b[1], s) << s) for b in bmvd]     # roundTransPrecInternal2Amvr
    hmin, hmax, vmin, vmax = Replay(R, key, ref_pl, S, M, bd, w, h, 0, 0, CTU, (0, 0, 0, 0), pw, ph).clip(x, y, False)
    o = M * S + M + y * S + x
    best, bmv, bidx, bbits, bpos = M64, rc, idx, 0, 0
    dist = 0
    for pos, (ph_, pv_) in enumerate(POS):
        t = [None, None]
        for c in range(nc):
            th = (ph_ << s) + base[c][0] + cand[c][0]
            tv = (pv_ << s) + base[c][1] + cand[c][1]
            tf = fpp(y, h, tv, ifp, ph, CTU)
            if tf != tv:
                tf = _rshift(tf, s) << s                            # roundTransPrecInternal2AmvrVertical
                STATS['fpp_moved'] += count and tf != tv
                tv = tf
            t[c] = (th, tv)
            if c == 0 or t[0] != t[1]:
                cx, cy = min(hmax, max(hmin, th)), min(vmax, max(vmin, tv))
                STATS['clip_moved'] += count and (cx, cy) != (th, tv)
                d = int(R.refshim_dist(1, fam, PO(key, o), S, PO(ref_pl, o + (cy >> 4) * S + (cx >> 4)), S, w, h, bd, 0))
                dist = B.u64(float(d) * weight)
            else:
                STATS['equal'] += count
            mb = (mvp_bits[c] + int(R.refshim_mv_bits(_rshift(th, s), _rshift(tv, s), _rshift(cand[c][0], s), _rshift(cand[c][1], s), 0, 0))) & M32
            ud = (dist + B.get_cost(lam, mb)) & M64
            if ud < best:
                best, bmv, bidx, bbits, bpos = ud, (th, tv), c, mb, pos
    if best == M64:
        return rc[0], rc[1], idx, bits, M64, M64                   # :2655-2659
    if count:
        STATS['mvp_changed'] += bidx != idx
        STATS['off_centre'] += bpos != 0
    bits = (bits + bbits) & M32
    return bmv[0], bmv[1], bidx, bits, best, (best - B.get_cost(lam, bbits) + B.get_cost(lam, bits)) & M64


def got(r):
    return (int(r['mv_hor']), int(r['mv_ver']), int(r['mvp_idx']), int(r['bits']), int(r['dist']), int(r['cost']))


def make_amvp(n, nc, idx, s, rs):
    """amvpInfo per PU: candidates that are multiples of 4, half of them rounded to the AMVR precision (as fillMvpCand leaves them), so both kinds of
    cBaseMvd occur and equal test vectors of the two candidates occur"""
    import vvenc_b200 as V
    a = np.zeros(n, dtype=V.AMVP_DT)
    for i in range(n):
        for c in (0, 1):
            step = (1 << s) if rs.randint(2) else 4
            a['cand_hor'][i, c] = rs.randint(-600 // step, 600 // step + 1) * step
            a['cand_ver'][i, c] = rs.randint(-400 // step, 400 // step + 1) * step
        if rs.randint(6) == 0:
            a['cand_ver'][i, 1 - idx] = 60000 // 64 * 64                   # far below: the FPP and clipMv limits act on its test vectors
        a['num_cand'][i] = nc; a['mvp_idx'][i] = idx
    return a


def _dev(t):
    import torch
    return torch.from_numpy(np.frombuffer(np.ascontiguousarray(t).tobytes(), dtype=np.uint8).copy()).cuda()


def _host(t, dt):
    return np.frombuffer(t.cpu().numpy().tobytes(), dtype=dt).copy()


def uni_call(eng, org_plane, ref_plane, pus, amvp, bits, w, h, par, me, tz):
    """vvb_tz_search_dev -> vvb_amvr_refine_dev on the device; then the host-buffer call on the same integer vectors.  Returns (int_mv, dev, host)."""
    import torch
    import vvenc_b200 as V
    vp = ctypes.c_void_p
    n = len(pus)
    d_pus, d_amvp, d_bits = _dev(pus), _dev(amvp), _dev(bits.astype(np.uint32))
    d_mv = torch.zeros(n * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
    d_out = torch.full((n * V.AMVR_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    eng._chk(eng.lib.vvb_tz_search_dev(eng.h, org_plane, ref_plane, vp(d_pus.data_ptr()), n, w, h, ctypes.byref(me), ctypes.byref(tz), None, 0, vp(d_mv.data_ptr())))
    eng._chk(eng.lib.vvb_amvr_refine_dev(eng.h, org_plane, ref_plane, vp(d_pus.data_ptr()), vp(d_mv.data_ptr()), vp(d_amvp.data_ptr()), vp(d_bits.data_ptr()), n, w, h,
                                         ctypes.byref(par), vp(d_out.data_ptr())))
    eng.synchronize()
    mv, dev = _host(d_mv, V.TZ_BEST_DT), _host(d_out, V.AMVR_BEST_DT)
    host = eng.amvr_refine(org_plane, ref_plane, pus, mv, amvp, bits, w, h, par)
    return mv, dev, host


def tz_pus(w, h, k, rs, amvp, pw=W, ph=H):
    import vvenc_b200 as V
    pus = np.zeros(k, dtype=V.TZ_PU_DT)
    pus['x'] = rs.randint(0, pw - w + 1, size=k); pus['y'] = rs.randint(0, ph - h + 1, size=k)
    far = rs.randint(4, size=k) == 0                                        # beyond a picture edge: clipped by xClipMvSearch
    lim = np.where(far, 60000, 24 * 16)
    pus['start_hor'] = rs.randint(-1 << 20, 1 << 20, size=k) % (2 * lim + 1) - lim
    pus['start_ver'] = rs.randint(-1 << 20, 1 << 20, size=k) % (2 * lim + 1) - lim
    idx = amvp['mvp_idx']
    pus['pred_hor'] = amvp['cand_hor'][np.arange(k), idx] // 4; pus['pred_ver'] = amvp['cand_ver'][np.arange(k), idx] // 4
    return pus


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_uni_chain_equals_the_restatement(eng, ref, bd):
    """vvb_tz_search_dev (imv_shift 2 / 4) -> vvb_amvr_refine_dev against the restatement at the device's integer vector, field by field, every setting with
    two shapes per bit depth; the host-buffer call gives the same bytes"""
    org, cur, _ = B._planes(bd, 800 + bd)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M, bit_depth=bd); eng.upload_plane(1, cur, W, H, M, bit_depth=bd)
    keep = dict(STATS)
    bad, n = [], 0
    for k, (dfunc, imv, ifp, nc, idx, eqb) in enumerate(SETTINGS):
        for w, h in (SHAPES[k % len(SHAPES)], SHAPES[(5 * k + bd) % len(SHAPES)]):
            rs = np.random.RandomState(100000 * bd + 100 * k + w + h)
            s = 4 if imv == 1 else 6
            amvp = make_amvp(6, nc, idx, s, rs)
            pus = tz_pus(w, h, 6, rs, amvp)
            pus['start_ver'][0] = 60000                                       # at the xClipMvSearch / ifp_lines bound
            bits = rs.randint(0, 60, size=6).astype(np.uint32)
            mvp_bits = (1, 1) if eqb else (1, 3)
            par = eng.amvr_par(LAM, dfunc, imv, mvp_bits, W, H, CTU, ifp)
            me = eng.me_par(LAM, 2, imv << 1)
            tz = eng.tz_par(64, W, H, CTU, extended=bool(k & 1), fast=not k & 1, sub_shift_mode=k % 3, ifp_lines=ifp)
            mv, dev, host = uni_call(eng, 0, 1, pus, amvp, bits, w, h, par, me, tz)
            assert host.tobytes() == dev.tobytes(), (w, h, dfunc, imv, ifp, nc, idx)
            for i in range(len(pus)):
                exp = restate(ref, org, cur, S, bd, int(pus['x'][i]), int(pus['y'][i]), w, h, (int(mv['mv_hor'][i]), int(mv['mv_ver'][i])), amvp[i],
                              int(bits[i]), dfunc, imv, mvp_bits, LAM, 1.0, W, H, ifp)
                n += 1
                if got(dev[i]) != exp:
                    bad.append((w, h, dfunc, imv, ifp, nc, idx, eqb, i, got(dev[i]), exp))
    d = {key: STATS[key] - keep[key] for key in STATS}
    assert bad == [], (len(bad), n, bad[:5])
    assert d['equal'] > 0 and d['fpp_moved'] > 0 and d['clip_moved'] > 0 and d['mvp_changed'] > 0 and d['off_centre'] > 0, d


def bi_pus(w, h, rs, amvp):
    pus, cands = B.make_pus(w, h, 5, rs)
    k = len(pus)
    idx = amvp['mvp_idx'][:k]
    pus['pred_hor'] = amvp['cand_hor'][np.arange(k), idx] // 4; pus['pred_ver'] = amvp['cand_ver'][np.arange(k), idx] // 4
    return pus, cands


def check_bi(R, eng, org, cur, S, bd, pus, amvp, cands, pred, w, h, par, mvp_bits, int_out, out, lam=LAM, bcw_stats=True):
    """the integer stage against refshim_pattern_search_member over the replayed start, the refinement against the restatement on a plane that holds each PU's
    target; returns the PUs that differ"""
    imv_shift = par.imv << 1
    tgt = org.astype(np.int32).copy()
    base = M * S + M
    for i in range(len(pus)):
        x, y = int(pus['x'][i]), int(pus['y'][i])
        tgt[M + y:M + y + h, M + x:M + x + w] = B.target(org[M + y:M + y + h, M + x:M + x + w], pred[i], bool(par.clip), bd)
    tgt = np.ascontiguousarray(tgt, dtype=np.int16)
    keep = B.LAM
    B.LAM = lam
    try:
        rp = B.BiReplay(R, tgt, cur, S, bd, w, h, par.sub_shift_mode, par.search_range, par.ifp_lines, imv_shift, par.pic_w, par.pic_h)
        bad = []
        for i in range(len(pus)):
            x, y = int(pus['x'][i]), int(pus['y'][i]); pq = (int(pus['pred_hor'][i]), int(pus['pred_ver'][i]))
            cf, cc = int(pus['cand_first'][i]), int(pus['cand_count'][i])
            l, r, t, b = rp.window(x, y, (int(pus['start_hor'][i]), int(pus['start_ver'][i])), pq, [tuple(int(v) for v in c) for c in cands[cf:cf + cc]])
            blk = np.array([[x, y, w, h, l, r, t, b, pq[0], pq[1]]], dtype=np.int32)
            o = np.zeros(4, dtype=np.int32)
            R.refshim_pattern_search_member(1, PO(tgt, base), S, PO(cur, base), S, P(blk), 1, bd, par.sub_shift_mode, lam, 2, imv_shift, P(o))
            mx, my = int(o[0]), int(o[1]); ibest = (int(o[2]) & M32) | ((int(o[3]) & M32) << 32)
            sad = (ibest - int(R.refshim_mv_cost(lam, mx, my, pq[0], pq[1], 2, imv_shift))) & M64
            gi = (int(int_out['mv_hor'][i]), int(int_out['mv_ver'][i]), int(int_out['sad'][i]), int(int_out['cost'][i]))
            wgt = 0.5 if int(pus['bcw_idx'][i]) == 2 else abs((8 - B.BCW[int(pus['bcw_idx'][i])] if par.ref_list == 0 else B.BCW[int(pus['bcw_idx'][i])]) / 8.0)
            exp = restate(R, tgt, cur, S, bd, x, y, w, h, (mx, my), amvp[i], int(pus['bits'][i]), par.dfunc, par.imv, mvp_bits, lam, wgt, par.pic_w, par.pic_h,
                          par.ifp_lines)
            if bcw_stats:
                unw = restate(R, tgt, cur, S, bd, x, y, w, h, (mx, my), amvp[i], int(pus['bits'][i]), par.dfunc, par.imv, mvp_bits, lam, 1.0, par.pic_w,
                              par.pic_h, par.ifp_lines, count=False)
                STATS['bcw_changed'] += exp[:3] != unw[:3]
            if gi != (mx, my, sad, ibest) or got(out[i]) != exp:
                bad.append((i, gi, (mx, my, sad, ibest), got(out[i]), exp))
        return bad
    finally:
        B.LAM = keep


@gpu
@pytest.mark.parametrize("bd", [10, 12])
def test_bipred_amvr_search_equals_the_members(eng, ref, bd):
    """the one-call bi branch for imv 1 / 2: all five BCW indices (make_pus cycles them), both lists, clip on and off, every dfunc, ifp_lines 0..2, over the
    twelve shapes; the _dev twin gives the bytes of the host-buffer call"""
    import torch
    import vvenc_b200 as V
    org, cur, oth = B._planes(bd, 900 + bd)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M, bit_depth=bd); eng.upload_plane(1, cur, W, H, M, bit_depth=bd)
    keep = dict(STATS)
    bad, seen = [], set()
    vp = ctypes.c_void_p
    for k, (dfunc, imv, rl, clip) in enumerate(itertools.product((1, 2, 3), (1, 2), (0, 1), (0, 1))):
        for si in (k % len(B.SHAPES), (7 * k + bd) % len(B.SHAPES)):
            w, h = B.SHAPES[si]
            rs = np.random.RandomState(7000 * bd + 31 * k + si)
            s = 4 if imv == 1 else 6
            nc = 1 if k % 4 == 3 else 2
            amvp = make_amvp(5, nc, (k // 2) % nc, s, rs)
            pus, cands = bi_pus(w, h, rs, amvp)
            amvp = amvp[:len(pus)]
            pred = B._pred_blocks(oth, pus, w, h, rs)
            mvp_bits = (1, 1 + k % 3)
            lam = LAM if k % 2 == 0 else 3000.0                                 # rate comparable to distortion: the BCW weight decides more often
            par = eng.bi_par(lam, (0, 1, 4, 8)[k % 4], W, H, CTU, dfunc, ref_list=rl, clip=clip, imv=imv, sub_shift_mode=k % 3, ifp_lines=(k + si) % 3)
            int_out, out = eng.bipred_amvr_search(0, 1, pus, amvp, w, h, par, mvp_bits, pred, cands)
            seen.add((dfunc, imv, rl, clip))
            bad += [(w, h, dfunc, imv, rl, clip) + b for b in check_bi(ref, eng, org, cur, S, bd, pus, amvp, cands, pred, w, h, par, mvp_bits, int_out, out, lam=lam)]
            d_pus, d_amvp, d_c, d_pr = _dev(pus), _dev(amvp), _dev(cands.astype(np.int32)), torch.from_numpy(pred).cuda()
            d_i = torch.zeros(len(pus) * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
            d_o = torch.zeros(len(pus) * V.AMVR_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
            mb = np.array(mvp_bits, dtype=np.uint32)
            torch.cuda.synchronize()
            eng._chk(eng.lib.vvb_bipred_amvr_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), vp(d_amvp.data_ptr()), len(pus), w, h, ctypes.byref(par), P(mb),
                                                        vp(d_c.data_ptr()) if len(cands) else None, len(cands), vp(d_pr.data_ptr()), vp(d_i.data_ptr()), vp(d_o.data_ptr())))
            eng.synchronize()
            assert _host(d_i, V.TZ_BEST_DT).tobytes() == int_out.tobytes() and _host(d_o, V.AMVR_BEST_DT).tobytes() == out.tobytes()
    assert len(seen) == 24
    d = {key: STATS[key] - keep[key] for key in STATS}
    assert bad == [], (len(bad), bad[:5])
    assert d['bcw_changed'] > 0 and d['equal'] > 0 and d['mvp_changed'] > 0 and d['off_centre'] > 0, d


@gpu
def test_persistent_loop_on_a_picture(eng, ref):
    """every 8x8 PU of a 1920x1080 10-bit picture in one chained call (more PUs than the grid holds resident warps), HAD_fast, IMV_4PEL, ifp_lines 1; a
    sample of PUs against the restatement and the whole call against the host-buffer call"""
    from test_gpu_frac_search import content
    PW, PH, MG = 1920, 1080, CTU + 12
    org, cur, _ = content(PW, PH, MG, 10, 77)
    S = PW + 2 * MG
    eng.upload_plane(0, org, PW, PH, MG); eng.upload_plane(1, cur, PW, PH, MG)
    rs = np.random.RandomState(8)
    ys, xs = np.mgrid[0:PH - 8 + 1:8, 0:PW - 8 + 1:8]
    n = xs.size
    amvp = make_amvp(n, 2, 0, 6, rs)
    amvp['mvp_idx'] = rs.randint(0, 2, size=n)
    pus = tz_pus(8, 8, n, rs, amvp, PW, PH)
    pus['x'] = xs.ravel(); pus['y'] = ys.ravel()
    bits = rs.randint(0, 100, size=n).astype(np.uint32)
    par = eng.amvr_par(LAM, 3, 2, (1, 1), PW, PH, CTU, 1)
    mv, dev, host = uni_call(eng, 0, 1, pus, amvp, bits, 8, 8, par, eng.me_par(LAM, 2, 4), eng.tz_par(64, PW, PH, CTU, fast=True, ifp_lines=1))
    assert host.tobytes() == dev.tobytes()
    for i in rs.choice(n, size=400, replace=False):
        exp = restate(ref, org, cur, S, 10, int(pus['x'][i]), int(pus['y'][i]), 8, 8, (int(mv['mv_hor'][i]), int(mv['mv_ver'][i])), amvp[i], int(bits[i]),
                      3, 2, (1, 1), LAM, 1.0, PW, PH, 1, count=False)
        assert got(dev[i]) == exp, (i, got(dev[i]), exp)


@gpu
def test_limits(eng, ref):
    """128x128 at 12 bits with full-contrast planes; a lambda whose getCost values exceed 2^32 (the refinement computes getCost directly); ruiBits near the
    uint32 wrap; the bi target at both ends of its range"""
    import vvenc_b200 as V
    bd, w, h = 12, 128, 128
    rs = np.random.RandomState(63)
    mx = (1 << bd) - 1
    org = np.ascontiguousarray((rs.randint(0, 2, size=(H + 2 * M, W + 2 * M)) * mx).astype(np.int16))
    cur = np.ascontiguousarray((rs.randint(0, 2, size=org.shape) * mx).astype(np.int16))
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M, bit_depth=bd); eng.upload_plane(1, cur, W, H, M, bit_depth=bd)
    big = (4294967295.0 / 3) ** 2 * 4.0                                    # getCost( 3 ) > 2^32
    b7 = int(ref.refshim_mv_bits(7, 0, 0, 0, 0, 0))
    assert B.get_cost(big, b7) > 1 << 32 and B.get_cost(big, b7) == int(ref.refshim_mv_cost(big, 7, 0, 0, 0, 0, 0))
    n = 4
    amvp = make_amvp(n, 2, 0, 4, rs)
    pus = np.zeros(n, dtype=V.TZ_PU_DT)
    pus['x'] = (0, W - w, 64, 128); pus['y'] = (0, H - h, 256, 128)
    pus['pred_hor'] = amvp['cand_hor'][:, 0] // 4; pus['pred_ver'] = amvp['cand_ver'][:, 0] // 4
    mv = np.zeros(n, dtype=V.TZ_BEST_DT)
    mv['mv_hor'] = (-130, 200, 3, -7); mv['mv_ver'] = (-130, 200, -5, 9)
    bits = np.array([0xfffffff0, 0xffffffff, 5, 0], dtype=np.uint32)
    for dfunc in (1, 2, 3):
        for lam, imv, mb in ((LAM, 1, (1, 1)), (big, 2, (0xfffffff8, 2)), ((4294967295.0 / 79) ** 2 * 0.999, 1, (1, 3))):
            par = eng.amvr_par(lam, dfunc, imv, mb, W, H, CTU, 1)
            out = eng.amvr_refine(0, 1, pus, mv, amvp, bits, w, h, par)
            for i in range(n):
                exp = restate(ref, org, cur, S, bd, int(pus['x'][i]), int(pus['y'][i]), w, h, (int(mv['mv_hor'][i]), int(mv['mv_ver'][i])), amvp[i], int(bits[i]),
                              dfunc, imv, mb, lam, 1.0, W, H, 1, count=False)
                assert got(out[i]) == exp, (dfunc, lam, i, got(out[i]), exp)
    # the bi target at both ends: org max / pred 0 -> 8190, org 0 / pred max -> -4095
    bpus = np.zeros(2, dtype=V.BI_PU_DT)
    bpus['x'] = (0, W - w); bpus['y'] = (0, H - h); bpus['start_hor'] = (-60000, 60000); bpus['start_ver'] = (-60000, 60000)
    bamvp = make_amvp(2, 2, 1, 6, rs)
    bpus['pred_hor'] = bamvp['cand_hor'][:, 1] // 4; bpus['pred_ver'] = bamvp['cand_ver'][:, 1] // 4
    bpus['bits'] = (0xfffffff0, 3); bpus['bcw_idx'] = (4, 0)
    pred = np.ascontiguousarray(((1 - org[M:M + h, M:M + w] // mx) * mx)[None].repeat(2, 0).astype(np.int16))
    for dfunc in (1, 2, 3):
        for clip in (0, 1):
            par = eng.bi_par((4294967295.0 / 79) ** 2 * 0.999, 8, W, H, CTU, dfunc, clip=clip, imv=2, sub_shift_mode=0)
            io, out = eng.bipred_amvr_search(0, 1, bpus, bamvp, w, h, par, (1, 1), pred)
            assert check_bi(ref, eng, org, cur, S, bd, bpus, bamvp, np.zeros((0, 2), np.int32), pred, w, h, par, (1, 1), io, out, lam=par.lam) == [], (dfunc, clip)


@gpu
def test_admission(eng, ref):
    """the VVB_ERR_ARG / VVB_ERR_UNSUPPORTED table of both calls, the member's three CHECK inputs, n == 0 without a launch, and the reference margin at the
    clipMv box's need and one pel less on each side, for the host-buffer call and the _dev sentinel"""
    import torch
    import vvenc_b200 as V
    import vvenc_b200._lib as L
    bd = 10
    org, cur, oth = B._planes(bd, 950)
    eng.upload_plane(0, org, W, H, M); eng.upload_plane(1, cur, W, H, M)
    rs = np.random.RandomState(4)
    lib, hh = eng.lib, eng.h
    amvp = make_amvp(4, 2, 0, 4, rs)
    pus = tz_pus(16, 16, 4, rs, amvp)
    mv = np.zeros(4, dtype=V.TZ_BEST_DT); mv['mv_hor'] = (1, -2, 3, 0); mv['mv_ver'] = (0, 5, -1, 2)
    bits = np.full(4, 9, dtype=np.uint32)
    par = eng.amvr_par(LAM, V.DF_HAD, 1, (1, 1), W, H, CTU)
    out = np.zeros(4, dtype=V.AMVR_BEST_DT)

    def call(pu=pus, m=mv, a=amvp, b=bits, n=4, w=16, h=16, p=par, o=out, org_plane=0, ref_plane=1):
        q = lambda x: P(x) if x is not None else None
        return lib.vvb_amvr_refine(hh, org_plane, ref_plane, q(pu), q(m), q(a), q(b), n, w, h, ctypes.byref(p) if p is not None else None, q(o))
    assert call() == L.VVB_OK
    for kw in (dict(pu=None), dict(m=None), dict(a=None), dict(b=None), dict(o=None), dict(p=None), dict(n=-1), dict(org_plane=7), dict(ref_plane=-1)):
        assert call(**kw) == L.VVB_ERR_ARG, kw
    ap = lambda **k: eng.amvr_par(**{**dict(lambda_=LAM, dfunc=V.DF_HAD, imv=1, mvp_bits=(1, 1), pic_w=W, pic_h=H, ctu_size=CTU), **k})
    for p in (ap(imv=-1), ap(imv=4), ap(lambda_=-1.0), ap(lambda_=float('nan')), ap(ctu_size=96), ap(pic_w=0), ap(ifp_lines=-1)):
        assert call(p=p) == L.VVB_ERR_ARG
    for p in (ap(imv=0), ap(imv=3), ap(dfunc=V.DF_SSE), ap(dfunc=V.DF_HAD_2SAD)):
        assert call(p=p) == L.VVB_ERR_UNSUPPORTED
    for (w, h) in ((2, 8), (256, 16), (12, 16)):
        assert call(w=w, h=h) == L.VVB_ERR_UNSUPPORTED, (w, h)
    # the member's CHECKs and positions: VVB_ERR_ARG from the host call, the sentinel from the _dev twin
    broken = []
    for f, v in (('num_cand', 0), ('num_cand', 3), ('mvp_idx', 2), ('mvp_idx', -1), ('cand_hor', 2), ('cand_ver', -6), ('pred', 1), ('x', -4), ('y', H)):
        a2, p2 = amvp.copy(), pus.copy()
        if f in ('x', 'y'):
            p2[f][1] = v
        elif f == 'pred':
            p2['pred_hor'][1] += v
        elif f.startswith('cand'):
            a2[f][1, 1] += v                                          # the other candidate: cBaseMvd[1] is checked whatever num_cand says
        else:
            a2[f][1] = v
        assert call(pu=p2, a=a2) == L.VVB_ERR_ARG, f
        broken.append((p2, a2))
    vp = ctypes.c_void_p
    for p2, a2 in broken:
        d_p, d_m, d_a, d_b = _dev(p2), _dev(mv), _dev(a2), _dev(bits)
        d_o = torch.full((4 * V.AMVR_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        assert lib.vvb_amvr_refine_dev(hh, 0, 1, vp(d_p.data_ptr()), vp(d_m.data_ptr()), vp(d_a.data_ptr()), vp(d_b.data_ptr()), 4, 16, 16, ctypes.byref(par),
                                       vp(d_o.data_ptr())) == L.VVB_OK
        eng.synchronize()
        dv = _host(d_o, V.AMVR_BEST_DT)
        assert got(dv[1]) == (0, 0, -1, 0, M64, M64)
        assert dv[[0, 2, 3]].tobytes() == eng.amvr_refine(0, 1, pus[[0, 2, 3]], mv[[0, 2, 3]], amvp[[0, 2, 3]], bits[[0, 2, 3]], 16, 16, par).tobytes()
    before = eng.launches
    assert call(n=0) == L.VVB_OK and eng.launches == before
    eng.upload_plane(2, cur, W, H, M, bit_depth=13)
    assert call(ref_plane=2) == L.VVB_ERR_UNSUPPORTED and call(org_plane=2) == L.VVB_ERR_UNSUPPORTED
    eng.free_plane(2)

    # the bi call: its own table, then the member's CHECKs, then n == 0
    bamvp = make_amvp(5, 2, 1, 4, rs)
    bpus, cands = bi_pus(16, 16, rs, bamvp)
    bamvp = bamvp[:len(bpus)]
    pred = B._pred_blocks(oth, bpus, 16, 16, rs)
    bp = lambda **k: eng.bi_par(**{**dict(lambda_=LAM, search_range=4, pic_w=W, pic_h=H, ctu_size=CTU, dfunc=V.DF_HAD, imv=1), **k})
    mb = np.array((1, 1), dtype=np.uint32)
    io, bo = np.zeros(len(bpus), dtype=V.TZ_BEST_DT), np.zeros(len(bpus), dtype=V.AMVR_BEST_DT)

    def bcall(pu=bpus, a=bamvp, n=len(bpus), p=bp(), m=mb, c=cands, nc=len(cands), pr=pred, i=io, o=bo, w=16, h=16, ref_plane=1):
        q = lambda x: P(x) if x is not None else None
        return lib.vvb_bipred_amvr_search(hh, 0, ref_plane, q(pu), q(a), n, w, h, ctypes.byref(p) if p is not None else None, q(m), q(c) if nc else None, nc,
                                          q(pr), q(i), q(o))
    assert bcall() == L.VVB_OK and bcall(i=None) == L.VVB_OK
    for kw in (dict(pu=None), dict(a=None), dict(p=None), dict(m=None), dict(pr=None), dict(o=None), dict(n=-1), dict(nc=-1), dict(c=None)):
        assert bcall(**kw) == L.VVB_ERR_ARG, kw
    for p in (bp(imv=4), bp(imv=-1), bp(ref_list=2), bp(search_range=9), bp(lambda_=float('inf'))):
        assert bcall(p=p) == L.VVB_ERR_ARG
    for p in (bp(imv=0), bp(imv=3), bp(dfunc=V.DF_SSE), bp(lambda_=1e30)):
        assert bcall(p=p) == L.VVB_ERR_UNSUPPORTED
    assert bcall(p=bp(fast_sub_pel=7, reduce_tap=-3)) == L.VVB_OK          # ignored
    for (w, h) in ((4, 8), (8, 4), (4, 4)):
        assert bcall(w=w, h=h) == L.VVB_ERR_UNSUPPORTED
    for f, v in (('num_cand', 0), ('mvp_idx', 2), ('cand_hor', 1), ('pred', 1), ('bcw_idx', 5), ('x', -4)):
        a2, p2 = bamvp.copy(), bpus.copy()
        if f in ('x', 'bcw_idx'):
            p2[f][1] = v
        elif f == 'pred':
            p2['pred_ver'][1] += v
        elif f == 'cand_hor':
            a2[f][1, 0] += v
        else:
            a2[f][1] = v
        assert bcall(pu=p2, a=a2) == L.VVB_ERR_ARG, f
    before = eng.launches
    assert bcall(n=0) == L.VVB_OK and eng.launches == before
    assert bcall(p=bp(imv=0), n=0) == L.VVB_ERR_UNSUPPORTED                 # vvb_bipred_search's branch, whatever n

    # the reference margin at the clipMv box's need and one pel less, per side: a PU at the left / top / right / bottom edge whose vector points beyond the
    # far end of the box; for the right and bottom sides a reference plane narrower / lower than the picture, so that side's need is the largest
    w = h = 16
    curp = np.pad(cur, 60, mode='edge'); MP = M + 60
    for side in range(4):
        x, y = (0, 64) if side == 0 else (64, 0) if side == 1 else (W - w, 64) if side == 2 else (64, H - h)
        vec = [(-200, 0), (0, -200), (200, 0), (0, 200)][side]
        rw, rh = (W - 150, H) if side == 2 else (W, H - 150) if side == 3 else (W, H)
        need = CTU + 7 if side < 2 else W + w + 7 - rw if side == 2 else H + h + 7 - rh
        for mg, ok in ((need, True), (need - 1, False)):
            eng.upload_plane(4, np.ascontiguousarray(curp[MP - mg:MP + rh + mg, MP - mg:MP + rw + mg]), rw, rh, mg)
            a1 = make_amvp(1, 2, 0, 4, rs)
            p1 = tz_pus(w, h, 1, rs, a1); p1['x'] = x; p1['y'] = y
            m1 = np.zeros(1, dtype=V.TZ_BEST_DT); m1['mv_hor'] = vec[0]; m1['mv_ver'] = vec[1]
            o1 = np.zeros(1, dtype=V.AMVR_BEST_DT)
            assert lib.vvb_amvr_refine(hh, 0, 4, P(p1), P(m1), P(a1), P(bits[:1]), 1, w, h, ctypes.byref(par), P(o1)) == (L.VVB_OK if ok else L.VVB_ERR_UNSUPPORTED)
            d_o = torch.full((V.AMVR_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
            d_p, d_m, d_a, d_b = _dev(p1), _dev(m1), _dev(a1), _dev(bits[:1])
            torch.cuda.synchronize()
            rc = lib.vvb_amvr_refine_dev(hh, 0, 4, vp(d_p.data_ptr()), vp(d_m.data_ptr()), vp(d_a.data_ptr()), vp(d_b.data_ptr()), 1, w, h, ctypes.byref(par),
                                         vp(d_o.data_ptr()))
            assert rc == (L.VVB_OK if ok else L.VVB_ERR_UNSUPPORTED), (side, mg)
            eng.synchronize()
            if ok:
                assert _host(d_o, V.AMVR_BEST_DT).tobytes() == o1.tobytes() and int(o1['cost'][0]) < 1 << 63
            bp1 = np.zeros(1, dtype=V.BI_PU_DT); bp1['x'] = x; bp1['y'] = y; bp1['bcw_idx'] = 2
            bp1['pred_hor'] = p1['pred_hor']; bp1['pred_ver'] = p1['pred_ver']
            rcb = lib.vvb_bipred_amvr_search(hh, 0, 4, P(bp1), P(a1), 1, w, h, ctypes.byref(bp()), P(mb), None, 0, P(pred[:1].copy()), None, P(o1))
            assert rcb == L.VVB_ERR_UNSUPPORTED if not ok else rcb in (L.VVB_OK, L.VVB_ERR_UNSUPPORTED), (side, mg, rcb)
    # the bi call's integer stage keeps vvb_bipred_search's per-PU rule: at a margin of ctu_size + 11 (enough for the refinement, one short of the integer
    # stage's ctu_size + 12 for a start clipped to the left end of the box) the host call refuses the PU and the _dev twin gives it the sentinel
    eng.upload_plane(4, np.ascontiguousarray(curp[MP - CTU - 11:MP + H + CTU + 11, MP - CTU - 11:MP + W + CTU + 11]), W, H, CTU + 11)
    b2 = bpus[:2].copy(); a2 = bamvp[:2].copy()
    b2['x'][0] = 0; b2['y'][0] = 64; b2['start_hor'][0] = -60000; b2['start_ver'][0] = 0; b2['cand_first'] = 0; b2['cand_count'] = 0
    pr2 = np.ascontiguousarray(pred[:2])
    assert lib.vvb_bipred_amvr_search(hh, 0, 4, P(b2), P(a2), 2, 16, 16, ctypes.byref(bp()), P(mb), None, 0, P(pr2), None, P(bo[:2].copy())) == L.VVB_ERR_UNSUPPORTED
    d_p, d_a, d_pr = _dev(b2), _dev(a2), torch.from_numpy(pr2).cuda()
    d_i = torch.full((2 * V.TZ_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
    d_o = torch.full((2 * V.AMVR_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    assert lib.vvb_bipred_amvr_search_dev(hh, 0, 4, vp(d_p.data_ptr()), vp(d_a.data_ptr()), 2, 16, 16, ctypes.byref(bp()), P(mb), None, 0, vp(d_pr.data_ptr()),
                                          vp(d_i.data_ptr()), vp(d_o.data_ptr())) == L.VVB_OK
    eng.synchronize()
    di, do = _host(d_i, V.TZ_BEST_DT), _host(d_o, V.AMVR_BEST_DT)
    assert (int(di['mv_hor'][0]), int(di['mv_ver'][0])) == (-(1 << 30), -(1 << 30)) and got(do[0]) == (0, 0, -1, 0, M64, M64)
    hi, ho = eng.bipred_amvr_search(0, 4, b2[1:], a2[1:], 16, 16, bp(), (1, 1), pr2[1:])
    assert di[1:].tobytes() == hi.tobytes() and do[1:].tobytes() == ho.tobytes()
    eng.free_plane(4)


def test_compiler_report():
    """-Xptxas -v shows no spills in amvr_refine_kernel, and the kernels whose distortion loaders gained the shared-memory source keep their SASS
    (tests/golden/dist_kernels.sass.sha256: cost_pattern_kernel, dist_list_kernel and dist_pool_kernel as built before the change)"""
    import os, re, shutil, subprocess
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'vvenc_b200', 'csrc')
    log = open(os.path.join(csrc, 'build.log')).read()
    blocks = re.findall(r"Compiling entry function '(\w+)'.*?\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log, re.S)
    mine = [b for b in blocks if 'amvr_refine_kernel' in b[0]]
    assert len(mine) == 8, mine                                  # <4, 8, 16, 32> x <AmvrOrgPlane, AmvrTarget>
    assert all(st == '0' and ld == '0' for (_, _, st, ld) in mine), mine
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    sass = subprocess.run([cuobjdump, '-sass', os.path.join(csrc, 'libvvenc_b200.so')], capture_output=True, text=True, check=True).stdout
    golden = [l.split() for l in open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dist_kernels.sass.sha256')).read().splitlines() if l.strip()]
    assert len(golden) >= 3
    for digest, name in golden:
        assert B.sass_digest(sass, re.escape(name)) == digest, name
