"""vvb_bipred_search, the bi-predictive branch of InterSearch::xMotionEstimation on the device, against the reference's members stage by stage (the replay and
SIMD checks run on the CPU, the rest need -m gpu).

There is no member for the whole branch.  The target 2 * org - pred has no probe entry either; its restatement here is AreaBuf::removeHighFreq's one line
(Buffer.h:474-475): dst = 2 * dst - src, ClipPel'd when m_bClipForBiPredMeEnabled.  refshim_pattern_search_member and refshim_frac_search_member copy only the
PU's own w x h block of the original plane, so a plane that holds each PU's target at its position serves any set of non-overlapping PUs.
  * start: a Python replay of :2051-2094 (xClipMvSearch with ifp_lines, changePrecision, the repeat test, the strict `<` on the probe's own SAD and MV cost,
    xSetSearchRange) gives the window; the clip arithmetic is test_gpu_tz_search's Replay.clip, which that file pins to xTZSearch.
  * integer: refshim_pattern_search_member over the replayed window equals the device's vector and uiBestSad.
  * fraction: refshim_frac_search_member at the member's integer vector equals the device's offsets and ruiCost.
  * final: the formula of :2117-2124 restated in IEEE double, getCost cross-checked against refshim_mv_cost.
"""
import ctypes
import itertools
import math

import numpy as np
import pytest

from _libs import have_ref, refshim, P, PO
from test_gpu_frac_search import content
from test_gpu_tz_search import Replay, _rshift

pytestmark = pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
gpu = pytest.mark.gpu

LAM = 57.25
SHAPES = [(8, 8), (16, 16), (32, 32), (64, 64), (128, 128), (128, 64), (64, 128), (16, 8), (8, 16), (32, 8), (8, 32), (64, 16)]
SETTINGS = list(itertools.product((1, 2, 3), (0, 1, 2), (0, 3), (0, 1, 2), (0, 1), (0, 1)))   # dfunc, reduce_tap, imv, fast_sub_pel, clip, ref_list
RANGES = (0, 1, 4, 8)
BCW = (-2, 3, 4, 5, 10)
W, H, CTU = 320, 576, 128            # five CTU rows: xClipMvSearch's ifp_lines clip applies to the PUs of the first rows
M = CTU + 12


def ref_setup(R):
    R.refshim_frac_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    R.refshim_pattern_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    R.refshim_tz_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double] + [ctypes.c_int] * 7 + [ctypes.c_void_p]
    R.refshim_dist.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_int] * 4
    R.refshim_dist.restype = ctypes.c_uint64
    R.refshim_mv_cost.argtypes = [ctypes.c_double] + [ctypes.c_int] * 6
    R.refshim_mv_cost.restype = ctypes.c_uint64
    R.refshim_mv_bits.argtypes = [ctypes.c_int] * 6
    R.refshim_mv_bits.restype = ctypes.c_uint32
    R.refshim_set_simd(b'AVX2')
    return R


@pytest.fixture(scope="module")
def ref():
    return ref_setup(refshim())


@pytest.fixture(scope="module")
def eng():
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def target(o, p, clip, bd):
    """AreaBuf::removeHighFreq (Buffer.h:474-475), restated: 2 * org - pred, ClipPel'd with clip"""
    t = 2 * o.astype(np.int32) - p.astype(np.int32)
    return np.clip(t, 0, (1 << bd) - 1) if clip else t


def u64(v):
    """(Distortion) of a double as the x86-64 encoder converts it: comisd against 2^63, cvttsd2si below, cvttsd2si of v - 2^63 with the top bit flipped at or
    above; cvttsd2si gives 0x8000000000000000 for NaN and outside the int64 range"""
    def cvtt(x):
        return int(x) & ((1 << 64) - 1) if -2.0 ** 63 <= x < 2.0 ** 63 else 1 << 63
    return cvtt(v - 2.0 ** 63) ^ (1 << 63) if v >= 2.0 ** 63 else cvtt(v)


def get_cost(lam, b):
    return u64(math.sqrt(lam) * float(b))


def final(lam, frac_cost, qx, qy, pred, imv_shift, bits, bcw_idx, ref_list):
    """InterSearch.cpp:2117-2124 restated (quarter-pel rcMv in, ruiBits and ruiCost out)"""
    eg = lambda v: 1 + 2 * (((2 * -v + 1) if v <= 0 else 2 * v).bit_length() - 1)
    mv_bits = eg((qx - pred[0]) >> imv_shift) + eg((qy - pred[1]) >> imv_shift)
    rb = (bits + mv_bits) & 0xffffffff
    w = 0.5 if bcw_idx == 2 else abs((8 - BCW[bcw_idx] if ref_list == 0 else BCW[bcw_idx]) / 8.0)
    return rb, u64(math.floor(w * (float(frac_cost) - float(get_cost(lam, mv_bits)))) + float(get_cost(lam, rb))), mv_bits


class BiReplay(Replay):
    """the start selection and the window of :2051-2094 on the probe's own SAD and MV cost over a target plane"""

    def __init__(self, R, tgt, cur, S, bd, w, h, mode, rng, ifp, imv_shift, pw, ph):
        super().__init__(R, tgt, cur, S, M, bd, w, h, mode, rng, CTU, (0, 0, 0, 0), pw, ph, ifp, imv_shift)

    def window(self, x0, y0, start, pred, cands):
        hmin, hmax, vmin, vmax = self.clip(x0, y0, True)
        cl = lambda v, lo, hi: min(hi, max(lo, v))
        o = self.base + y0 * self.S + x0

        def cost(mv):
            x, y = _rshift(cl(mv[0], hmin, hmax), 4), _rshift(cl(mv[1], vmin, vmax), 4)
            sad = int(self.R.refshim_dist(1, 1, PO(self.org, o), self.S, PO(self.cur, o + y * self.S + x), self.S, self.w, self.h, self.bd, self.sub))
            return sad + int(self.R.refshim_mv_cost(LAM, x, y, pred[0], pred[1], 2, self.imv))
        best, init = cost(start), start
        for i, c in enumerate(cands):
            if c in cands[:i]:
                continue
            v = cost(c)
            if v < best:
                best, init = v, c
        # xSetSearchRange: top left by clipMv, bottom right by xClipMvSearch
        chmin, chmax, cvmin, cvmax = self.clip(x0, y0, False)
        px, py = cl(init[0], chmin, chmax), cl(init[1], cvmin, cvmax)
        r = self.rng << 4
        win = (_rshift(cl(px - r, chmin, chmax), 4), _rshift(cl(px + r, hmin, hmax), 4),
               _rshift(cl(py - r, cvmin, cvmax), 4), _rshift(cl(py + r, vmin, vmax), 4))
        STATS['ifp_clipped'] += win[3] != _rshift(cl(py + r, cvmin, cvmax), 4)
        STATS['empty'] += win[0] > win[1] or win[2] > win[3]
        return win


STATS = {'ifp_clipped': 0, 'empty': 0}       # windows whose bottom the ifp_lines clip moved, and empty windows (xPatternSearch then answers (0, 0))


def layout(w, h, k, rs):
    """k non-overlapping PU positions of one shape"""
    cells = [(x, y) for y in range(0, H - h + 1, h) for x in range(0, W - w + 1, w)]
    idx = rs.choice(len(cells), size=min(k, len(cells)), replace=False)
    return [cells[i] for i in idx]


def make_pus(w, h, k, rs, ncand_max=4):
    import vvenc_b200 as V
    pos = layout(w, h, k, rs)
    pus = np.zeros(len(pos), dtype=V.BI_PU_DT)
    cands = []
    for i, (x, y) in enumerate(pos):
        pus['x'][i] = x; pus['y'][i] = y
        far = rs.randint(4) == 0             # beyond a picture edge: clipped by xClipMvSearch
        lim = 4000 if far else 20 * 16
        pus['start_hor'][i] = rs.randint(-lim, lim + 1); pus['start_ver'][i] = rs.randint(-lim, lim + 1)
        pus['pred_hor'][i] = rs.randint(-200, 201); pus['pred_ver'][i] = rs.randint(-200, 201)
        nc = rs.randint(0, ncand_max + 1)
        pus['cand_first'][i] = len(cands); pus['cand_count'][i] = nc
        for j in range(nc):
            if j and rs.randint(3) == 0:
                cands.append(cands[-1 - rs.randint(j)])                           # a repeat of an earlier candidate
            else:
                cands.append((int(rs.randint(-lim, lim + 1)), int(rs.randint(-lim, lim + 1))))
        pus['bits'][i] = rs.randint(0, 40)
        pus['bcw_idx'][i] = i % 5
    return pus, np.array(cands, dtype=np.int32).reshape(-1, 2)


def check_call(R, org, cur, S, bd, pus, cands, pred, w, h, par, dev):
    """each stage of dev (BI_BEST_DT) against its member; returns the number of PUs that differ"""
    pw, ph = par.pic_w, par.pic_h
    clip, imv_shift, rl = bool(par.clip), 1 if par.imv == 3 else 0, par.ref_list
    tgt = org.astype(np.int32).copy()
    base = M * S + M
    for i in range(len(pus)):
        x, y = int(pus['x'][i]), int(pus['y'][i])
        tgt[M + y:M + y + h, M + x:M + x + w] = target(org[M + y:M + y + h, M + x:M + x + w], pred[i], clip, bd)
    tgt = np.ascontiguousarray(tgt, dtype=np.int16)
    rp = BiReplay(R, tgt, cur, S, bd, w, h, par.sub_shift_mode, par.search_range, par.ifp_lines, imv_shift, pw, ph)
    bad = 0
    for i in range(len(pus)):
        x, y = int(pus['x'][i]), int(pus['y'][i]); pred_q = (int(pus['pred_hor'][i]), int(pus['pred_ver'][i]))
        cf, cc = int(pus['cand_first'][i]), int(pus['cand_count'][i])
        cl = [tuple(int(v) for v in c) for c in cands[cf:cf + cc]]
        l, r, t, b = rp.window(x, y, (int(pus['start_hor'][i]), int(pus['start_ver'][i])), pred_q, cl)
        blk = np.array([[x, y, w, h, l, r, t, b, pred_q[0], pred_q[1]]], dtype=np.int32)
        o = np.zeros(4, dtype=np.int32)
        R.refshim_pattern_search_member(1, PO(tgt, base), S, PO(cur, base), S, P(blk), 1, bd, par.sub_shift_mode, LAM, 2, imv_shift, P(o))
        mx, my = int(o[0]), int(o[1]); ibest = (int(o[2]) & 0xffffffff) | ((int(o[3]) & 0xffffffff) << 32)
        ruisad = (ibest - int(R.refshim_mv_cost(LAM, mx, my, pred_q[0], pred_q[1], 2, imv_shift))) & ((1 << 64) - 1)
        if par.fast_sub_pel == 2:
            half, qter, fcost = (0, 0), (0, 0), ruisad
        else:
            fb = np.array([[x, y, w, h, mx, my, pred_q[0], pred_q[1]]], dtype=np.int32)
            fo = np.zeros(6, dtype=np.int32)
            R.refshim_frac_search_member(1, PO(tgt, base), S, PO(cur, base), S, P(fb), 1, bd, LAM, par.reduce_tap, par.dfunc - 1, int(par.imv == 3), par.fast_sub_pel, P(fo))
            half, qter, fcost = (int(fo[0]), int(fo[1])), (int(fo[2]), int(fo[3])), (int(fo[4]) & 0xffffffff) | ((int(fo[5]) & 0xffffffff) << 32)
        qx, qy = 4 * mx + 2 * half[0] + qter[0], 4 * my + 2 * half[1] + qter[1]
        bits, cost, mv_bits = final(LAM, fcost, qx, qy, pred_q, imv_shift, int(pus['bits'][i]), int(pus['bcw_idx'][i]), rl)
        assert get_cost(LAM, mv_bits) == int(R.refshim_mv_cost(LAM, qx, qy, pred_q[0], pred_q[1], 0, imv_shift))
        d = dev[i]
        got = ((int(d['int_hor']), int(d['int_ver'])), int(d['int_best']), (int(d['half_hor']), int(d['half_ver'])), (int(d['qter_hor']), int(d['qter_ver'])),
               int(d['frac_cost']), (int(d['mv_hor']), int(d['mv_ver'])), int(d['bits']), int(d['cost']))
        exp = ((mx, my), ibest, half, qter, fcost, (4 * qx, 4 * qy), bits, cost)
        bad += got != exp
    return bad


def test_simd_members_agree_on_extreme_targets(ref):
    """the scalar (opt 0) and AVX2 (opt 1) SAD and Hadamard members on targets at both ends of their range: org = max, pred = 0 and org = 0, pred = max"""
    for bd in (8, 10):
        mx = (1 << bd) - 1
        for (w, h) in SHAPES:
            rs = np.random.RandomState(w * h + bd)
            cur = np.ascontiguousarray(rs.randint(0, mx + 1, size=(h, w)), dtype=np.int16)
            for o, p in ((mx, 0), (0, mx)):
                t = np.ascontiguousarray(target(np.full((h, w), o), np.full((h, w), p), False, bd), dtype=np.int16)
                for df in (1, 2):
                    a = int(ref.refshim_dist(0, df, P(t), w, P(cur), w, w, h, bd, 0))
                    b = int(ref.refshim_dist(1, df, P(t), w, P(cur), w, w, h, bd, 0))
                    assert a == b, (bd, w, h, o, p, df, a, b)
                    if df == 1:
                        assert a == int(np.abs(t.astype(np.int64) - cur).sum())


def _planes(bd, seed):
    org, cur, _ = content(W, H, M, bd, seed)
    oth, _, _ = content(W, H, M, bd, seed + 1)
    return org, cur, oth


def _pred_blocks(oth, pus, w, h, rs):
    """the other list's prediction: a block of a second plane near the PU"""
    out = np.zeros((len(pus), h, w), dtype=np.int16)
    for i in range(len(pus)):
        x, y = int(pus['x'][i]) + rs.randint(-3, 4) + M, int(pus['y'][i]) + rs.randint(-3, 4) + M
        out[i] = oth[y:y + h, x:x + w]
    return out


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_bipred_search_equals_the_members(eng, ref, bd):
    import vvenc_b200 as V
    org, cur, oth = _planes(bd, 500 + bd)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M, bit_depth=bd); eng.upload_plane(1, cur, W, H, M, bit_depth=bd)
    bad = []; n = 0; seen = set(); maxc = 0
    STATS.update(ifp_clipped=0, empty=0)
    for si, (w, h) in enumerate(SHAPES):
        for k, (dfunc, rt, imv, fast, clip, rl) in enumerate(SETTINGS):
            if k % 4 != si % 4:                  # each setting with three shapes per bit depth
                continue
            rs = np.random.RandomState(1000 * bd + 37 * si + k)
            rng = RANGES[(k // 4 + si) % 4]
            pus, cands = make_pus(w, h, 5, rs, 15 if k % 3 == 1 else 4)        # up to m_uniMvListMaxSize candidates
            if k % 3:
                pus['start_ver'][0] = 60000            # below the ifp_lines bound: the window around the clipMv'd start can be empty
            pred = _pred_blocks(oth, pus, w, h, rs)
            par = eng.bi_par(LAM, rng, W, H, CTU, dfunc, ref_list=rl, clip=clip, imv=imv, fast_sub_pel=fast, reduce_tap=rt,
                             sub_shift_mode=k % 3, ifp_lines=k % 3)
            if dfunc == 1 and fast == 1 and w >= 64:        # outside the domain: the member's early-exit partial sums enter its pattern id
                with pytest.raises(V.VvbError):
                    eng.bipred_search(0, 1, pus, w, h, par, pred, cands)
                continue
            dev = eng.bipred_search(0, 1, pus, w, h, par, pred, cands)
            n += len(pus); seen.add((dfunc, rt, imv, fast, clip, rl, rng)); maxc = max(maxc, int(pus['cand_count'].max()))
            if check_call(ref, org, cur, S, bd, pus, cands, pred, w, h, par, dev):
                bad.append((w, h, dfunc, rt, imv, fast, clip, rl, rng))
    assert len({s[:6] for s in seen}) == len(SETTINGS) and {s[6] for s in seen} == set(RANGES)
    assert maxc == 15 and STATS['ifp_clipped'] > 10 and STATS['empty'] > 0, (maxc, STATS)
    assert bad == [], (len(bad), bad[:10])


@gpu
def test_chain_tz_frac_bipred_on_the_device(eng, ref):
    """vvb_tz_search_dev -> vvb_frac_search_dev -> start vectors -> vvb_bipred_search_dev for every PU of 8x8..128x128 on a 1920x1080 10-bit pair, against the
    members in the same order; the host-buffer call equals the _dev call"""
    import torch
    import vvenc_b200 as V
    PW, PH, RNG = 1920, 1080, 64
    MG = CTU + 12
    org, cur, _ = content(PW, PH, MG, 10, 91)
    oth, _, _ = content(PW, PH, MG, 10, 92)
    S = PW + 2 * MG; base = MG * S + MG
    eng.upload_plane(0, org, PW, PH, MG); eng.upload_plane(1, cur, PW, PH, MG)
    me = eng.me_par(LAM, 2, 0)
    tz = eng.tz_par(RNG, PW, PH, CTU, extended=False, fast=True, integer_et=False, first_search_stop=True)
    fpar = eng.frac_par(LAM, V.DF_HAD, 2, False, 1)
    bpar = eng.bi_par(LAM, 4, PW, PH, CTU, V.DF_HAD, ref_list=1, fast_sub_pel=1)
    rs = np.random.RandomState(6)
    vp = ctypes.c_void_p
    for s in (8, 16, 32, 64, 128):
        ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
        pus = np.zeros(xs.size, dtype=V.TZ_PU_DT)
        pus['x'] = xs.ravel(); pus['y'] = ys.ravel()
        pus['start_hor'] = rs.randint(-40 * 16, 40 * 16 + 1, size=xs.size); pus['start_ver'] = rs.randint(-24 * 16, 24 * 16 + 1, size=xs.size)
        q = lambda v: np.where(v >= 0, (v + 1) >> 2, (v + 2) >> 2)
        pus['pred_hor'] = q(pus['start_hor'].astype(np.int64)); pus['pred_ver'] = q(pus['start_ver'].astype(np.int64))
        pred = np.stack([oth[MG + y + 2:MG + y + 2 + s, MG + x - 1:MG + x - 1 + s] for x, y in zip(pus['x'], pus['y'])]).astype(np.int16)
        d_pus = torch.from_numpy(np.frombuffer(pus.tobytes(), dtype=np.uint8).copy()).cuda()
        d_mv = torch.zeros(len(pus) * V.TZ_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        d_fr = torch.zeros(len(pus) * V.FRAC_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        eng._chk(eng.lib.vvb_tz_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), len(pus), s, s, ctypes.byref(me), ctypes.byref(tz), None, 0, vp(d_mv.data_ptr())))
        eng._chk(eng.lib.vvb_frac_search_dev(eng.h, 0, 1, vp(d_pus.data_ptr()), vp(d_mv.data_ptr()), len(pus), s, s, ctypes.byref(fpar), vp(d_fr.data_ptr())))
        eng.synchronize()                       # the torch kernels below run on torch's stream, not on the context's
        # start vectors: rcMv of the uni search in internal units, on the device
        mvt = d_mv.view(torch.int32).view(-1, 8)[:, :2]
        frt = d_fr.view(torch.int16).view(-1, 8)[:, :4].to(torch.int32)
        start = ((mvt * 4 + frt[:, 0:2] * 2 + frt[:, 2:4]) * 4)
        bi = np.zeros(len(pus), dtype=V.BI_PU_DT)
        for f in ('x', 'y', 'pred_hor', 'pred_ver'):
            bi[f] = pus[f]
        bi['bits'] = 7; bi['bcw_idx'] = np.arange(len(pus)) % 5
        d_bi = torch.from_numpy(np.frombuffer(bi.tobytes(), dtype=np.uint8).copy()).cuda().view(len(pus), 36)
        d_bi[:, 8:16] = start.contiguous().view(torch.uint8).view(len(pus), 8)
        d_pred = torch.from_numpy(pred).cuda()
        d_out = torch.zeros(len(pus) * V.BI_BEST_DT.itemsize, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        eng._chk(eng.lib.vvb_bipred_search_dev(eng.h, 0, 1, vp(d_bi.data_ptr()), len(pus), s, s, ctypes.byref(bpar), None, 0, vp(d_pred.data_ptr()), vp(d_out.data_ptr())))
        eng.synchronize()
        dev = np.frombuffer(d_out.cpu().numpy().tobytes(), dtype=V.BI_BEST_DT)
        # the members in the same order
        blk = np.zeros((len(pus), 6), dtype=np.int32)
        blk[:, 0] = pus['x']; blk[:, 1] = pus['y']; blk[:, 2] = s; blk[:, 3] = s; blk[:, 4] = pus['start_hor']; blk[:, 5] = pus['start_ver']
        tzm = np.zeros((len(pus), 8), dtype=np.int64)
        assert ref.refshim_tz_search_member(1, PO(org, base), S, PO(cur, base), S, PW, PH, MG, P(blk), len(blk), 10, 0, LAM, RNG, CTU, 0, 1, 0, 1, 0, P(tzm)) == 0
        fb = np.zeros((len(pus), 8), dtype=np.int32)
        fb[:, :4] = blk[:, :4]; fb[:, 4] = tzm[:, 0]; fb[:, 5] = tzm[:, 1]; fb[:, 6] = pus['pred_hor']; fb[:, 7] = pus['pred_ver']
        fo = np.zeros((len(pus), 6), dtype=np.int32)
        ref.refshim_frac_search_member(1, PO(org, base), S, PO(cur, base), S, P(fb), len(fb), 10, LAM, 2, 1, 0, 1, P(fo))
        bi['start_hor'] = ((tzm[:, 0] * 4 + fo[:, 0] * 2 + fo[:, 2]) * 4); bi['start_ver'] = ((tzm[:, 1] * 4 + fo[:, 1] * 2 + fo[:, 3]) * 4)
        sub = np.arange(len(pus)) if s >= 64 else rs.choice(len(pus), size=300, replace=False)
        # non-overlapping by construction (a grid of s x s cells): one target plane serves them all
        assert check_call(ref, org, cur, S, 10, bi[sub], np.zeros((0, 2), np.int32), pred[sub], s, s, bpar, dev[sub]) == 0, s
        host = eng.bipred_search(0, 1, bi, s, s, bpar, pred)
        assert host.tobytes() == dev.tobytes(), s


@gpu
def test_bipred_search_admission(eng, ref):
    import torch
    import vvenc_b200 as V
    import vvenc_b200._lib as L
    bd = 10
    org, cur, oth = _planes(bd, 700)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M); eng.upload_plane(1, cur, W, H, M)
    rs = np.random.RandomState(3)
    pus, cands = make_pus(16, 16, 4, rs)
    pred = _pred_blocks(oth, pus, 16, 16, rs)
    par = eng.bi_par(LAM, 4, W, H, CTU, V.DF_HAD)
    out = np.zeros(len(pus), dtype=V.BI_BEST_DT)
    lib, h = eng.lib, eng.h

    def call(pu=pus, n=len(pus), w=16, hh=16, p=par, c=cands, nc=len(cands), pr=pred, o=out, org_plane=0, ref_plane=1):
        return lib.vvb_bipred_search(h, org_plane, ref_plane, P(pu) if pu is not None else None, n, w, hh, ctypes.byref(p) if p is not None else None,
                                     P(c) if c is not None and nc else None, nc, P(pr) if pr is not None else None, P(o) if o is not None else None)
    assert call() == L.VVB_OK
    for kw in (dict(pu=None), dict(p=None), dict(pr=None), dict(o=None), dict(n=-1), dict(nc=-1), dict(c=None), dict(org_plane=7), dict(ref_plane=-1)):
        assert call(**kw) == L.VVB_ERR_ARG, kw
    bp = lambda **k: eng.bi_par(**{**dict(lambda_=LAM, search_range=4, pic_w=W, pic_h=H, ctu_size=CTU, dfunc=V.DF_HAD), **k})
    for p in (bp(search_range=-1), bp(search_range=9), bp(sub_shift_mode=3), bp(ctu_size=96), bp(ref_list=2), bp(fast_sub_pel=3), bp(reduce_tap=3),
              bp(imv=4), bp(imv=-1), bp(lambda_=-1.0), bp(lambda_=float('nan')), bp(lambda_=float('inf')), bp(ifp_lines=-1)):
        assert call(p=p) == L.VVB_ERR_ARG
    for p in (bp(imv=1), bp(imv=2), bp(dfunc=V.DF_SSE), bp(dfunc=V.DF_HAD_2SAD)):
        assert call(p=p) == L.VVB_ERR_UNSUPPORTED
    assert call(p=bp(dfunc=V.DF_SAD, fast_sub_pel=1), w=64, hh=16) == L.VVB_ERR_UNSUPPORTED
    for (w, hh) in ((4, 4), (4, 8), (8, 4), (256, 16), (12, 16)):
        assert call(w=w, hh=hh) == L.VVB_ERR_UNSUPPORTED, (w, hh)
    assert call(p=bp(ctu_size=16, search_range=4), w=32, hh=16) == L.VVB_ERR_UNSUPPORTED
    for f, v in (('x', -4), ('y', H), ('cand_first', 1000), ('cand_count', -1), ('bcw_idx', 5)):
        p2 = pus.copy(); p2[f][1] = v
        assert call(pu=p2) == L.VVB_ERR_ARG, f
    before = eng.launches
    assert call(n=0) == L.VVB_OK and eng.launches == before
    eng.upload_plane(2, cur, W, H, M, bit_depth=13)
    assert call(ref_plane=2) == L.VVB_ERR_UNSUPPORTED and call(org_plane=2) == L.VVB_ERR_UNSUPPORTED
    eng.free_plane(2)

    # the read box at the margin and one pel beyond: a smaller reference margin, a PU at the left / top / right / bottom edge whose start is clipped to the
    # far end of xClipMvSearch's box; the window then reaches the box's end and the fractional stage 5 columns / 4 rows beyond it
    w = hh = 16
    for side in range(4):
        x, y = (0, 64) if side == 0 else (64, 0) if side == 1 else (W - w, 64) if side == 2 else (64, H - hh)
        st = [(-60000, 0), (0, -60000), (60000, 0), (0, 60000)][side]
        need = [CTU + 12, CTU + 11, w + 12, hh + 11][side]
        for mg, ok in ((need, True), (need - 1, False)):
            orgm = np.ascontiguousarray(org[M - mg:M + H + mg, M - mg:M + W + mg]); curm = np.ascontiguousarray(cur[M - mg:M + H + mg, M - mg:M + W + mg])
            eng.upload_plane(3, orgm, W, H, mg); eng.upload_plane(4, curm, W, H, mg)
            p1 = np.zeros(2, dtype=V.BI_PU_DT)
            p1['x'] = x; p1['y'] = y; p1['start_hor'] = st[0]; p1['start_ver'] = st[1]; p1['bcw_idx'] = 2; p1['pred_hor'] = 3; p1['pred_ver'] = -5
            p1['x'][1] = 32; p1['y'][1] = 32; p1['start_hor'][1] = 0; p1['start_ver'][1] = 0
            pr1 = np.ascontiguousarray(pred[:2])
            par1 = eng.bi_par(LAM, 4, W, H, CTU, V.DF_HAD, fast_sub_pel=0)
            o1 = np.zeros(2, dtype=V.BI_BEST_DT)
            rc = lib.vvb_bipred_search(h, 3, 4, P(p1), 2, w, hh, ctypes.byref(par1), None, 0, P(pr1), P(o1))
            assert rc == (L.VVB_OK if ok else L.VVB_ERR_UNSUPPORTED), (side, mg)
            d_pu = torch.from_numpy(np.frombuffer(p1.tobytes(), dtype=np.uint8).copy()).cuda()
            d_pr = torch.from_numpy(pr1).cuda()
            d_o = torch.full((2 * V.BI_BEST_DT.itemsize,), 0x55, dtype=torch.uint8, device='cuda')
            torch.cuda.synchronize()
            assert lib.vvb_bipred_search_dev(h, 3, 4, ctypes.c_void_p(d_pu.data_ptr()), 2, w, hh, ctypes.byref(par1), None, 0, ctypes.c_void_p(d_pr.data_ptr()),
                                             ctypes.c_void_p(d_o.data_ptr())) == L.VVB_OK
            eng.synchronize()
            dv = np.frombuffer(d_o.cpu().numpy().tobytes(), dtype=V.BI_BEST_DT)
            assert check_call(ref, orgm, curm, W + 2 * mg, bd, p1[1:], np.zeros((0, 2), np.int32), pr1[1:], w, hh, par1, dv[1:]) == 0 if mg == M else True
            if ok:
                assert o1.tobytes() == dv.tobytes()
            else:
                assert int(dv['cost'][0]) == int(dv['frac_cost'][0]) == int(dv['int_best'][0]) == (1 << 64) - 1
                assert int(dv['mv_hor'][0]) == int(dv['mv_ver'][0]) == int(dv['int_hor'][0]) == int(dv['bits'][0]) == 0
                assert int(dv['cost'][1]) < (1 << 63)
    for pl in (3, 4):
        eng.free_plane(pl)


@gpu
@pytest.mark.parametrize("dfunc", [2, 3])
def test_bipred_search_format_limits(eng, ref, dfunc):
    """128x128 at 12 bits with 2 * org - pred at both ends of its range (org 4095 / pred 0 -> 8190, org 0 / pred 4095 -> -4095) against a reference of 0 / 4095,
    so the SAD and the Hadamard sums are near their tops, and a lambda whose MV-rate table top fills 32 bits"""
    import vvenc_b200 as V
    bd, w, hh = 12, 128, 128
    rs = np.random.RandomState(62)
    mx = (1 << bd) - 1
    org = np.ascontiguousarray((rs.randint(0, 2, size=(H + 2 * M, W + 2 * M)) * mx).astype(np.int16))
    cur = np.ascontiguousarray((rs.randint(0, 2, size=org.shape) * mx).astype(np.int16))
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M, bit_depth=bd); eng.upload_plane(1, cur, W, H, M, bit_depth=bd)
    lam = (4294967295.0 / 79) ** 2 * 0.999
    pus = np.zeros(2, dtype=V.BI_PU_DT)
    pus['x'] = (0, W - w); pus['y'] = (0, H - hh); pus['start_hor'] = (-60000, 60000); pus['start_ver'] = (-60000, 60000)
    pus['pred_hor'] = (32767, -32768); pus['pred_ver'] = (32767, -32768); pus['bits'] = (0xfffffff0, 3); pus['bcw_idx'] = (4, 0)
    pred = np.ascontiguousarray(((1 - org[M:M + hh, M:M + w] // mx) * mx)[None].repeat(2, 0).astype(np.int16))
    for fast in (0, 1, 2):
        for clip in (0, 1):
            par = eng.bi_par(lam, 8, W, H, CTU, dfunc, clip=clip, fast_sub_pel=fast, sub_shift_mode=0)
            dev = eng.bipred_search(0, 1, pus, w, hh, par, pred)
            global LAM
            keep, LAM = LAM, lam
            try:
                assert check_call(ref, org, cur, S, bd, pus, np.zeros((0, 2), np.int32), pred, w, hh, par, dev) == 0, (fast, clip)
            finally:
                LAM = keep


@gpu
def test_final_cost_conversion_ends(eng, ref):
    """the (Distortion) conversion at both of its ends on the device, fast_sub_pel 2 and weight 1.25 (bcw_idx 4 on list 1):
    a PU whose target equals the reference block at its vector (pred = 2 * org - ref there) has a SAD of 0, so with few bits the expression is negative and
    wraps to 2^64 - k; a PU whose start lies below the ifp_lines bound has an empty window, cost MAX_DISTORTION, and the expression at or above 2^64 becomes 0"""
    import vvenc_b200 as V
    bd, w, hh = 10, 16, 16
    org, cur, _ = _planes(bd, 900)
    S = W + 2 * M
    eng.upload_plane(0, org, W, H, M); eng.upload_plane(1, cur, W, H, M)
    pus = np.zeros(2, dtype=V.BI_PU_DT)
    (x0, y0), v = (64, 320), (5, -3)
    pus['x'] = (x0, 64); pus['y'] = (y0, 0)
    pus['start_hor'] = (16 * v[0], 0); pus['start_ver'] = (16 * v[1], 60000)
    pus['pred_hor'] = (-2000, 0); pus['pred_ver'] = (1500, 0); pus['bits'] = (0, 2); pus['bcw_idx'] = 4
    pred = np.zeros((2, hh, w), dtype=np.int16)
    o = org[M + y0:M + y0 + hh, M + x0:M + x0 + w].astype(np.int32)
    r = cur[M + y0 + v[1]:M + y0 + v[1] + hh, M + x0 + v[0]:M + x0 + v[0] + w].astype(np.int32)
    pred[0] = 2 * o - r
    par = eng.bi_par(LAM, 0, W, H, CTU, V.DF_HAD, ref_list=1, fast_sub_pel=2, sub_shift_mode=0, ifp_lines=1)
    dev = eng.bipred_search(0, 1, pus, w, hh, par, pred)
    assert check_call(ref, org, cur, S, bd, pus, np.zeros((0, 2), np.int32), pred, w, hh, par, dev) == 0
    assert (int(dev['int_hor'][0]), int(dev['int_ver'][0]), int(dev['frac_cost'][0])) == (v[0], v[1], 0)
    assert int(dev['cost'][0]) >= 1 << 63
    assert int(dev['int_best'][1]) == (1 << 64) - 1 and int(dev['cost'][1]) == 0


def sass_digest(sass, name):
    """sha256 of one function's instructions in `cuobjdump -sass` text (addresses and encodings dropped)"""
    import hashlib, re
    m = re.search(r"Function : (" + name + r")\n(.*?)(?=\n\s*Function :|\Z)", sass, re.S)
    assert m, name
    ins = [re.sub(r'/\*[0-9a-f]{4,}\*/', '', l).split(';')[0].strip() for l in m.group(2).splitlines() if re.match(r'\s+/\*[0-9a-f]{4,}\*/', l)]
    return hashlib.sha256('\n'.join(ins).encode()).hexdigest()


def test_compiler_report():
    """-Xptxas -v shows no spills in the kernels of this call, and frac_search_kernel<FracOrgPlane> keeps the SASS recorded in
    tests/golden/frac_search_kernel.sass.sha256 (DESIGN §3 compares it with the kernel before it became a template)"""
    import os, re, shutil, subprocess
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'vvenc_b200', 'csrc')
    log = open(os.path.join(csrc, 'build.log')).read()
    blocks = re.findall(r"Compiling entry function '(\w+)'.*?\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log, re.S)
    mine = [(n, st, ld) for (n, st, ld) in blocks if 'bipred_int_kernel' in n or 'frac_search_kernel' in n]
    assert len(mine) == 6, mine                                  # bipred_int_kernel<4, 8, 16, 32>, frac_search_kernel<FracOrgPlane>, <FracOrgTarget>
    assert all(st == '0' and ld == '0' for (_, st, ld) in mine), mine
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    sass = subprocess.run([cuobjdump, '-sass', os.path.join(csrc, 'libvvenc_b200.so')], capture_output=True, text=True, check=True).stdout
    golden = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'frac_search_kernel.sass.sha256')).read().split()[0]
    assert sass_digest(sass, r'_ZN3vvb18frac_search_kernelINS_12FracOrgPlaneEJEEEv\w*') == golden
