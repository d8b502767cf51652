"""vvb_tz_search, InterSearch::xTZSearch walked on the device for every PU of a call, against the reference (all but the replay check need -m gpu).

  * the member (refshim_tz_search_member: InterSearch::xTZSearch called on the unmodified reference objects) on the planes of the TZ binding test
    (cases.search_case seed 909, 256x160): every combination of extended / fast / integer early termination / first-search stop, search ranges 14, 80
    and 128, sub-sampling modes 0..2, twelve PU shapes, bit depths 8, 10 and 12.  mv, ruiSAD, uiBestSad and uiBestDistance must be equal for every PU.
  * extra start candidates (m_BlkUniMvInfoBuffer): the probe cannot fill that buffer, so a Python replay of xTZSearch on the probe's own SAD and MV
    cost is first pinned to the member without candidates, then used as the yardstick for PUs with 1..4 candidates (clipped ones, winning ones, ties),
    with ifp_lines 0..2 and MV-rate shifts 0, 2, 4, which the probe cannot set.
  * scale: every 8x8..64x64 PU of a 1920x1080 10-bit picture pair in one call per shape, more PUs than the grid holds resident warps.
  * admission: shapes (PUs larger than the CTU included), the reference margin at both limits of the reach of the clip rules (before and beyond the picture), bit depth, null pointers, negative counts, and the _dev twin.
"""
import ctypes
import itertools

import numpy as np
import pytest

import cases as C
from _libs import have_ref, refshim, P, PO

pytestmark = pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
gpu = pytest.mark.gpu

LAM = 57.0
SHAPES = [(8, 8), (16, 16), (32, 32), (64, 64), (128, 128), (8, 16), (16, 8), (32, 8), (8, 32), (64, 16), (4, 8), (8, 4)]
FLAGS = list(itertools.product((0, 1), repeat=4))            # extended, fast, integer_et, first_search_stop
RANGES = (14, 80, 128)
W, H = 256, 160


def _ctu(w, h):
    """the smallest CTU of 32, 64, 128 that holds the PU (a PU never exceeds its CTU)"""
    return 128 if max(w, h) > 64 else 64 if max(w, h) > 32 else 32


@pytest.fixture(scope="module")
def eng():
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def ref():
    R = refshim()
    dbl = ctypes.c_double
    R.refshim_tz_search_member.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, dbl] + [ctypes.c_int] * 7 + [ctypes.c_void_p]
    R.refshim_dist.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_int] * 4
    R.refshim_set_simd(b'AVX2')
    return R


def _planes(bit_depth, margin):
    """the 10-bit planes of the binding test at another bit depth (8: >> 2, 12: << 2 plus low bits) and margin"""
    tz = C.search_case(seed=909, W=W, H=H, margin=margin)
    org, cur = tz['org'].astype(np.int32), tz['ref'].astype(np.int32)
    if bit_depth == 8:
        org, cur = org >> 2, cur >> 2
    elif bit_depth == 12:
        rs = np.random.RandomState(12)
        org = (org << 2) | rs.randint(0, 4, size=org.shape); cur = (cur << 2) | rs.randint(0, 4, size=cur.shape)
    return np.ascontiguousarray(org, dtype=np.int16), np.ascontiguousarray(cur, dtype=np.int16), tz['stride'], margin


def _quarter(v):
    """Mv::changePrecision( MV_PRECISION_INTERNAL, MV_PRECISION_QUARTER )"""
    return (v + 1) >> 2 if v >= 0 else (v + 2) >> 2


def _pus(w, h, k, seed, pw=W, ph=H):
    rs = np.random.RandomState(seed)
    blk = np.zeros((k, 6), dtype=np.int32)
    for i in range(k):
        blk[i] = (rs.randint(0, (pw - w) // 4 + 1) * 4, rs.randint(0, (ph - h) // 4 + 1) * 4, w, h, rs.randint(-20 * 16, 20 * 16 + 1), rs.randint(-12 * 16, 12 * 16 + 1))
    return blk


def _tz_pus(blk, cand_first=None, cand_count=None):
    import vvenc_b200 as V
    p = np.zeros(len(blk), dtype=V.TZ_PU_DT)
    p['x'] = blk[:, 0]; p['y'] = blk[:, 1]; p['start_hor'] = blk[:, 4]; p['start_ver'] = blk[:, 5]
    p['pred_hor'] = [_quarter(int(v)) for v in blk[:, 4]]; p['pred_ver'] = [_quarter(int(v)) for v in blk[:, 5]]
    if cand_first is not None:
        p['cand_first'] = cand_first; p['cand_count'] = cand_count
    return p


def _member(R, org, cur, S, margin, blk, bd, mode, rng, ctu, flags, pw=W, ph=H):
    ext, fast, iet, stop = flags
    base = margin * S + margin
    out = np.zeros((len(blk), 8), dtype=np.int64)
    rc = R.refshim_tz_search_member(1, PO(org, base), S, PO(cur, base), S, pw, ph, margin, P(np.ascontiguousarray(blk)), len(blk), bd, mode, LAM, rng, ctu,
                                    ext, fast, iet, stop, 0, P(out))
    assert rc == 0
    return out


def _device(eng, blk, w, h, mode, rng, ctu, flags, pw=W, ph=H, cands=None, cand_first=None, cand_count=None, ifp=0, imv=0):
    ext, fast, iet, stop = flags
    tz = eng.tz_par(rng, pw, ph, ctu, extended=ext, fast=fast, integer_et=iet, first_search_stop=stop, sub_shift_mode=mode, ifp_lines=ifp)
    return eng.tz_search(0, 1, _tz_pus(blk, cand_first, cand_count), w, h, eng.me_par(LAM, 2, imv), tz, cands)


def _same(dev, mem):
    return (np.array_equal(dev['mv_hor'], mem[:, 0]) and np.array_equal(dev['mv_ver'], mem[:, 1]) and np.array_equal(dev['sad'].astype(np.int64), mem[:, 2])
            and np.array_equal(dev['cost'].astype(np.int64), mem[:, 4]) and np.array_equal(dev['best_distance'].astype(np.int64), mem[:, 5]))


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_tz_search_equals_the_member(eng, ref, bd):
    bad = []; n = 0; moved = 0
    for margin in (96, 144):                                  # 128x128 PUs (CTU 128) reach 135 pels beyond the picture
        org, cur, S, m = _planes(bd, margin)
        eng.upload_plane(0, org, W, H, m, bit_depth=bd); eng.upload_plane(1, cur, W, H, m, bit_depth=bd)
        for (w, h) in SHAPES:
            if (_ctu(w, h) == 128) != (margin == 144):
                continue
            blk = _pus(w, h, 6, 100 * w + h + bd)
            for flags in FLAGS:
                for rng in RANGES:
                    for mode in (0, 1, 2):
                        mem = _member(ref, org, cur, S, m, blk, bd, mode, rng, _ctu(w, h), flags)
                        dev = _device(eng, blk, w, h, mode, rng, _ctu(w, h), flags)
                        n += len(blk); moved += int((mem[:, :2] != 0).any(axis=1).sum())
                        if not _same(dev, mem):
                            bad.append((w, h, flags, rng, mode))
    assert bad == [], bad[:10]
    assert n == 3 * 16 * 3 * len(SHAPES) * 6 and moved > n // 2


# ---- a Python replay of InterSearch::xTZSearch (InterSearch.cpp:2297-2573) on the probe's SAD and MV cost, with extra start candidates ----------------
OFFX = ((0, -1, -1, 0, -1, 1, -1, -1, 1), (0, 0, 1, 1, -1, 1, 0, 1, 0))
OFFY = ((0, 0, -1, -1, 1, -1, 0, 1, 0), (0, -1, -1, 0, -1, 1, 1, 1, 1))


def _rshift(v, s):
    o = 1 << (s - 1)
    return (v + o - 1) >> s if v >= 0 else (v + o) >> s


def _cdiv2(v):
    return int(v / 2)                                          # C integer division


class Replay:
    def __init__(self, R, org, cur, S, margin, bd, w, h, mode, rng, ctu, flags, pw=W, ph=H, ifp=0, imv=0):
        self.R, self.org, self.cur, self.S, self.base, self.bd, self.w, self.h = R, org, cur, S, margin * S + margin, bd, w, h
        self.sub = 1 if (mode == 1 and h > 8 and w <= 128) or (mode == 2 and h > 8) else 0
        self.rng, self.ctu, self.pw, self.ph, self.ifp, self.imv = rng, ctu, pw, ph, ifp, imv
        self.ext, self.fast, self.iet, self.stop = [bool(f) for f in flags]

    def clip(self, x, y, search):
        hmax = (self.pw + 8 - x - 1) << 4; hmin = (-self.ctu - 8 - x + 1) * 16
        lh = self.ph + 8
        l2 = self.ctu.bit_length() - 1
        if search and self.ifp and (y >> l2) + self.ifp + 1 < (self.ph + self.ctu - 1) // self.ctu:
            lh = (((y >> l2) + self.ifp + 1) << l2) - self.h - 4
        return hmin, hmax, (-self.ctu - 8 - y + 1) * 16, (lh - y - 1) << 4

    def run(self, x0, y0, start, pred, cands):
        R = self.R
        sadc = {}

        def cost(x, y):
            if (x, y) not in sadc:
                o = self.base + y0 * self.S + x0
                sad = R.refshim_dist(1, 1, PO(self.org, o), self.S, PO(self.cur, o + y * self.S + x), self.S, self.w, self.h, self.bd, self.sub)
                sadc[(x, y)] = sad + R.refshim_mv_cost(LAM, x, y, pred[0], pred[1], 2, self.imv)
            return sadc[(x, y)]
        st = dict(best=2 ** 64 - 1, x=0, y=0, dist=0, rnd=0, nr=0)

        def helpp(x, y, nr, d):
            c = cost(x, y)
            if c < st['best']:
                st.update(best=c, x=x, y=y, dist=d, rnd=0, nr=nr)
        sr = {}

        def diamond(sx, sy, d, corners):
            top, bottom, left, right = sy - d, sy + d, sx - d, sx + d
            st['rnd'] += 1
            if d == 1:
                if top >= sr['t']:
                    if corners:
                        if left >= sr['l']: helpp(left, top, 1, d)
                        helpp(sx, top, 2, d)
                        if right <= sr['r']: helpp(right, top, 3, d)
                    else:
                        helpp(sx, top, 2, d)
                if left >= sr['l']: helpp(left, sy, 4, d)
                if right <= sr['r']: helpp(right, sy, 5, d)
                if bottom <= sr['b']:
                    if corners:
                        if left >= sr['l']: helpp(left, bottom, 6, d)
                        helpp(sx, bottom, 7, d)
                        if right <= sr['r']: helpp(right, bottom, 8, d)
                    else:
                        helpp(sx, bottom, 7, d)
            elif d <= 8:
                h2 = d >> 1
                t2, b2, l2, r2 = sy - h2, sy + h2, sx - h2, sx + h2
                if top >= sr['t']: helpp(sx, top, 2, d)
                if t2 >= sr['t']:
                    if l2 >= sr['l']: helpp(l2, t2, 1, h2)
                    if r2 <= sr['r']: helpp(r2, t2, 3, h2)
                if left >= sr['l']: helpp(left, sy, 4, d)
                if right <= sr['r']: helpp(right, sy, 5, d)
                if b2 <= sr['b']:
                    if l2 >= sr['l']: helpp(l2, b2, 6, h2)
                    if r2 <= sr['r']: helpp(r2, b2, 8, h2)
                if bottom <= sr['b']: helpp(sx, bottom, 7, d)
            else:
                if top >= sr['t']: helpp(sx, top, 0, d)
                if left >= sr['l']: helpp(left, sy, 0, d)
                if right <= sr['r']: helpp(right, sy, 0, d)
                if bottom <= sr['b']: helpp(sx, bottom, 0, d)
                for i in range(1, 4):
                    yt, yb, xl, xr = top + (d >> 2) * i, bottom - (d >> 2) * i, sx - (d >> 2) * i, sx + (d >> 2) * i
                    if yt >= sr['t']:
                        if xl >= sr['l']: helpp(xl, yt, 0, d)
                        if xr <= sr['r']: helpp(xr, yt, 0, d)
                    if yb <= sr['b']:
                        if xl >= sr['l']: helpp(xl, yb, 0, d)
                        if xr <= sr['r']: helpp(xr, yb, 0, d)

        def two_point():
            n = st['nr']
            for k in (0, 1):
                x, y = st['x'] + OFFX[k][n], st['y'] + OFFY[k][n]
                if sr['l'] <= x <= sr['r'] and sr['t'] <= y <= sr['b']:
                    helpp(x, y, 0, 2)

        hmin, hmax, vmin, vmax = self.clip(x0, y0, True)
        mx = _rshift(_rshift(min(hmax, max(hmin, start[0])), 2), 2); my = _rshift(_rshift(min(vmax, max(vmin, start[1])), 2), 2)
        helpp(mx, my, 0, 0)
        if not self.fast and (mx or my) and (st['x'] or st['y']):
            helpp(0, 0, 0, 0)
        for (ch, cv) in cands:
            x, y = _rshift(min(hmax, max(hmin, ch)), 4), _rshift(min(vmax, max(vmin, cv)), 4)
            c = cost(x, y)
            if c < st['best']:
                st.update(best=c, x=x, y=y)
        cmn = self.clip(x0, y0, False)
        r16 = (self.rng >> (1 if self.fast else 0)) << 4
        px, py = min(cmn[1], max(cmn[0], st['x'] * 16)), min(cmn[3], max(cmn[2], st['y'] * 16))
        sr.update(l=_rshift(min(cmn[1], max(cmn[0], px - r16)), 4), t=_rshift(min(cmn[3], max(cmn[2], py - r16)), 4),
                  r=_rshift(min(hmax, max(hmin, px + r16)), 4), b=_rshift(min(vmax, max(vmin, py + r16)), 4))
        sx, sy = st['x'], st['y']
        if self.iet:
            diamond(sx, sy, 1, False)
            if (st['x'], st['y']) == (sx, sy):
                done = True
                if self.w * self.h > 64:
                    st['rnd'] += 1
                    for (x, y, nr) in ((sx - 1, sy - 1, 1), (sx + 1, sy - 1, 3), (sx - 1, sy + 1, 6), (sx + 1, sy + 1, 8)):
                        if (y >= sr['t'] if nr < 6 else y <= sr['b']) and (x >= sr['l'] if nr in (1, 6) else x <= sr['r']):
                            helpp(x, y, nr, 1)
                    done = (st['x'], st['y']) == (sx, sy)
                if done:
                    return st['x'], st['y'], st['best'] - R.refshim_mv_cost(LAM, st['x'], st['y'], pred[0], pred[1], 2, self.imv), st['best'], st['dist']
        sx, sy = st['x'], st['y']
        zero = sx == 0 and sy == 0
        d = 1
        while d <= self.rng:
            diamond(sx, sy, d, self.ext)
            if self.stop and st['rnd'] >= 3:
                break
            d *= 2
        if self.ext and not zero:
            d = 1
            while d <= (self.rng >> 1):
                diamond(0, 0, d, False); d *= 2
        if st['dist'] == 1:
            st['dist'] = 0; two_point()
        ras = 8 if self.fast else 5
        if self.ext:
            win, l, r, t, b = ras, sr['l'], sr['r'], sr['t'], sr['b']
            if not st['dist'] >= ras:
                win += 1; l, r, t, b = _cdiv2(l), _cdiv2(r), _cdiv2(t), _cdiv2(b)
            st['dist'] = win
            for y in range(t, b + 1, win):
                for x in range(l, r + 1, win):
                    helpp(x, y, 0, win)
        elif st['dist'] >= ras:
            st['dist'] = ras
            for y in range(sr['t'], sr['b'] + 1, ras):
                for x in range(sr['l'], sr['r'] + 1, ras):
                    helpp(x, y, 0, ras)
        while st['dist'] > 0:
            sx, sy = st['x'], st['y']
            st['dist'] = 0; st['nr'] = 0
            d = 1
            while d < self.rng + 1:
                diamond(sx, sy, d, self.ext)
                if self.fast and st['rnd'] >= 2:
                    break
                d *= 2
            if st['dist'] == 1:
                st['dist'] = 0
                if st['nr'] != 0:
                    two_point()
        return st['x'], st['y'], st['best'] - R.refshim_mv_cost(LAM, st['x'], st['y'], pred[0], pred[1], 2, self.imv), st['best'], st['dist']


def test_replay_equals_the_member_without_candidates(ref):
    """(CPU) the yardstick of the candidate test, pinned first: the whole flag x range x sub-sampling matrix at 10 bits, two PUs per shape"""
    org, cur, S, m = _planes(10, 96)
    bad = []; n = 0
    for (w, h) in SHAPES:
        if _ctu(w, h) == 128:
            continue
        blk = _pus(w, h, 2, 7 * w + h)
        for flags in FLAGS:
            for rng in RANGES:
                for mode in (0, 1, 2):
                    mem = _member(ref, org, cur, S, m, blk, 10, mode, rng, _ctu(w, h), flags)
                    rp = Replay(ref, org, cur, S, m, 10, w, h, mode, rng, _ctu(w, h), flags)
                    for i, b in enumerate(blk):
                        got = rp.run(int(b[0]), int(b[1]), (int(b[4]), int(b[5])), (_quarter(int(b[4])), _quarter(int(b[5]))), [])
                        n += 1
                        if tuple(int(v) for v in got) != (int(mem[i, 0]), int(mem[i, 1]), int(mem[i, 2]), int(mem[i, 4]), int(mem[i, 5])):
                            bad.append((w, h, flags, rng, mode, i))
    assert bad == [], bad[:10]
    assert n == 11 * 16 * 3 * 3 * 2


@gpu
def test_tz_search_with_start_candidates_equals_the_replay(eng, ref):
    """also with ifp_lines > 0 (the bottom clip of xClipMvSearch for PUs in the first CTU rows) and AMVR shifts of the MV rate, which the member probe
    fixes at 0; `clipped` counts the walks the ifp clip changes, `imv_moved` those the shifted MV rate changes"""
    org, cur, S, m = _planes(10, 96)
    eng.upload_plane(0, org, W, H, m, bit_depth=10); eng.upload_plane(1, cur, W, H, m, bit_depth=10)
    rs = np.random.RandomState(31)
    bad = []; n = 0; won = 0; clipped = 0; imv_moved = 0
    for (w, h) in ((8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (8, 32), (4, 8)):
        blk = _pus(w, h, 8, 3 * w + h + 1)
        cands, first, count = [], [], []
        for i, b in enumerate(blk):
            k = 1 + i % 4
            first.append(len(cands)); count.append(k)
            pool = [(32, -48),                                                # the true pan of the picture pair (wins where the start does not)
                    (int(b[4]), int(b[5])),                                   # the start vector again: ties the current best
                    (int(rs.choice([-1, 1])) * 60000, int(rs.choice([-1, 1])) * 60000),   # far outside: clipped by xClipMvSearch
                    (int(rs.randint(-400, 401)), int(rs.randint(-300, 301)))]
            for j in range(k):
                cands.append(pool[(i + j) % 4])
        cands = np.array(cands, dtype=np.int32)
        for flags in ((0, 0, 0, 0), (1, 0, 0, 0), (0, 1, 0, 1), (1, 1, 1, 0), (0, 0, 1, 1), (1, 1, 1, 1)):
            for (rng, ifp, imv) in ((14, 0, 0), (80, 0, 0), (80, 1, 2), (80, 2, 4), (14, 1, 0)):
                mode = (w + rng) % 3
                ctu = _ctu(w, h)
                dev = _device(eng, blk, w, h, mode, rng, ctu, flags, cands=cands, cand_first=first, cand_count=count, ifp=ifp, imv=imv)
                rp = Replay(ref, org, cur, S, m, 10, w, h, mode, rng, ctu, flags, ifp=ifp, imv=imv)
                rp0 = Replay(ref, org, cur, S, m, 10, w, h, mode, rng, ctu, flags, ifp=0, imv=imv) if ifp else None
                rpi = Replay(ref, org, cur, S, m, 10, w, h, mode, rng, ctu, flags, ifp=ifp, imv=0) if imv else None
                for i, b in enumerate(blk):
                    cl = [(int(c[0]), int(c[1])) for c in cands[first[i]:first[i] + count[i]]]
                    args = (int(b[0]), int(b[1]), (int(b[4]), int(b[5])), (_quarter(int(b[4])), _quarter(int(b[5]))))
                    got = rp.run(*args, cl)
                    won += int(got != rp.run(*args, []))
                    clipped += int(rp0 is not None and got != rp0.run(*args, cl))
                    imv_moved += int(rpi is not None and got[:2] != rpi.run(*args, cl)[:2])
                    n += 1
                    d = dev[i]
                    if (int(d['mv_hor']), int(d['mv_ver']), int(d['sad']), int(d['cost']), int(d['best_distance'])) != tuple(int(v) for v in got):
                        bad.append((w, h, flags, rng, i))
    assert bad == [], bad[:10]
    assert won > n // 10                                       # the candidates change the outcome of a good share of the walks
    assert clipped > 10 and imv_moved > 0


@gpu
def test_tz_search_at_picture_scale(eng, ref):
    """every 8x8..64x64 PU of a 1920x1080 10-bit picture pair (SearchRange 128, fast settings), one call per shape"""
    import torch
    PW, PH, m = 1920, 1080, 144
    rs = np.random.RandomState(4242)
    S = PW + 2 * m
    b = rs.randint(0, 1024, size=(PH + 2 * m + 8, S + 8))
    sm = (b + np.roll(b, 1, 0) + np.roll(b, 1, 1) + np.roll(b, (1, 1), (0, 1))) // 4
    org = np.ascontiguousarray(sm[4:4 + PH + 2 * m, 4:4 + S], dtype=np.int16)
    cur = np.ascontiguousarray(np.clip(sm[1:1 + PH + 2 * m, 7:7 + S] + rs.randint(-9, 10, size=org.shape), 0, 1023), dtype=np.int16)
    eng.upload_plane(0, org, PW, PH, m, bit_depth=10); eng.upload_plane(1, cur, PW, PH, m, bit_depth=10)
    resident = torch.cuda.get_device_properties(0).multi_processor_count * 64           # at most 64 resident warps per SM
    flags = (0, 1, 0, 1)
    for s in (8, 16, 32, 64):
        ys, xs = np.mgrid[0:PH - s + 1:s, 0:PW - s + 1:s]
        blk = np.zeros((xs.size, 6), dtype=np.int32)
        blk[:, 0] = xs.ravel(); blk[:, 1] = ys.ravel(); blk[:, 2] = s; blk[:, 3] = s
        blk[:, 4] = rs.randint(-64 * 16, 64 * 16 + 1, size=xs.size); blk[:, 5] = rs.randint(-40 * 16, 40 * 16 + 1, size=xs.size)
        if s == 8:
            assert len(blk) > resident
        mem = _member(ref, org, cur, S, m, blk, 10, 1, 128, 128, flags, PW, PH)
        dev = _device(eng, blk, s, s, 1, 128, 128, flags, PW, PH)
        assert _same(dev, mem), s


@gpu
def test_tz_search_admission(eng, ref):
    import torch
    import vvenc_b200 as V
    from vvenc_b200 import _lib as L
    org, cur, S, m = _planes(10, 96)
    eng.upload_plane(0, org, W, H, m, bit_depth=10); eng.upload_plane(1, cur, W, H, m, bit_depth=10)
    blk = _pus(16, 16, 5, 3)
    me = eng.me_par(LAM, 2, 0)
    tz = eng.tz_par(80, W, H, 32, extended=1, sub_shift_mode=1)
    for (w, h) in ((2, 8), (8, 2), (12, 8), (8, 24), (256, 8), (8, 256), (64, 16), (16, 64)):     # the last two exceed the CTU of 32
        with pytest.raises(V.VvbError) as e:
            eng.tz_search(0, 1, _tz_pus(_pus(4, 4, 2, 1)), w, h, me, tz)
        assert e.value.code == L.VVB_ERR_UNSUPPORTED, (w, h)
    # the reference margin on both sides of the reach: 32x32 PUs with CTU 64 read at most 64 + 7 pels left of / above the picture and 32 + 7 beyond it
    ref_blk = _pus(32, 32, 6, 77)
    want = _member(ref, org, cur, S, m, ref_blk, 10, 0, 80, 64, (1, 0, 0, 0))
    for mg in (71, 70):
        sub = np.ascontiguousarray(cur[m - mg:m + H + mg, m - mg:m + W + mg])
        eng.upload_plane(2, sub, W, H, mg, bit_depth=10)
        tz64 = eng.tz_par(80, W, H, 64, extended=1)
        if mg == 71:
            assert _same(eng.tz_search(0, 2, _tz_pus(ref_blk), 32, 32, me, tz64), want)
        else:
            with pytest.raises(V.VvbError) as e:
                eng.tz_search(0, 2, _tz_pus(ref_blk), 32, 32, me, tz64)
            assert e.value.code == L.VVB_ERR_UNSUPPORTED
    # the other side: a reference plane 40 pels narrower than the picture needs 32 + 7 + 40 pels of margin on its right
    tz32 = eng.tz_par(80, W, H, 32, extended=1)
    want = _member(ref, org, cur, S, m, ref_blk, 10, 0, 80, 32, (1, 0, 0, 0))
    for mg in (79, 78):
        sub = np.ascontiguousarray(cur[m - mg:m + H + mg, m - mg:m + W - 40 + mg])
        eng.upload_plane(2, sub, W - 40, H, mg, bit_depth=10)
        if mg == 79:
            assert _same(eng.tz_search(0, 2, _tz_pus(ref_blk), 32, 32, me, tz32), want)
        else:
            with pytest.raises(V.VvbError) as e:
                eng.tz_search(0, 2, _tz_pus(ref_blk), 32, 32, me, tz32)
            assert e.value.code == L.VVB_ERR_UNSUPPORTED
    eng.upload_plane(3, cur, W, H, m, bit_depth=14)
    with pytest.raises(V.VvbError) as e:
        eng.tz_search(0, 3, _tz_pus(blk), 16, 16, me, tz)
    assert e.value.code == L.VVB_ERR_UNSUPPORTED
    # malformed arguments
    lib, hnd = eng.lib, eng.h
    pus = _tz_pus(blk); out = np.zeros(len(pus), dtype=V.TZ_BEST_DT)
    A = L.VVB_ERR_ARG
    assert lib.vvb_tz_search(hnd, 0, 1, None, 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 0, P(out)) == A
    assert lib.vvb_tz_search(hnd, 0, 1, P(pus), 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 0, None) == A
    assert lib.vvb_tz_search(hnd, 0, 1, P(pus), 5, 16, 16, None, ctypes.byref(tz), None, 0, P(out)) == A
    assert lib.vvb_tz_search(hnd, 0, 1, P(pus), 5, 16, 16, ctypes.byref(me), None, None, 0, P(out)) == A
    assert lib.vvb_tz_search(hnd, 0, 1, P(pus), -1, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 0, P(out)) == A
    assert lib.vvb_tz_search(hnd, 0, 1, P(pus), 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, -1, P(out)) == A
    assert lib.vvb_tz_search(hnd, 0, 1, P(pus), 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 2, P(out)) == A      # candidates without a buffer
    bad = pus.copy(); bad['cand_count'][2] = 1                                                                              # range outside cands
    assert lib.vvb_tz_search(hnd, 0, 1, P(bad), 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 0, P(out)) == A
    bad = pus.copy(); bad['x'][1] = W - 8                                                                                    # PU outside the picture
    assert lib.vvb_tz_search(hnd, 0, 1, P(bad), 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 0, P(out)) == A
    assert lib.vvb_tz_search_dev(hnd, 0, 1, None, 5, 16, 16, ctypes.byref(me), ctypes.byref(tz), None, 0, P(out)) == A
    # the _dev twin on device buffers gives the host-buffer call's results
    cands = np.array([[32, -48], [900, 900], [-60000, 12]], dtype=np.int32)
    pus['cand_first'] = [0, 1, 0, 2, 3]; pus['cand_count'] = [1, 2, 3, 1, 0]
    host = eng.tz_search(0, 1, pus, 16, 16, me, tz, cands)
    d_pus = torch.from_numpy(pus.view(np.uint8).copy()).cuda()
    d_c = torch.from_numpy(cands.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(pus) * 32, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    assert lib.vvb_tz_search_dev(hnd, 0, 1, d_pus.data_ptr(), len(pus), 16, 16, ctypes.byref(me), ctypes.byref(tz), d_c.data_ptr(), len(cands), d_out.data_ptr()) == 0
    eng.synchronize()
    dev = np.frombuffer(d_out.cpu().numpy().tobytes(), dtype=V.TZ_BEST_DT)
    assert np.array_equal(dev, host)
