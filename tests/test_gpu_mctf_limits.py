"""MCTF kernels at the limits of their number formats and geometry, against a plain int64 restatement of MCTF::motionErrorLuma (MCTF.cpp:122-257):
  * the error list and the search grid at full contrast, 8 and 10 bits, blocks 8..64 (64 x 64 included), all 16 phases in x and y, both filter sets,
    odd and even source alignment, vectors reaching the edge of a 128-pel margin;
  * stage B (the integer grid), the wavefront of the upper / left neighbours and the whole pyramid at unit 32 (64 x 64 blocks on the coarse levels),
    expected from vvenc_b200/mctf_host.py driven by the int64 errors;
  * the apply stage at its extremes (full contrast, 8 references, unit 4, trailing partial units, the planar clamp, error 0x7fffffff);
  * the 10-bit admission of every MCTF entry, and which kernels the stage-B and wavefront cases run.
An error is exact up to INT32_MAX and saturates to 0x7fffffff above it: under the strict `error < best.error` chains a saturated candidate never beats
a finite best, which is what the reference's early exit decides.  The reference is undefined only when the first candidate of a chain overflows already;
the level cases assert in int64 that this does not happen."""
import ctypes
import os
import numpy as np
import pytest
from _libs import oracle, P

INT_MAX = 0x7fffffff
MARGIN = 128                                   # MCTF_PADDING
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v7_mctf_limits.npz')


@pytest.fixture(scope="module")
def eng():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def golden_v7():
    return np.load(GOLDEN)


def _V():
    import vvenc_b200 as V
    return V


# ---------------------------------------------------------------------------------------------------- the int64 reference
_FILTERS = []


def filters():
    """the 6-tap (entries 1..6 of the 8-wide rows) and 4-tap MCTF filter tables, [16 phases][taps]"""
    if not _FILTERS:
        f8 = np.zeros((16, 8), dtype=np.int16); f4 = np.zeros((16, 4), dtype=np.int16)
        oracle().orc_mctf_filters(P(f8), P(f4))
        _FILTERS.extend([f8[:, 1:7].astype(np.int64), f4.astype(np.int64)])
    return _FILTERS


def err_exact(org, ref, x, y, mvx, mvy, w, h, bd, tap4):
    """motionErrorLuma of block (x, y, w, h) -- array coordinates of the padded planes -- at vector (mvx, mvy) in 1/16 pel, in int64 without an early
    exit: integer vectors take the plain SSE, fractional ones the separable filter with a clip after each pass (MCTF.cpp:122-257)"""
    fx, fy = mvx & 15, mvy & 15
    o = org[y:y + h, x:x + w].astype(np.int64)
    if fx == 0 and fy == 0:
        dx, dy = int(mvx / 16), int(mvy / 16)
        d = o - ref[y + dy:y + dy + h, x + dx:x + dx + w]
        return int((d * d).sum())
    dx, dy = mvx >> 4, mvy >> 4
    f = filters()[1 if tap4 else 0]
    taps, back = f.shape[1], (1 if tap4 else 2)
    maxv = (1 << bd) - 1
    win = ref[y + dy - back:y + dy - back + h + taps - 1, x + dx - back:x + dx - back + w + taps - 1].astype(np.int64)
    t = sum(f[fx, k] * win[:, k:k + w] for k in range(taps))
    t = np.clip((t + 32) >> 6, 0, maxv)
    v = sum(f[fy, k] * t[k:k + h, :] for k in range(taps))
    v = np.clip((v + 32) >> 6, 0, maxv)
    d = v - o
    return int((d * d).sum())


def sat(e):
    return min(int(e), INT_MAX)


class Int64Provider:
    """mctf_host provider on a padded picture pair (margin m) from err_exact, saturated to 0x7fffffff.  With check_first, the first candidate evaluated
    for a block (the start of its `error < best.error` chain) must be below INT32_MAX exactly -- the one case where the reference is undefined."""

    def __init__(self, org, ref, m, bd, tap4=0, check_first=True):
        self.org = org; self.ref = ref; self.m = m; self.bd = bd; self.tap4 = tap4
        self.check_first = check_first; self.seen = set(); self.exact_max = 0; self.saturated = 0

    def _err(self, c):
        e = err_exact(self.org, self.ref, int(c['x']) + self.m, int(c['y']) + self.m, int(c['mvx']), int(c['mvy']), int(c['w']), int(c['h']), self.bd, self.tap4)
        self.exact_max = max(self.exact_max, e); self.saturated += e > INT_MAX
        return e

    def _first(self, c, e):
        key = (int(c['x']), int(c['y']))
        if key not in self.seen:
            self.seen.add(key)
            assert not self.check_first or e < INT_MAX, ('the first candidate of a chain overflows', key, e)

    def errors(self, cands):
        out = np.zeros(len(cands), dtype=np.int32)
        for i, c in enumerate(cands):
            e = self._err(c)
            self._first(c, e)
            out[i] = sat(e)
        return out

    def grid(self, blocks, step, radius):
        k1 = 2 * radius + 1
        out = np.zeros((len(blocks), k1, k1), dtype=np.int32)
        for b, blk in enumerate(blocks):
            for j in range(k1):
                for i in range(k1):
                    c = blk.copy(); c['mvx'] = int(blk['mvx']) + (i - radius) * step; c['mvy'] = int(blk['mvy']) + (j - radius) * step
                    e = self._err(c)
                    if i == 0 and j == 0:
                        self._first(c, e)
                    out[b, j, i] = sat(e)
        return out

    def calc_var(self, blocks):
        O = oracle(); O.orc_mctf_calc_var.restype = ctypes.c_double
        S = self.org.shape[1]
        return np.array([O.orc_mctf_calc_var(ctypes.c_void_p(self.org.ctypes.data + 2 * ((int(b['y']) + self.m) * S + int(b['x']) + self.m)), S, int(b['w']), int(b['h']))
                         for b in blocks])


def test_int64_reference_equals_oracle():
    """err_exact equals orc_mctf_err_list (which test_oracle_vs_reference.py pins to the reference) wherever the int32 sums of the oracle cannot wrap:
    random and full-contrast content, every phase, both filter sets, 8 and 10 bits, blocks 8..64"""
    O = oracle()
    rs = np.random.RandomState(7)
    m, W, H = 24, 160, 128
    S = W + 2 * m
    for bd in (8, 10):
        mx = (1 << bd) - 1
        org = rs.randint(0, mx + 1, size=(H + 2 * m, S)).astype(np.int16)
        ref = np.where(rs.randint(0, 2, size=org.shape) == 1, mx, 0).astype(np.int16)
        ref[:, :S // 2] = np.clip(org[:, :S // 2] + rs.randint(-60, 61, size=(H + 2 * m, S // 2)), 0, mx)
        for tap4 in (0, 1):
            desc = []
            for k in range(300):
                w, h = [(8, 8), (16, 16), (32, 32), (64, 32), (32, 64), (64, 64), (24, 8)][k % 7]
                if bd == 10 and w * h > 2048:
                    w, h = 32, 32                       # full contrast at 10 bits: 2048 pels * 1023^2 stays below 2^31
                desc.append([int(rs.randint(0, W - w + 1)) + m, int(rs.randint(0, H - h + 1)) + m, (k % 16) + 16 * int(rs.randint(-8, 9)) if k % 5 else 16 * int(rs.randint(-8, 9)),
                             ((k // 16) % 16) + 16 * int(rs.randint(-8, 9)), w, h])
            desc = np.ascontiguousarray(desc, dtype=np.int32)
            exp = np.zeros(len(desc), dtype=np.int32)
            O.orc_mctf_err_list(tap4, P(org), S, P(ref), S, P(desc), len(desc), bd, P(exp))
            got = [err_exact(org, ref, *[int(v) for v in d], bd, tap4) for d in desc]
            assert max(got) <= INT_MAX and got == exp.tolist(), (bd, tap4)


# ---------------------------------------------------------------------------------------------------- content
def contrast_pair(seed, W, H, m, bd):
    """padded org / ref (margin m) of 32 x 32 tiles: org column stripes 0 / max over a small texture; ref the same stripes, the inverted stripes, a
    checkerboard at full range or random pels -- SSEs of 64 x 64 blocks spread from near 0 to far above 2^31"""
    rs = np.random.RandomState(seed)
    mx = (1 << bd) - 1
    shape = (H + 2 * m, W + 2 * m)
    yy, xx = np.mgrid[0:shape[0], 0:shape[1]]
    tex = rs.randint(0, 8, size=shape)
    stripes = np.where(xx & 1, mx - tex, tex)
    org = stripes
    kind = ((yy // 32) * 7 + (xx // 32) * 3) % 4
    ref = np.select([kind == 0, kind == 1, kind == 2], [stripes, mx - stripes, np.where((xx + yy) & 1, mx, 0)], rs.randint(0, mx + 1, size=shape))
    return np.ascontiguousarray(org.astype(np.int16)), np.ascontiguousarray(ref.astype(np.int16))


def reach_ok(x, y, mvx, mvy, w, h, W, H):
    """the pels the kernels may read for this candidate (two more rows and columns than the filter, for the pair staging) lie within the 128-pel margin"""
    dx, dy = mvx >> 4, mvy >> 4
    return x + dx - 4 >= -MARGIN and y + dy - 4 >= -MARGIN and x + dx + w + 4 <= W + MARGIN and y + dy + h + 4 <= H + MARGIN


SHAPES = ((8, 8), (16, 16), (32, 32), (64, 64), (64, 8), (8, 64), (24, 40), (64, 32), (48, 64))


def error_list_cands(rs, W, H, n):
    """n candidates: every shape, all 16 x 16 phase pairs, odd and even x, vectors up to the margin's edge (one in eight reaches it)"""
    V = _V()
    c = np.zeros(n, dtype=V.MCTF_DT)
    k = 0
    while k < n:
        w, h = SHAPES[k % len(SHAPES)]
        x = int(rs.randint(0, W - w + 1)); y = int(rs.randint(0, H - h + 1))
        x = (x & ~1) | (k & 1)                                   # odd and even source alignment
        if x + w > W:
            x -= 2
        fx, fy = k % 16, (k // 16) % 16
        if k % 8 == 7:                                         # towards the edge of the margin
            sx = -1 if rs.randint(0, 2) else 1; sy = -1 if rs.randint(0, 2) else 1
            dx = (-(MARGIN - 4) - x) if sx < 0 else (W + MARGIN - 4 - w - x)
            dy = (-(MARGIN - 4) - y) if sy < 0 else (H + MARGIN - 4 - h - y)
            if (k // 8) % 2:
                fx = fy = 0
                dx = (-MARGIN - x) if sx < 0 else (W + MARGIN - w - x)
                dy = (-MARGIN - y) if sy < 0 else (H + MARGIN - h - y)
        else:
            dx, dy = int(rs.randint(-40, 41)), int(rs.randint(-40, 41))
        mvx, mvy = 16 * dx + fx, 16 * dy + fy
        if not reach_ok(x, y, mvx, mvy, w, h, W, H) and (fx or fy):
            continue
        c[k] = (x, y, mvx, mvy, w, h)
        k += 1
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10])
def test_error_list_full_contrast(eng, bd):
    W, H = 256, 192
    org, ref = contrast_pair(100 + bd, W, H, MARGIN, bd)
    eng.upload_plane(0, org, W, H, MARGIN, bd); eng.upload_plane(1, ref, W, H, MARGIN, bd)
    rs = np.random.RandomState(bd)
    for tap4 in (0, 1):
        c = error_list_cands(rs, W, H, 1024)
        got = eng.mctf_error_batch(0, 1, c, bool(tap4))
        exact = np.array([err_exact(org, ref, int(e['x']) + MARGIN, int(e['y']) + MARGIN, int(e['mvx']), int(e['mvy']), int(e['w']), int(e['h']), bd, tap4) for e in c])
        exp = np.minimum(exact, INT_MAX).astype(np.int32)
        bad = np.nonzero(got != exp)[0]
        assert len(bad) == 0, (tap4, len(bad), [(c[i].tolist(), int(got[i]), int(exact[i])) for i in bad[:4]])
        if bd == 10:
            assert (exact > INT_MAX).sum() >= 3 and ((exact > 2 ** 30) & (exact <= INT_MAX)).sum() > 20


GRIDS = ((16, 8), (16, 5), (4, 3), (2, 1), (1, 1), (6, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10])
def test_search_grid_full_contrast(eng, bd):
    W, H = 256, 192
    org, ref = contrast_pair(200 + bd, W, H, MARGIN, bd)
    eng.upload_plane(0, org, W, H, MARGIN, bd); eng.upload_plane(1, ref, W, H, MARGIN, bd)
    rs = np.random.RandomState(20 + bd)
    V = _V()
    sat_seen = 0
    for (step, radius) in GRIDS:
        for tap4 in (0, 1):
            shapes = ((64, 64), (64, 64), (32, 32), (8, 8), (64, 16), (40, 24))
            b = np.zeros(len(shapes), dtype=V.MCTF_DT)
            for i, (w, h) in enumerate(shapes):
                x = (int(rs.randint(0, W - w + 1)) & ~1) | (i & 1)
                x = min(x, W - w)
                y = int(rs.randint(0, H - h + 1))
                cx, cy = 16 * int(rs.randint(-12, 13)) + int(rs.randint(0, 16)), 16 * int(rs.randint(-12, 13)) + int(rs.randint(0, 16))
                if i == 1:                                     # the grid's corner reaches the margin's edge
                    cx = 16 * (-(MARGIN - 4) - x) + radius * step; cy = 16 * (H + MARGIN - 4 - h - y) - radius * step - 15
                b[i] = (x, y, cx, cy, w, h)
            got = eng.mctf_search_grid(0, 1, b, step, radius, bool(tap4))
            k1 = 2 * radius + 1
            exact = np.zeros((len(b), k1, k1), dtype=np.int64)
            for i, blk in enumerate(b):
                for j in range(k1):
                    for ii in range(k1):
                        mvx = int(blk['mvx']) + (ii - radius) * step; mvy = int(blk['mvy']) + (j - radius) * step
                        assert reach_ok(int(blk['x']), int(blk['y']), mvx, mvy, int(blk['w']), int(blk['h']), W, H)
                        exact[i, j, ii] = err_exact(org, ref, int(blk['x']) + MARGIN, int(blk['y']) + MARGIN, mvx, mvy, int(blk['w']), int(blk['h']), bd, tap4)
            exp = np.minimum(exact, INT_MAX).astype(np.int32)
            sat_seen += int((exact > INT_MAX).sum())
            assert np.array_equal(got, exp), (step, radius, tap4, [(b[i].tolist(), int(got[i, j, k]), int(exact[i, j, k])) for i, j, k in np.argwhere(got != exp)[:4]])
    assert bd == 8 or sat_seen > 0


# ---------------------------------------------------------------------------------------------------- levels
def stripe_pair(seed, W, H, half_period, shift_of, bd=10, noise=2):
    """unpadded org / ref: column stripes 0 / max of half-period half_period over a texture of at most 12 (so that a half-mismatched 64 x 64 block stays
    below 2^31 and a fully mismatched one lies above it); ref(y, x) = org(y, x - s) + noise, s = shift_of(block column, block row) of the 64 x 64 block"""
    rs = np.random.RandomState(seed)
    mx = (1 << bd) - 1
    pad = 32
    yy, xx = np.mgrid[0:H + 2 * pad, 0:W + 2 * pad]
    tex = rs.randint(0, 13, size=yy.shape)
    full = np.where(((xx - pad) // half_period) & 1, mx - tex, tex)
    org = full[pad:pad + H, pad:pad + W]
    ref = np.zeros((H, W), dtype=np.int64)
    for by in range(0, H, 64):
        for bx in range(0, W, 64):
            s = shift_of(bx // 64, by // 64)
            ref[by:by + 64, bx:bx + 64] = full[pad + by:pad + by + 64, pad + bx - s:pad + bx - s + 64][:H - by, :W - bx]
    ref = np.clip(ref + rs.randint(-noise, noise + 1, size=ref.shape), 0, mx)
    return np.ascontiguousarray(org.astype(np.int16)), np.ascontiguousarray(ref.astype(np.int16))


def level_case(which):
    """(org, ref) of the stage-B case (64-wide blocks on column stripes of half-period 1, every odd horizontal displacement fully mismatched) and of the
    wavefront case (half-period 2; shifts 1 and 3 alternate between neighbouring 64 x 64 blocks, so the upper and the left neighbour's vector is fully
    mismatched on the current block, while the first grid candidate (-8, -8) is only half mismatched)"""
    W, H = 328, 200
    if which == 'stage_b':
        return stripe_pair(31, W, H, 1, lambda bx, by: 2)
    return stripe_pair(32, W, H, 2, lambda bx, by: 1 if (bx + by) % 2 == 0 else 3)


def run_level(eng, which, bd=10):
    from vvenc_b200 import mctf_host as MH
    org, ref = level_case(which)
    H, W = org.shape
    po, pr = MH.pad_edge(org, MARGIN), MH.pad_edge(ref, MARGIN)
    eng.upload_plane(50, po, W, H, MARGIN, bd); eng.upload_plane(51, pr, W, H, MARGIN, bd)
    got = eng.mctf_estimate_level(50, 51, W, H, 64, None, 2, False)
    prov = Int64Provider(po, pr, MARGIN, bd)
    exp = MH.estimate_level(prov, W, H, 64, None, 2, False, bd)
    return got, exp, prov


@pytest.mark.gpu
def test_stage_b_integer_grid_64x64(eng):
    """vvb_mctf_estimate_level with 64 x 64 blocks: the integer grid (mctf_int_grid_kernel) sees SSEs of 4096 * ~1000^2 at every odd displacement"""
    got, exp, prov = run_level(eng, 'stage_b')
    assert prov.saturated > 100 and prov.exact_max > 2 ** 31 + 2 ** 30
    assert np.array_equal(got['x'], exp['x']) and np.array_equal(got['y'], exp['y']), (got['x'].tolist(), exp['x'].tolist())
    assert np.array_equal(got['error'], exp['error'])
    assert (exp['x'] == 32).mean() > 0.75 and (exp['error'] < INT_MAX).all()      # the true shift (2 pels) wherever the window stays inside the picture


@pytest.mark.gpu
def test_wavefront_neighbours_above_2_31(eng):
    """stage D (mctf_wave_kernel): the upper and the left neighbour's final vectors cost more than 2^31 on the current block; they must lose"""
    from vvenc_b200 import mctf_host as MH
    got, exp, prov = run_level(eng, 'wave')
    org, ref = level_case('wave')
    po, pr = MH.pad_edge(org, MARGIN), MH.pad_edge(ref, MARGIN)
    # the neighbour vectors really are above 2^31 on the blocks they are offered to
    byn, bxn = exp['x'].shape
    over = 0
    for by in range(byn):
        for bx in range(bxn):
            h = min(64, org.shape[0] - 64 * by) & ~7; w = min(64, org.shape[1] - 64 * bx) & ~7
            for (nx, ny) in ((bx, by - 1), (bx - 1, by)):
                if nx >= 0 and ny >= 0 and w == 64 and h == 64:
                    e = err_exact(po, pr, 64 * bx + MARGIN, 64 * by + MARGIN, int(exp['x'][ny, nx]), int(exp['y'][ny, nx]), w, h, 10, 0)
                    over += e > INT_MAX
    assert over >= 8
    assert np.array_equal(got['x'], exp['x']) and np.array_equal(got['y'], exp['y']), (got['x'].tolist(), exp['x'].tolist())
    assert np.array_equal(got['error'], exp['error'])


PYR_W, PYR_H = 520, 264


def pyramid_case(which):
    """unit-32 pyramid pictures: 'smooth' -- ordinary content (smoothed noise, a half-pel shift, noise); 'stripes' -- column stripes of half-period 16,
    which stay at full contrast down to the quarter-resolution level, shifted by 32 pels (a multiple of the period on every level)"""
    if which == 'stripes':
        return stripe_pair(41, PYR_W, PYR_H, 16, lambda bx, by: 32)
    rs = np.random.RandomState(40)
    W, H = PYR_W, PYR_H
    base = rs.randint(0, 1024, size=(H + 16, W + 16))
    sm = (base + np.roll(base, 1, 0) + np.roll(base, 1, 1) + np.roll(base, (1, 1), (0, 1))) // 4
    org = np.ascontiguousarray(sm[8:8 + H, 8:8 + W].astype(np.int16))
    a = sm[8 + 3:8 + 3 + H, 8 - 5:8 - 5 + W]; b = sm[8 + 3:8 + 3 + H, 8 - 4:8 - 4 + W]
    ref = np.ascontiguousarray(np.clip((a + b + 1) // 2 + rs.randint(-5, 6, size=org.shape), 0, 1023).astype(np.int16))
    return org, ref


def pyramid_expected(org, ref, check_first=True):
    from vvenc_b200 import mctf_host as MH
    provs = []

    def make_provider(o, r):
        provs.append(Int64Provider(MH.pad_edge(o, MARGIN), MH.pad_edge(r, MARGIN), MARGIN, 10, 0, check_first))
        return provs[-1]
    return MH.estimate_pyramid(make_provider, org, ref, 32, False, 10, 0), provs


def test_pyramid_unit32_replay_equals_reference_golden(golden_v7):
    """the host replay over the int64 errors equals the reference's own motionEstimationMCTF at unit 32 on in-range content (golden field)"""
    org, ref = pyramid_case('smooth')
    exp, provs = pyramid_expected(org, ref)
    assert max(p.exact_max for p in provs) <= INT_MAX
    g = golden_v7['pyramid_smooth']
    assert np.array_equal(exp['x'], g[..., 0]) and np.array_equal(exp['y'], g[..., 1])
    assert np.array_equal(exp['error'], g[..., 2]) and np.array_equal(exp['rmsme'].astype(np.int32), g[..., 3])


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["smooth", "stripes"])
def test_pyramid_unit32(eng, which):
    """vvb_mctf_estimate_pyramid at unit 32: 64 x 64 blocks on the three coarse levels, 32 x 32 on the final one"""
    org, ref = pyramid_case(which)
    H, W = org.shape
    from vvenc_b200 import mctf_host as MH
    eng.upload_plane(52, MH.pad_edge(org, MARGIN), W, H, MARGIN); eng.upload_plane(53, MH.pad_edge(ref, MARGIN), W, H, MARGIN)
    got = eng.mctf_estimate_pyramid(52, 53, W, H, 32, False, 0, False)
    exp, provs = pyramid_expected(org, ref)
    if which == 'stripes':
        assert sum(p.saturated for p in provs) > 100
    assert got.shape == exp['x'].shape
    assert np.array_equal(got['x'], exp['x']) and np.array_equal(got['y'], exp['y']), np.argwhere((got['x'] != exp['x']) | (got['y'] != exp['y']))[:6]
    assert np.array_equal(got['error'], exp['error']) and np.array_equal(got['rmsme'], exp['rmsme'])


# ---------------------------------------------------------------------------------------------------- apply
# label, W, H, unit, references, tap4, planar, content
APPLY_CASES = (('contrast, 8 references', 96, 64, 16, 8, 0, 1, 'contrast'), ('contrast, 4-tap', 64, 64, 32, 3, 1, 1, 'contrast'),
               ('unit 4, trailing 2', 42, 26, 4, 4, 1, 1, 'contrast'), ('unit 8, trailing 6 / 2', 70, 50, 8, 2, 0, 1, 'smooth'),
               ('unit 16, trailing 2 / 6', 66, 54, 16, 5, 0, 0, 'contrast'), ('planar clamp', 64, 48, 8, 4, 0, 1, 'ramps'))


def apply_case(k):
    """case dict of impls.mctf_apply_expected for APPLY_CASES[k]"""
    label, W, H, bs, n, tap4, planar, kind = APPLY_CASES[k]
    rs = np.random.RandomState(300 + k)
    mx, m = 1023, 24
    S = W + 2 * m
    yy, xx = np.mgrid[0:H + 2 * m, 0:S]
    if kind == 'contrast':                 # checkerboards at full range: the unclipped first pass overshoots both ends
        org = np.where((xx + yy) & 1, mx, 0)
        refs = [np.where(((xx + yy + r) & 1) if r % 3 else (xx & 1), mx, 0) for r in range(n)]
    elif kind == 'ramps':                  # 8-pel saw teeth of slope 146 against flat planes: the planar fit's b1 / b2 leave int16
        org = rs.randint(0, 4, size=yy.shape)
        saw = [np.clip(146 * (xx % 8), 0, mx), np.clip(146 * (yy % 8), 0, mx), mx - np.clip(146 * (xx % 8), 0, mx), mx - np.clip(146 * (yy % 8), 0, mx)]
        refs = [saw[r % 4] for r in range(n)]
    else:
        base = rs.randint(0, mx + 1, size=(H + 2 * m + 2, S + 2))
        org = (base[:-2, :-2] + base[1:-1, 1:-1] + base[2:, 2:] + base[1:-1, :-2]) // 4
        refs = [np.clip(org + rs.randint(-200, 201, size=org.shape), 0, mx) for _ in range(n)]
    nb = ((W + bs - 1) // bs) * ((H + bs - 1) // bs)
    mvs = np.zeros((n, nb, 4), dtype=np.int32)
    if kind == 'ramps':
        mvs[..., 0] = 16 * rs.randint(-1, 2, size=(n, nb)) * 8; mvs[..., 1] = 16 * rs.randint(-1, 2, size=(n, nb)) * 8   # whole teeth: the ramp stays in the block
    else:
        mvs[..., 0] = rs.randint(-16 * 6, 16 * 6 + 1, size=(n, nb)); mvs[..., 1] = rs.randint(-16 * 6, 16 * 6 + 1, size=(n, nb))
    mvs[..., 2] = rs.choice([3, 50, 101, 400, INT_MAX], size=(n, nb))
    mvs[..., 3] = rs.choice([0, 1, 23, 0xffff], size=(n, nb))
    mvs[0, ::2, 2] = INT_MAX; mvs[0, ::3, 3] = 0xffff
    strengths = np.array([0.85, 0.57, 0.41, 0.33, 0.30, 0.20, 0.18, 0.15][:n], dtype=np.float64)
    return dict(org=np.ascontiguousarray(org.astype(np.int16)), refs=[np.ascontiguousarray(r.astype(np.int16)) for r in refs], stride=S, margin=m, W=W, H=H,
                mvs=mvs, strengths=strengths, ws=0.4, sigma=9 * (128.0 + 3.0 / 256.0 * 32 ** 3), bs=bs, bd=10, num_refs=n), tap4, planar


def planar_clamps(case):
    """number of blocks whose planar fit clamps b1 or b2 to +-32767 (restated in Python from applyPlanarCorrectionCore, MCTF.cpp:372-420)"""
    m, bs = case['margin'], case['bs']
    hits = 0
    nbx = (case['W'] + bs - 1) // bs
    for r in range(case['num_refs']):
        for b in range(case['mvs'].shape[1]):
            mvx, mvy, _, rms = [int(v) for v in case['mvs'][r, b]]
            if rms == 0 or (mvx | mvy) & 15:
                continue
            bx, by = (b % nbx) * bs, (b // nbx) * bs
            w, h = min(bs, case['W'] - bx), min(bs, case['H'] - by)
            if w != h:
                continue
            o = case['org'][m + by:m + by + h, m + bx:m + bx + w].astype(np.int64)
            d = case['refs'][r][m + by + (mvy >> 4):m + by + (mvy >> 4) + h, m + bx + (mvx >> 4):m + bx + (mvx >> 4) + w].astype(np.int64)
            z = d - o
            n = w * h; xs = np.arange(w)[None, :]; ys = np.arange(h)[:, None]
            xsum = (n * (w - 1)) >> 1
            mw = min(rms * rms, 512)
            denom = n * [0, 1, 20, 336, 5440, 87296][int(np.log2(w))]
            for num in (mw * (int((xs * z).sum()) * n - xsum * int(z.sum())), mw * (int((ys * z).sum()) * n - xsum * int(z.sum()))):
                q = (num - (denom >> 1) if num < 0 else num + (denom >> 1))
                q = -((-q) // denom) if q < 0 else q // denom
                hits += abs(q) > 32767
    return hits


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(APPLY_CASES)))
def test_apply_extremes(eng, golden_v7, k):
    import impls
    case, tap4, planar = apply_case(k)
    W, H, m, n = case['W'], case['H'], case['margin'], case['num_refs']
    eng.upload_plane(0, case['org'], W, H, m)
    for r in range(n):
        eng.upload_plane(1 + r, case['refs'][r], W, H, m)
    V = _V()
    mv = np.zeros(case['mvs'].shape[:2], dtype=V.MCTF_MV_DT)
    mv['x'] = case['mvs'][..., 0]; mv['y'] = case['mvs'][..., 1]; mv['error'] = case['mvs'][..., 2]; mv['rmsme'] = case['mvs'][..., 3]
    got = eng.mctf_apply(0, list(range(1, 1 + n)), mv, case['bs'], case['strengths'], case['ws'], case['sigma'], W, H, planar=bool(planar), low_res_filter=bool(tap4))
    exp = impls.mctf_apply_expected(oracle(), 'orc', case, tap4, planar)
    assert np.array_equal(exp, golden_v7['apply_%d' % k]), APPLY_CASES[k][0]
    assert np.array_equal(got, exp), (APPLY_CASES[k][0], np.argwhere(got != exp)[:4])
    if APPLY_CASES[k][7] == 'ramps':
        assert planar_clamps(case) >= 8


# ---------------------------------------------------------------------------------------------------- admission
def _admission_calls(eng, o, r):
    """the five MCTF entries that had no bit-depth check, on planes o / r; each returns the library's status"""
    import vvenc_b200._lib as L
    V = _V()
    lib, h = eng.lib, eng.h
    c = np.zeros(2, dtype=V.MCTF_DT); c[0] = (0, 0, 17, -5, 16, 16); c[1] = (16, 8, 32, 0, 8, 8)
    e = np.zeros(2 * 9, dtype=np.int32); var = np.zeros(2, dtype=np.float64)
    out = np.zeros((24, 40), dtype=V.MCTF_MV_DT)
    lp = L.vvb_mctf_level_par(16, 2, 0, 0, 0, 0, 0, 40, 24)
    pp = L.vvb_mctf_pyr_par(8, 0, 0, 0)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    return {'error_batch': lib.vvb_mctf_error_batch(h, o, r, p(c), 2, 0, p(e)),
            'search_grid': lib.vvb_mctf_search_grid(h, o, r, p(c), 2, 16, 1, 0, p(e)),
            'calc_var': lib.vvb_mctf_calc_var(h, max(o, r), p(c), 2, p(var)),           # one plane: the wider one
            'estimate_level': lib.vvb_mctf_estimate_level(h, o, r, ctypes.byref(lp), None, p(out)),
            'estimate_pyramid': lib.vvb_mctf_estimate_pyramid(h, o, r, ctypes.byref(pp), p(out))}


@pytest.mark.gpu
def test_admission_up_to_10_bits(eng):
    import vvenc_b200._lib as L
    W, H = 320, 192
    rs = np.random.RandomState(5)
    for pid, bd in ((54, 10), (55, 11), (56, 12)):
        pl = rs.randint(0, 1 << 10, size=(H + 2 * MARGIN, W + 2 * MARGIN)).astype(np.int16)
        eng.upload_plane(pid, pl, W, H, MARGIN, bd)
    ok = _admission_calls(eng, 54, 54)
    assert all(v == L.VVB_OK for v in ok.values()), ok
    for (o, r) in ((55, 54), (54, 55), (56, 54), (54, 56), (55, 55), (56, 56)):
        rc = _admission_calls(eng, o, r)
        assert all(v == L.VVB_ERR_UNSUPPORTED for v in rc.values()), (o, r, rc)
        assert b'10 bit' in eng.lib.vvb_last_error(eng.h)


# ---------------------------------------------------------------------------------------------------- which kernels run
def kernel_selection_cases():
    """[(label, setup)] for tests/_kernel_selection_run.py: the stage-B case runs mctf_int_grid_kernel, the wavefront case mctf_wave_kernel"""
    from test_gpu_format_limits import ran
    cases = []
    for which, kernel in (('stage_b', 'mctf_int_grid_kernel'), ('wave', 'mctf_wave_kernel')):
        def setup(eng, which=which, kernel=kernel):
            from vvenc_b200 import mctf_host as MH
            org, ref = level_case(which)
            H, W = org.shape
            eng.upload_plane(50, MH.pad_edge(org, MARGIN), W, H, MARGIN); eng.upload_plane(51, MH.pad_edge(ref, MARGIN), W, H, MARGIN)
            return (lambda: eng.mctf_estimate_level(50, 51, W, H, 64, None, 2, False)), (lambda names: ran(names, kernel))
        cases.append(('MCTF level %s 64x64: %s' % (which, kernel), setup))
    return cases


@pytest.mark.gpu
def test_kernel_selection():
    import json, subprocess, sys
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_kernel_selection_run.py')
    out = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [script, 'test_gpu_mctf_limits'], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]
    assert [r['case'] for r in rows] == [label for label, _ in kernel_selection_cases()]
    assert [r for r in rows if not r['ok']] == [], rows
