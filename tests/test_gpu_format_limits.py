"""Search and distortion kernels at the limits of their number formats, bit for bit against the CPU oracle (64-bit sums, MV rate without a table):
  * 8 / 10 / 11 / 12-bit full-contrast planes through the dense search, both SAD-pyramid engines, the pattern kernels and the fractional grid
    (the in-CTA pyramid keeps 8x8 box sums of the window as uint16 lanes: 64 * 1023 fits, 64 * 2047 does not, so planes above 10 bits take engine 0),
  * both sides of the two host rules that choose 32-bit argmin keys, and the lambda limit of the 32-bit MV cost table,
  * MV rates of predictors at the ends of int16, lambda 0 on flat planes (every cost ties: the first vector wins),
  * distortions wider than 32 bits: exact through the uint64 entry points, saturated in the uint32 cost tables, and never deciding on a wrapped value."""
import math
import re
import struct
import numpy as np
import pytest
from _libs import oracle, P, PO

pytestmark = pytest.mark.gpu

OUTSIDE = 0xffffffff              # pattern cost of a point outside the search range
SAT_PATTERN = 0xfffffffe          # largest distortion a pattern cost table or vvb_best.sad reports
SAT_POOL = 0xffffffff             # largest distortion a pool cost reports
INVALID = (0, 0, 0xffffffff, 0xffffffffffffffff)


@pytest.fixture(scope="module")
def eng():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def _V():
    import vvenc_b200 as V
    return V


# ---------------------------------------------------------------------------------------------------- content
def contrast_planes(seed, W, H, m, bd_org, bd_ref=None, tile=64):
    """org / ref planes (margin m) of 64x64 tiles of three kinds: org near 0 under ref near the top of its bit depth, the opposite, and random pels"""
    bd_ref = bd_org if bd_ref is None else bd_ref
    rs = np.random.RandomState(seed)
    S = W + 2 * m
    shape = (H + 2 * m, S)
    ho, hr = (1 << bd_org) - 1, (1 << bd_ref) - 1
    org = rs.randint(0, ho + 1, size=shape)
    ref = rs.randint(0, hr + 1, size=shape)
    ty = (np.arange(shape[0]) - m) // tile
    tx = (np.arange(shape[1]) - m) // tile
    kind = (ty[:, None] + tx[None, :]) % 3
    lo_o, lo_r = rs.randint(0, 4, size=shape), rs.randint(0, 4, size=shape)
    org = np.where(kind == 0, lo_o, np.where(kind == 1, ho - lo_o, org))
    ref = np.where(kind == 0, hr - lo_r, np.where(kind == 1, lo_r, ref))
    return np.ascontiguousarray(org.astype(np.int16)), np.ascontiguousarray(ref.astype(np.int16)), S


def upload(eng, org, ref, W, H, m, bd_org, bd_ref=None):
    eng.upload_plane(0, org, W, H, m, bd_org)
    eng.upload_plane(1, ref, W, H, m, bd_org if bd_ref is None else bd_ref)


def kernel_names(fn):
    """result of fn() and the names in a torch.profiler trace of it (tests/_kernel_selection_run.py).  A trace now and then holds the API calls but no
    kernel record at all; the call is repeated then (every call profiled here is a pure function of its inputs)."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        if any('_kernel' in n for n in names):
            break
    return out, names


def ran(names, kernel):
    return any(kernel in n for n in names)


def key32_flags(names):
    """KEY32 template argument of every sad_search_kernel<USE_TMA, PARENT, KEY32> launch with PARENT = true"""
    out = set()
    for n in names:
        mm = re.search(r'sad_search_kernel<(\w+), (\w+), (\w+)>', n)
        if mm and mm.group(2) == 'true':
            out.add(mm.group(3) == 'true')
    return out


# ---------------------------------------------------------------------------------------------------- host rules, restated
def mv_cost_max(lam):
    """last entry of the MV cost table: Distortion( sqrt(lambda) * 79 ) in IEEE double, as makeMePar computes it"""
    return int(math.sqrt(lam) * 79)


def order_bits(positions):
    ob = 1
    while (1 << ob) < positions:
        ob += 1
    return ob


def in_cta_rule(bd, nx, ny, lam):
    """pyramidV2Usable for an 8x8 base: planes up to 10 bits, 16x16 cost (4 * 64 pels + MV cost) below 2^(32 - ob) and PYR_NEVER / 4"""
    ob = order_bits(nx * ny)
    c = 256 * ((1 << bd) - 1) + mv_cost_max(lam)
    return bd <= 10 and ob <= 16 and c < (1 << (32 - ob)) and c < (1 << 24)


def key32_rule(bd, nx, ny, lam, w=8):
    """32-bit keys of the round-1 base kernel (sadSearchLaunch): parent cost (4 members of w x w + MV cost) below 2^(32 - ob) - 1"""
    ob = order_bits(nx * ny)
    c = 4 * w * w * ((1 << bd) - 1) + mv_cost_max(lam)
    return ob <= 16 and c < (1 << (32 - ob)) - 1


def lambda_edge(ok):
    """(largest double lambda with ok(lambda), the next double above it); ok holds at 0 and fails at 1e300 and changes once"""
    f2i = lambda f: struct.unpack('<q', struct.pack('<d', f))[0]
    i2f = lambda i: struct.unpack('<d', struct.pack('<q', i))[0]
    a, b = f2i(0.0), f2i(1e300)
    assert ok(0.0) and not ok(1e300)
    while b - a > 1:
        mid = (a + b) // 2
        if ok(i2f(mid)):
            a = mid
        else:
            b = mid
    return i2f(a), i2f(b)


# ---------------------------------------------------------------------------------------------------- oracle replays
def replay(org, ref, S, m, rows, lam, cost_scale=2, imv_shift=0, sub_shift=0, table_stride=0):
    """xPatternSearch of every row (x, y, w, h, left, right, top, bottom, pred_hor, pred_ver) -> dx, dy, 64-bit cost (+ SAD tables)"""
    O = oracle()
    rows = np.ascontiguousarray(rows, dtype=np.int32)
    n = len(rows)
    out = np.zeros((n, 4), dtype=np.int32)
    tab = np.zeros((n, max(1, table_stride)), dtype=np.uint32)
    base = m * S + m
    O.orc_full_search(PO(org, base), S, PO(ref, base), S, P(rows), n, sub_shift, float(lam), cost_scale, imv_shift, P(out),
                      P(tab) if table_stride else None, table_stride)
    cost = out[:, 2].view(np.uint32).astype(np.uint64) | (out[:, 3].view(np.uint32).astype(np.uint64) << np.uint64(32))
    res = (out[:, 0].astype(np.int64), out[:, 1].astype(np.int64), cost)
    return (res, tab) if table_stride else res


def block_rows(bl, size):
    return np.stack([bl['x'], bl['y'], np.full(len(bl), size), np.full(len(bl), size), bl['left'], bl['right'], bl['top'], bl['bottom'],
                     bl['pred_hor'], bl['pred_ver']], axis=1).astype(np.int32)


def assert_best(got, exp, what):
    dx, dy, cost = exp
    bad = [i for i in range(len(got)) if (int(got['dx'][i]), int(got['dy'][i]), int(got['cost'][i])) != (int(dx[i]), int(dy[i]), int(cost[i]))]
    assert bad == [], (what, len(bad), [(i, (int(got['dx'][i]), int(got['dy'][i]), int(got['cost'][i])), (int(dx[i]), int(dy[i]), int(cost[i]))) for i in bad[:4]])


def pyramid_levels(W, H, rng, rs, pred=None):
    V = _V()
    blks = []
    for (xs, ys) in V.candidates.pyramid_lists(8, 4, W, H):
        bl = np.zeros(len(xs), dtype=V.BLOCK_DT)
        bl['x'] = xs; bl['y'] = ys; bl['left'], bl['right'], bl['top'], bl['bottom'] = rng
        if pred is None:
            bl['pred_hor'] = rs.randint(-60, 61, len(xs)); bl['pred_ver'] = rs.randint(-60, 61, len(xs))
        else:
            bl['pred_hor'] = pred[0][np.arange(len(xs)) % len(pred[0])]; bl['pred_ver'] = pred[1][np.arange(len(xs)) % len(pred[1])]
        blks.append(bl)
    return blks


def check_pyramid(res, blks, org, ref, S, m, lam, roots=None, imv_shift=0, what=''):
    """every block of every level (or the trees of `roots` plus every block outside the 64x64 trees) against the replay"""
    n64 = len(blks[3])
    for l in range(4):
        n = 1 << (2 * (3 - l))
        if roots is None:
            idx = np.arange(len(blks[l]))
        else:
            idx = np.concatenate([np.arange(r * n, (r + 1) * n) for r in roots] + [np.arange(n64 * n, len(blks[l]))])
        exp = replay(org, ref, S, m, block_rows(blks[l][idx], 8 << l), lam, 2, imv_shift)
        assert_best(res[l][idx], exp, (what, 'level', l))


# ---------------------------------------------------------------------------------------------------- bit depth through the integer search
PYR_W = PYR_H = 64 * 12 + 56            # 144 roots of 64x64 (more than SMs: runs of two carry the window), then 32 / 16 / 8 roots right and below
PYR_CHECK = [0, 1, 10, 11, 12, 13, 70, 71, 72, 131, 142, 143]


@pytest.mark.parametrize("r", [8, 16, 32])
@pytest.mark.parametrize("bd", [8, 10, 11, 12])
def test_pyramid_full_contrast(eng, bd, r):
    """both pyramid engines on full-contrast planes: 8x8 box sums of the window at their format limit (64 * 1023 at 10 bits) and beyond it.
    Which engine runs is checked by test_kernel_selection."""
    m = 48
    org, ref, S = contrast_planes(100 + bd, PYR_W, PYR_H, m, bd)
    upload(eng, org, ref, PYR_W, PYR_H, m, bd)
    rs = np.random.RandomState(r)
    blks = pyramid_levels(PYR_W, PYR_H, (-r, r, -r, r), rs)
    lam = 61.5
    par = eng.me_par(lam, 2, 0, 0)
    try:
        for engine in (1, 0):
            eng.set_pyramid_engine(engine)
            res = eng.sad_search_pyramid(0, 1, blks, 8, par, 2 * r + 1, 2 * r + 1)
            check_pyramid(res, blks, org, ref, S, m, lam, roots=PYR_CHECK, what=(bd, r, engine))
    finally:
        eng.set_pyramid_engine(1)


def search_blocks(rs, size, W, H, quads, rng):
    V = _V()
    if quads:
        xs, ys = V.candidates.quad_order_grid(size, W, H)
    else:                                               # scattered blocks, odd columns included: one block per CTA, 16-bit window staging
        n = 12
        xs = np.minimum(rs.randint(0, (W - size) // 4 + 1, n) * 4 + rs.randint(0, 2, n), W - size); ys = rs.randint(0, H - size + 1, n)
    bl = np.zeros(len(xs), dtype=V.BLOCK_DT)
    bl['x'] = xs; bl['y'] = ys; bl['left'], bl['right'], bl['top'], bl['bottom'] = rng
    bl['pred_hor'] = rs.randint(-60, 61, len(xs)); bl['pred_ver'] = rs.randint(-60, 61, len(xs))
    return bl


@pytest.mark.parametrize("bd", [8, 10, 11, 12])
def test_dense_search_full_contrast(eng, bd):
    """vvb_sad_search (best vectors and SAD tables) on full-contrast planes: z-order quads and single blocks, TMA window staging on and off"""
    W, H, m = 256, 192, 48
    org, ref, S = contrast_planes(200 + bd, W, H, m, bd)
    upload(eng, org, ref, W, H, m, bd)
    rs = np.random.RandomState(bd)
    lam = 33.5
    try:
        for tma in (1, 0):
            eng.set_tma_staging(tma)
            for size in (8, 16, 32, 64):
                for quads in (True, False):
                    rng = (-16, 16, -13, 15)
                    bl = search_blocks(rs, size, W, H, quads, rng)
                    best, tab = eng.sad_search(0, 1, bl, size, size, eng.me_par(lam, 2, 0, 0), want_tables=True)
                    exp, etab = replay(org, ref, S, m, block_rows(bl, size), lam, table_stride=tab.shape[1])
                    assert_best(best, exp, (bd, tma, size, quads))
                    assert np.array_equal(tab, etab), (bd, tma, size, quads, np.argwhere(tab != etab)[:4])
    finally:
        eng.set_tma_staging(2)


RING = [(0, 0)] + [(dx, dy) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dx or dy] + [(dx, dy) for dy in (-2, 0, 2) for dx in (-2, 0, 2) if dx or dy] + \
       [(3, -7), (-8, 8), (0, 0)]
WIDE = RING + [(12, -9), (-11, 10)]


def mv_pattern(pts):
    pat = np.zeros(len(pts), dtype=_V().MV_DT)
    pat['dx'] = [p[0] for p in pts]; pat['dy'] = [p[1] for p in pts]
    return pat


def pattern_blocks(rs, n, w, h, W, H, rng=(-20, 18, -16, 20), pred=None):
    V = _V()
    bl = np.zeros(n, dtype=V.BLOCK_DT)
    bl['x'] = np.minimum(rs.randint(0, (W - w) // 4 + 1, n) * 4 + rs.randint(0, 2, n), W - w); bl['y'] = rs.randint(0, H - h + 1, n)
    bl['left'], bl['right'], bl['top'], bl['bottom'] = rng
    if pred is None:
        bl['pred_hor'] = rs.randint(-60, 61, n); bl['pred_ver'] = rs.randint(-60, 61, n)
    else:
        bl['pred_hor'] = pred[0][np.arange(n) % len(pred[0])]; bl['pred_ver'] = pred[1][np.arange(n) % len(pred[1])]
    bl['start_x'] = rs.randint(-9, 10, n); bl['start_y'] = rs.randint(-9, 10, n)
    return bl


def expect_pattern(fam, org, ref, S, m, bl, w, h, pat, lam, imv_shift=0):
    """cost table (inside: min(distortion, 0xfffffffe), outside: 0xffffffff) and best (dx, dy, sad, 64-bit cost) of the pattern, first strictly smaller wins"""
    O = oracle()
    base = m * S + m
    cost = np.zeros((len(bl), len(pat)), dtype=np.uint64)
    best = []
    for bi, b in enumerate(bl):
        x, y = int(b['x']), int(b['y'])
        bc = None
        for k in range(len(pat)):
            mx, my = int(b['start_x']) + int(pat['dx'][k]), int(b['start_y']) + int(pat['dy'][k])
            if not (b['left'] <= mx <= b['right'] and b['top'] <= my <= b['bottom']):
                cost[bi, k] = OUTSIDE
                continue
            d = O.orc_dist(fam, PO(org, base + y * S + x), S, PO(ref, base + (y + my) * S + x + mx), S, w, h, 0)
            cost[bi, k] = min(d, SAT_PATTERN)
            c = d + O.orc_mv_cost(float(lam), mx, my, int(b['pred_hor']), int(b['pred_ver']), 2, imv_shift)
            if bc is None or c < bc[3]:
                bc = (mx, my, min(d, SAT_PATTERN), c)
        best.append(INVALID if bc is None else bc)
    return cost, best


def check_pattern(eng, fam, org, ref, S, m, bl, w, h, pat, lam, imv_shift=0, what=''):
    V = _V()
    par = eng.me_par(lam, 2, imv_shift, 0)
    call = (lambda: eng.sad_pattern(0, 1, bl, w, h, pat, par)) if fam == V.DF_SAD else (lambda: eng.cost_pattern(fam, 0, 1, bl, w, h, pat, par))
    cost, best = call()
    ecost, ebest = expect_pattern(fam, org, ref, S, m, bl, w, h, pat, lam, imv_shift)
    bad = np.argwhere(cost != ecost)
    assert len(bad) == 0, (what, fam, w, h, [(tuple(i), int(cost[tuple(i)]), int(ecost[tuple(i)])) for i in bad[:3]])
    got = [(int(b['dx']), int(b['dy']), int(b['sad']), int(b['cost'])) for b in best]
    assert got == ebest, (what, fam, w, h, [(i, g, e) for i, (g, e) in enumerate(zip(got, ebest)) if g != e][:3])


def pattern_cases():
    V = _V()
    return [(V.DF_SAD, 16, 16, RING, None), (V.DF_SAD, 64, 64, WIDE, None),
            (V.DF_HAD, 8, 8, RING, 'had8_direct_kernel'), (V.DF_HAD, 16, 16, RING, 'had8_ring_kernel'), (V.DF_HAD, 32, 32, RING, 'had8_ring_kernel'),
            (V.DF_HAD, 64, 64, RING, 'had8_ring_kernel'), (V.DF_HAD, 16, 16, WIDE, 'cost_pattern_kernel'), (V.DF_HAD, 16, 8, RING, 'cost_pattern_kernel'),
            (V.DF_SSE, 32, 32, RING, 'cost_pattern_kernel'), (V.DF_SSE, 128, 128, RING, 'cost_pattern_kernel')]


@pytest.mark.parametrize("bd", [8, 10, 11, 12])
def test_patterns_full_contrast(eng, bd):
    """vvb_sad_pattern and vvb_cost_pattern on full-contrast planes: SAD, SSE (above 32 bits for 128x128 at 10 bits and 32x32 at 12: the table saturates,
    the decision does not), HAD on had8_direct_kernel, had8_ring_kernel (packed differences up to 10 bits) and the generic kernel"""
    W, H, m = 256, 192, 48
    org, ref, S = contrast_planes(300 + bd, W, H, m, bd)
    upload(eng, org, ref, W, H, m, bd)
    rs = np.random.RandomState(30 + bd)
    for (fam, w, h, pts, _) in pattern_cases():
        bl = pattern_blocks(rs, 6, w, h, W, H)
        check_pattern(eng, fam, org, ref, S, m, bl, w, h, mv_pattern(pts), 21.0, what=bd)


def test_mixed_bit_depths(eng):
    """a 12-bit original against an 8-bit reference: the key-width rules and the pyramid routing take the wider of the two bit depths"""
    W, H, m, r = 64 * 4 + 56, 64 * 2 + 56, 48, 32
    org, _, S = contrast_planes(400, W, H, m, 12)
    _, ref, _ = contrast_planes(401, W, H, m, 8)
    upload(eng, org, ref, W, H, m, 12, 8)
    rs = np.random.RandomState(4)
    lam = 61.5
    blks = pyramid_levels(W, H, (-r, r, -r, r), rs)
    try:
        for engine in (1, 0):
            eng.set_pyramid_engine(engine)
            res = eng.sad_search_pyramid(0, 1, blks, 8, eng.me_par(lam, 2, 0, 0), 2 * r + 1, 2 * r + 1)
            check_pyramid(res, blks, org, ref, S, m, lam, what=('mixed', engine))
    finally:
        eng.set_pyramid_engine(1)
    for size in (8, 32):
        bl = search_blocks(rs, size, W, H, True, (-r, r, -r, r))
        best = eng.sad_search(0, 1, bl, size, size, eng.me_par(lam, 2, 0, 0))
        assert_best(best, replay(org, ref, S, m, block_rows(bl, size), lam), ('mixed dense', size))
    V = _V()
    for w in (8, 32):                                              # had8_direct_kernel, had8_ring_kernel<false, ..>
        bl = pattern_blocks(rs, 6, w, w, W, H)
        check_pattern(eng, V.DF_HAD, org, ref, S, m, bl, w, w, mv_pattern(RING), 21.0, what='mixed')


def test_frac_grid_12bit(eng):
    """vvb_frac_cost_grid at 12 bits (entry point limit) on full-contrast planes: the register-tile kernel (square 8..64) and the generic one, every filter set"""
    V = _V()
    W, H, m, bd = 256, 192, 48, 12
    org, ref, S = contrast_planes(500, W, H, m, bd)
    upload(eng, org, ref, W, H, m, bd)
    rs = np.random.RandomState(5)
    O = oracle()
    fams = {1: V.DF_SAD, 2: V.DF_HAD, 3: V.DF_HAD_FAST}
    shapes = [(1, 8, 8), (2, 8, 8), (2, 16, 16), (1, 32, 32), (2, 64, 64), (2, 16, 8), (3, 32, 32), (1, 4, 16)]
    for li, (fam, w, h) in enumerate(shapes):
        n = 5
        b = np.zeros((n, 6), dtype=np.int32)
        for k in range(n):
            b[k] = (int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1)), w, h, int(rs.randint(-9, 10)), int(rs.randint(-9, 10)))
        blk = np.zeros(n, dtype=V.BLOCK_DT)
        blk['x'] = b[:, 0]; blk['y'] = b[:, 1]; blk['start_x'] = b[:, 4]; blk['start_y'] = b[:, 5]
        rt, alt = ((2, 0), (0, 0), (1, 0), (2, 1))[li % 4]
        if w * h == 16:
            rt = 2
        got = eng.frac_cost_grid(fams[fam], 0, 1, blk, w, h, rt, alt)
        exp = np.zeros((n, 7, 7), dtype=np.uint32)
        base = m * S + m
        O.orc_frac_cost_grid(PO(org, base), S, PO(ref, base), S, P(np.ascontiguousarray(b)), n, fam, bd, rt, alt, P(exp))
        assert np.array_equal(got, exp), (fam, w, h, rt, alt, np.argwhere(got != exp)[:5])


# ---------------------------------------------------------------------------------------------------- key-width thresholds
THR_W = THR_H = 64 * 2 + 56


@pytest.mark.parametrize("bd,r", [(10, 32), (8, 16)])
def test_in_cta_rule_both_sides(eng, bd, r):
    """the largest lambda the in-CTA rule admits and the next double both equal the replay on full-contrast planes (the first runs sad_pyramid8_kernel,
    the second does not: test_kernel_selection)"""
    m, n = 48, 2 * r + 1
    org, ref, S = contrast_planes(600 + bd, THR_W, THR_H, m, bd)
    upload(eng, org, ref, THR_W, THR_H, m, bd)
    blks = pyramid_levels(THR_W, THR_H, (-r, r, -r, r), np.random.RandomState(6))
    lam_in, lam_out = lambda_edge(lambda l: in_cta_rule(bd, n, n, l))
    assert in_cta_rule(bd, n, n, lam_in) and not in_cta_rule(bd, n, n, lam_out)
    for lam in (lam_in, lam_out):
        res = eng.sad_search_pyramid(0, 1, blks, 8, eng.me_par(lam, 2, 0, 0), n, n)
        check_pyramid(res, blks, org, ref, S, m, lam, what=(bd, r, lam))


@pytest.mark.parametrize("bd,r,engine", [(10, 16, 0), (12, 8, 1)])
def test_key32_rule_both_sides(eng, bd, r, engine):
    """the largest lambda the round-1 base kernel's 32-bit key rule admits and the next double both equal the replay on full-contrast planes (the first
    runs sad_search_kernel<.., true, true>, the second the 64-bit keys; at 12 bits the pyramid goes to engine 0 whatever engine is selected)"""
    m, n = 48, 2 * r + 1
    org, ref, S = contrast_planes(700 + bd, THR_W, THR_H, m, bd)
    upload(eng, org, ref, THR_W, THR_H, m, bd)
    blks = pyramid_levels(THR_W, THR_H, (-r, r, -r, r), np.random.RandomState(7))
    lam_in, lam_out = lambda_edge(lambda l: key32_rule(bd, n, n, l))
    assert key32_rule(bd, n, n, lam_in) and not key32_rule(bd, n, n, lam_out)
    try:
        eng.set_pyramid_engine(engine)
        for lam in (lam_in, lam_out):
            res = eng.sad_search_pyramid(0, 1, blks, 8, eng.me_par(lam, 2, 0, 0), n, n)
            check_pyramid(res, blks, org, ref, S, m, lam, what=(bd, r, lam))
    finally:
        eng.set_pyramid_engine(1)


def test_lambda_limit_of_the_mv_cost_table(eng):
    """the largest lambda whose MV cost table fits 32 bits searches exactly (dense, pyramid, pattern); the next double is VVB_ERR_UNSUPPORTED everywhere"""
    from vvenc_b200 import _lib as L
    V = _V()
    W, H, m, bd = THR_W, THR_H, 48, 10
    org, ref, S = contrast_planes(800, W, H, m, bd)
    upload(eng, org, ref, W, H, m, bd)
    rs = np.random.RandomState(8)
    lam_max, lam_rej = lambda_edge(lambda l: mv_cost_max(l) <= 0xffffffff)
    blks = pyramid_levels(W, H, (-8, 8, -8, 8), rs)
    bl = search_blocks(rs, 16, W, H, True, (-8, 8, -8, 8))
    pb = pattern_blocks(rs, 6, 16, 16, W, H)
    res = eng.sad_search_pyramid(0, 1, blks, 8, eng.me_par(lam_max, 2, 0, 0), 17, 17)
    check_pyramid(res, blks, org, ref, S, m, lam_max, what='lambda max')
    assert_best(eng.sad_search(0, 1, bl, 16, 16, eng.me_par(lam_max, 2, 0, 0)), replay(org, ref, S, m, block_rows(bl, 16), lam_max), 'lambda max dense')
    check_pattern(eng, V.DF_SAD, org, ref, S, m, pb, 16, 16, mv_pattern(RING), lam_max, what='lambda max')
    check_pattern(eng, V.DF_HAD, org, ref, S, m, pb, 16, 16, mv_pattern(RING), lam_max, what='lambda max')
    par = eng.me_par(lam_rej, 2, 0, 0)
    for call in (lambda: eng.sad_search_pyramid(0, 1, blks, 8, par, 17, 17), lambda: eng.sad_search(0, 1, bl, 16, 16, par),
                 lambda: eng.sad_pattern(0, 1, pb, 16, 16, mv_pattern(RING), par), lambda: eng.cost_pattern(V.DF_HAD, 0, 1, pb, 16, 16, mv_pattern(RING), par)):
        with pytest.raises(V.VvbError) as ei:
            call()
        assert ei.value.code == L.VVB_ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------- MV-rate extremes
@pytest.mark.parametrize("imv", [0, 1, 2])
def test_mv_rate_extreme_predictors(eng, imv):
    """predictors at -32768 / +32767: about 33 bits per component, near the end of the 80-entry rate table and of the pyramid's bit-count bytes"""
    V = _V()
    W, H, m, bd = THR_W, THR_H, 48, 10
    org, ref, S = contrast_planes(900 + imv, W, H, m, bd)
    upload(eng, org, ref, W, H, m, bd)
    rs = np.random.RandomState(90 + imv)
    pred = (np.array([-32768, 32767, -32768, 32767, 5], dtype=np.int16), np.array([-32768, -32768, 32767, 32767, -7], dtype=np.int16))
    lam = 80.0
    par = eng.me_par(lam, 2, imv, 0)
    blks = pyramid_levels(W, H, (-12, 12, -12, 12), rs, pred)
    try:
        for engine in (1, 0):
            eng.set_pyramid_engine(engine)
            res = eng.sad_search_pyramid(0, 1, blks, 8, par, 25, 25)
            check_pyramid(res, blks, org, ref, S, m, lam, imv_shift=imv, what=('mv', imv, engine))
    finally:
        eng.set_pyramid_engine(1)
    for size in (8, 16):
        bl = search_blocks(rs, size, W, H, True, (-12, 12, -12, 12))
        bl['pred_hor'] = pred[0][np.arange(len(bl)) % 5]; bl['pred_ver'] = pred[1][np.arange(len(bl)) % 5]
        assert_best(eng.sad_search(0, 1, bl, size, size, par), replay(org, ref, S, m, block_rows(bl, size), lam, 2, imv), ('mv dense', imv, size))
    for (fam, w, pts) in ((V.DF_SAD, 16, WIDE), (V.DF_HAD, 8, RING), (V.DF_HAD, 16, RING), (V.DF_HAD, 16, WIDE)):   # generic, direct, ring, generic
        bl = pattern_blocks(rs, 10, w, w, W, H, pred=pred)
        check_pattern(eng, fam, org, ref, S, m, bl, w, w, mv_pattern(pts), lam, imv_shift=imv, what=('mv', imv))


def test_lambda_zero_on_flat_planes(eng):
    """lambda 0 on flat planes: every cost is 0, so the first vector in evaluation order wins (top-left of the range, the first pattern point inside it)"""
    V = _V()
    W, H, m, bd = THR_W, THR_H, 48, 10
    S = W + 2 * m
    flat = np.full((H + 2 * m, S), 611, dtype=np.int16)
    upload(eng, flat, flat.copy(), W, H, m, bd)
    rs = np.random.RandomState(10)
    par = eng.me_par(0.0, 2, 0, 0)
    rng = (-7, 9, -5, 11)
    blks = pyramid_levels(W, H, rng, rs)
    try:
        for engine in (1, 0):
            eng.set_pyramid_engine(engine)
            res = eng.sad_search_pyramid(0, 1, blks, 8, par, 17, 17)
            check_pyramid(res, blks, flat, flat, S, m, 0.0, what=('flat', engine))
            for l in range(4):
                assert (res[l]['dx'] == rng[0]).all() and (res[l]['dy'] == rng[2]).all() and (res[l]['cost'] == 0).all(), (engine, l)
    finally:
        eng.set_pyramid_engine(1)
    for size in (8, 32):
        bl = search_blocks(rs, size, W, H, True, rng)
        best = eng.sad_search(0, 1, bl, size, size, par)
        assert_best(best, replay(flat, flat, S, m, block_rows(bl, size), 0.0), ('flat dense', size))
        assert (best['dx'] == rng[0]).all() and (best['dy'] == rng[2]).all()
    pat = mv_pattern([(-30, 0), (5, 3), (0, 0), (-1, -1), (1, 1)] + RING)     # the first point is outside every range: the second one wins
    for (fam, w) in ((V.DF_SAD, 16), (V.DF_HAD, 8), (V.DF_HAD, 16)):            # radius 30: the generic kernel
        bl = pattern_blocks(rs, 6, w, w, W, H, rng=(-20, 20, -20, 20))
        bl['start_x'] = 0; bl['start_y'] = 0
        check_pattern(eng, fam, flat, flat, S, m, bl, w, w, pat, 0.0, what='flat')
    for (fam, w) in ((V.DF_HAD, 8), (V.DF_HAD, 32)):                           # had8_direct_kernel, had8_ring_kernel
        bl = pattern_blocks(rs, 6, w, w, W, H, rng=(-20, 20, -20, 20))
        check_pattern(eng, fam, flat, flat, S, m, bl, w, w, mv_pattern(RING), 0.0, what='flat')


# ---------------------------------------------------------------------------------------------------- distortions wider than 32 bits
def contrast_blocks(rs, w, h, bd):
    """(org, cur) pairs: org 0 under cur at the maximum, opposite checkerboards, random pels"""
    hi = (1 << bd) - 1
    chk = (np.add.outer(np.arange(h), np.arange(w)) & 1) * hi
    return [(np.zeros((h, w)), np.full((h, w), hi)), (chk, hi - chk), (rs.randint(0, hi + 1, (h, w)), rs.randint(0, hi + 1, (h, w)))]


@pytest.mark.parametrize("bd,w,h", [(10, 64, 64), (10, 128, 64), (10, 128, 128), (12, 32, 32), (12, 64, 32), (12, 128, 128)])
def test_wide_distortions(eng, bd, w, h):
    """SSE / SAD / HAD / HAD_2SAD of full-contrast blocks: exact through vvb_dist_block and vvb_dist_batch (uint64), saturated at 0xffffffff through
    vvb_dist_pool on 8-aligned positions (streaming kernels) and unaligned ones (generic kernel)"""
    V = _V()
    O = oracle()
    rs = np.random.RandomState(bd * 1000 + w + h)
    pairs = contrast_blocks(rs, w, h, bd)
    nb, m = len(pairs), 16
    W, H = nb * (w + 16), h + 8
    S = W + 2 * m
    org = np.zeros((H + 2 * m, S), dtype=np.int16); cur = np.zeros_like(org)
    pos = np.array([(k * (w + 16), 4) for k in range(nb)])
    for k, (o, c) in enumerate(pairs):
        org[m + 4:m + 4 + h, m + pos[k, 0]:m + pos[k, 0] + w] = o; cur[m + 4:m + 4 + h, m + pos[k, 0]:m + pos[k, 0] + w] = c
    eng.upload_plane(2, org, W, H, m, bd); eng.upload_plane(3, cur, W, H, m, bd)
    base = m * S + m
    fams = (V.DF_SSE, V.DF_SAD, V.DF_HAD, V.DF_HAD_2SAD)
    exact = {}
    for fam in fams:
        for k in range(nb):
            o = base + 4 * S + int(pos[k, 0])
            e = O.orc_dist(fam, PO(org, o), S, PO(cur, o), S, w, h, 0)
            exact[fam, k] = e
            oc = np.ascontiguousarray(pairs[k][0].astype(np.int16)); cc = np.ascontiguousarray(pairs[k][1].astype(np.int16))
            assert eng.dist_block(fam, oc, w, cc, w, w, h, bd) == e, ('block', fam, k)
    if bd == 10 and (w, h) == (64, 64):
        assert exact[V.DF_SSE, 0] == 4096 * 1023 ** 2 < 1 << 32         # the largest 10-bit SSE that still fits 32 bits
    if (w, h) != (64, 64) or bd == 12:
        assert exact[V.DF_SSE, 0] >= 1 << 32
    cands = np.zeros(len(fams) * nb, dtype=V.CAND_DT)
    for i, (fam, k) in enumerate((f, k) for f in fams for k in range(nb)):
        cands[i] = (2, int(pos[k, 0]), 4, 3, int(pos[k, 0]), 4, w, h, fam, 0, (0, 0))
    got = eng.dist_batch(cands)
    assert [int(v) for v in got] == [exact[f, k] for f in fams for k in range(nb)]
    # pool: K = 3 candidates (the three cur blocks) per original block; positions 8-aligned, then one pel off
    pool = np.stack([np.stack([p[1] for p in pairs]) for _ in range(nb)]).astype(np.int16)
    for shift in (0, 1):
        blocks = np.zeros(nb, dtype=V.POS_DT)
        blocks['x'] = pos[:, 0] + shift; blocks['y'] = 4
        if shift:                                          # the originals move with the positions
            org2 = np.zeros_like(org)
            org2[:, shift:] = org[:, :-shift]
            eng.upload_plane(2, org2, W, H, m, bd)
        else:
            org2 = org
        for fam in fams:
            out = eng.dist_pool(fam, 2, blocks, w, h, nb, pool)
            for bi in range(nb):
                for k in range(nb):
                    e = O.orc_dist(fam, PO(org2, base + 4 * S + int(blocks['x'][bi])), S, P(np.ascontiguousarray(pool[bi, k])), w, w, h, 0)
                    assert int(out[bi, k]) == min(e, SAT_POOL), (fam, shift, bi, k, int(out[bi, k]), e)


def test_sse_pattern_decides_on_the_full_distortion(eng):
    """12-bit 32x32 blocks of constant pels: at (0, 0) the SSE is exactly 2^32 (0 when truncated to 32 bits), at (32, 0) it is 4 286 578 688; the exact
    minimum is (32, 0), the truncated one would be (0, 0)"""
    V = _V()
    O = oracle()
    bd, w, m, T = 12, 32, 48, 32
    W = H = 8 * T
    S = W + 2 * m
    org = np.full((H + 2 * m, S), 4095, dtype=np.int16)
    ref = np.full_like(org, 1000)
    at = lambda tx, ty: (slice(m + ty * T, m + (ty + 1) * T), slice(m + tx * T, m + (tx + 1) * T))
    ref[at(2, 2)] = 2047; ref[at(3, 2)] = 2049; ref[at(2, 5)] = 2047; ref[at(1, 5)] = 2049
    upload(eng, org, ref, W, H, m, bd)
    pat = mv_pattern([(0, 0), (32, 0), (-32, 0), (0, 32), (0, -32)])
    bl = np.zeros(2, dtype=V.BLOCK_DT)
    bl['x'] = [2 * T, 2 * T]; bl['y'] = [2 * T, 5 * T]; bl['left'], bl['right'], bl['top'], bl['bottom'] = (-40, 40, -40, 40)
    bl['pred_hor'] = [3, -3]; bl['pred_ver'] = [0, 4]
    lam = 4.0
    base = m * S + m
    for bi in range(2):
        x, y = int(bl['x'][bi]), int(bl['y'][bi])
        d = [O.orc_dist(V.DF_SSE, PO(org, base + y * S + x), S, PO(ref, base + (y + int(p['dy'])) * S + x + int(p['dx'])), S, w, w, 0) for p in pat]
        mv = [O.orc_mv_cost(lam, int(p['dx']), int(p['dy']), int(bl['pred_hor'][bi]), int(bl['pred_ver'][bi]), 2, 0) for p in pat]
        exact = int(np.argmin([a + b for a, b in zip(d, mv)]))
        wrapped = int(np.argmin([(a & 0xffffffff) + b for a, b in zip(d, mv)]))
        assert d[0] == 1 << 32 and exact != wrapped, (bi, d, exact, wrapped)
    check_pattern(eng, V.DF_SSE, org, ref, S, m, bl, w, w, pat, lam, what='sse decision')


# ---------------------------------------------------------------------------------------------------- which kernels the host rules choose
def kernel_selection_cases():
    """[(label, setup)]: setup(eng) uploads the planes of the case and returns (call, expect); expect(kernel names of a trace of call()) holds when the
    host rules chose the kernels they should -- both sides of the in-CTA rule and of the 32-bit key rule, the bit-depth routing of the pyramid and of the
    packed Hadamard kernels, and the pattern and pool kernels the value tests above rely on"""
    V = _V()
    W, H, m = THR_W, THR_H, 48
    cases = []

    def pyramid(label, bd, r, lam, engine, bd_ref=None):
        n = 2 * r + 1
        wide = max(bd, bd if bd_ref is None else bd_ref)
        in_cta = engine == 1 and in_cta_rule(wide, n, n, lam)
        key32 = key32_rule(wide, n, n, lam)

        def setup(eng):
            org, _, _ = contrast_planes(1000 + bd, W, H, m, bd)
            _, ref, _ = contrast_planes(1001 + bd, W, H, m, bd if bd_ref is None else bd_ref)
            upload(eng, org, ref, W, H, m, bd, bd_ref)
            eng.set_pyramid_engine(engine)
            blks = pyramid_levels(W, H, (-r, r, -r, r), np.random.RandomState(r))
            par = eng.me_par(lam, 2, 0, 0)
            return (lambda: eng.sad_search_pyramid(0, 1, blks, 8, par, n, n)), \
                (lambda names: ran(names, 'sad_pyramid8_kernel') == in_cta and (in_cta or key32_flags(names) == {key32}))
        cases.append(('%s bd %d/%d r %d lambda %r engine %d: in-CTA %s, key32 %s' % (label, bd, bd if bd_ref is None else bd_ref, r, lam, engine, in_cta, key32),
                      setup))

    for bd in (8, 10, 11, 12):
        for r in (8, 16, 32):
            for engine in (1, 0):
                pyramid('routing', bd, r, 61.5, engine)
    for engine in (1, 0):
        pyramid('mixed', 12, 32, 61.5, engine, bd_ref=8)
    for (bd, r) in ((10, 32), (8, 16)):
        n = 2 * r + 1
        for lam in lambda_edge(lambda l: in_cta_rule(bd, n, n, l)):
            pyramid('in-CTA rule', bd, r, lam, 1)
    for (bd, r, engine) in ((10, 16, 0), (12, 8, 1)):
        n = 2 * r + 1
        for lam in lambda_edge(lambda l: key32_rule(bd, n, n, l)):
            pyramid('key32 rule', bd, r, lam, engine)

    def pattern(fam, w, h, pts, kernel, bd, bd_ref=None):
        packed = max(bd, bd if bd_ref is None else bd_ref) <= 10
        want = kernel + ('<%s' % ('true' if packed else 'false') if kernel.startswith('had8_') else '')

        def setup(eng):
            org, _, _ = contrast_planes(1100 + bd, W, H, m, bd)
            _, ref, _ = contrast_planes(1101 + bd, W, H, m, bd if bd_ref is None else bd_ref)
            upload(eng, org, ref, W, H, m, bd, bd_ref)
            bl = pattern_blocks(np.random.RandomState(w + h), 6, w, h, W, H)
            par = eng.me_par(21.0, 2, 0, 0)
            return (lambda: eng.cost_pattern(fam, 0, 1, bl, w, h, mv_pattern(pts), par)), (lambda names: ran(names, want))
        cases.append(('pattern dfunc %d %dx%d radius %d bd %d/%d: %s' % (fam, w, h, max(max(abs(a), abs(b)) for a, b in pts), bd,
                                                                         bd if bd_ref is None else bd_ref, want), setup))

    for bd in (10, 12):
        for (fam, w, h, pts, kernel) in pattern_cases():
            if kernel:
                pattern(fam, w, h, pts, kernel, bd)
    pattern(V.DF_HAD, 8, 8, RING, 'had8_direct_kernel', 12, bd_ref=8)
    pattern(V.DF_HAD, 32, 32, RING, 'had8_ring_kernel', 12, bd_ref=8)

    def pool(shift):
        want, not_want = ('dist_pool_kernel', 'sad_pool_stream_kernel') if shift else ('sad_pool_stream_kernel', 'dist_pool_kernel')

        def setup(eng):
            rs = np.random.RandomState(12)
            org, _, _ = contrast_planes(1200, W, H, m, 10)
            eng.upload_plane(2, org, W, H, m, 10)
            blocks = np.zeros(3, dtype=V.POS_DT)
            blocks['x'] = [0 + shift, 24 + shift, 48 + shift]; blocks['y'] = [0, 8, 40]
            pl = rs.randint(0, 1024, size=(3, 2, 128, 128)).astype(np.int16)
            return (lambda: eng.dist_pool(V.DF_SSE, 2, blocks, 128, 128, 2, pl)), (lambda names: ran(names, want) and not ran(names, not_want))
        cases.append(('SSE pool 128x128, positions %s: %s' % ('one pel off the 8-pel grid' if shift else 'on the 8-pel grid', want), setup))

    pool(0)
    pool(1)
    return cases


def test_kernel_selection():
    """which kernels ran, on both sides of every host rule above, read from torch.profiler traces (tests/_kernel_selection_run.py).  The traces are taken
    in a process of their own: after many short profiling sessions, later traces of the same process were seen to hold no kernel record at all."""
    import json, os, subprocess, sys
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_kernel_selection_run.py')
    out = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [script], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]
    assert [r['case'] for r in rows] == [label for label, _ in kernel_selection_cases()]
    bad = [r for r in rows if not r['ok']]
    assert bad == [], (len(bad), bad[:4])
