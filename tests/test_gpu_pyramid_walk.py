"""Row walk of the in-CTA SAD pyramid (pyramid_kernels.cuh): one CTA per SM walks a run of consecutive 64x64 roots and carries the shared half of each
reference window to the root on its right.  Every level's result must equal an independent xPatternSearch replay (oracle) with the block's own range and
predictor, on lists that make runs of uneven length, break the carry in the middle of a row and cross the limit where the staging area fits."""
import numpy as np
import pytest
from _libs import oracle, P, PO

pytestmark = pytest.mark.gpu

INVALID = (0, 0, 0xffffffff, 0xffffffffffffffff)


@pytest.fixture(scope="module")
def eng():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def _planes(rs, W, H, m, bd):
    S = W + 2 * m
    a = rs.randint(0, 1 << bd, size=(H + 2 * m, S)).astype(np.int16)
    b = np.clip(np.roll(a, (2, -3), (0, 1)) + rs.randint(-12, 13, size=a.shape), 0, (1 << bd) - 1).astype(np.int16)
    return np.ascontiguousarray(a), np.ascontiguousarray(b), S


def _run(eng, seed, W, H, rng, bd=10, edit=None, check_roots=None):
    """rng = (left, right, top, bottom) of every block; edit(blks) may change the lists; check_roots: the 64x64 roots whose trees are replayed (all if None)"""
    import vvenc_b200 as V
    O = oracle()
    rs = np.random.RandomState(seed)
    m = 48
    a, b, S = _planes(rs, W, H, m, bd)
    eng.upload_plane(0, a, W, H, m, bd); eng.upload_plane(1, b, W, H, m, bd)
    base = m * S + m
    lists = V.candidates.pyramid_lists(8, 4, W, H)
    blks = []
    for (xs, ys) in lists:
        bl = np.zeros(len(xs), dtype=V.BLOCK_DT)
        bl['x'] = xs; bl['y'] = ys; bl['left'], bl['right'], bl['top'], bl['bottom'] = rng
        bl['pred_hor'] = rs.randint(-40, 40, len(xs)); bl['pred_ver'] = rs.randint(-40, 40, len(xs))
        blks.append(bl)
    nRoots = len(blks[3])
    broken = edit(blks) if edit else set()
    nx, ny = rng[1] - rng[0] + 1, rng[3] - rng[2] + 1
    lam = 61.5
    res = eng.sad_search_pyramid(0, 1, blks, 8, eng.me_par(lam, 2, 0, 0), nx, ny)
    roots = range(nRoots) if check_roots is None else check_roots
    for l in range(4):
        n = 1 << (2 * (3 - l))
        if check_roots is None:
            idx = np.arange(len(blks[l]))                          # also the blocks of the smaller roots below and right of the 64x64 grid
        else:
            idx = np.concatenate([np.arange(r * n, (r + 1) * n) for r in roots])
        ob = np.zeros((len(idx), 10), dtype=np.int32)
        for k, i in enumerate(idx):
            bb = blks[l][i]
            ob[k] = (bb['x'], bb['y'], 8 << l, 8 << l, bb['left'], bb['right'], bb['top'], bb['bottom'], bb['pred_hor'], bb['pred_ver'])
        out = np.zeros((len(ob), 4), dtype=np.int32)
        O.orc_full_search(PO(a, base), S, PO(b, base), S, P(ob), len(ob), 0, lam, 2, 0, P(out), None, 0)
        got = res[l]
        bad = []
        for k, i in enumerate(idx):
            g = (int(got['dx'][i]), int(got['dy'][i]), int(got['cost'][i]))
            if i < nRoots * n and (i // n) in broken:
                if (g[0], g[1], int(got['sad'][i]), g[2]) != INVALID:
                    bad.append((i, 'invalid expected', g))
            elif g != (out[k][0], out[k][1], int(out[k][2]) & 0xffffffff):
                bad.append((i, g, tuple(out[k][:3])))
        assert bad == [], (W, H, rng, bd, l, len(bad), bad[:4])
    return nRoots


def test_walk_runs_of_one_and_two(eng):
    # 12 x 12 roots + a column of 32x32 roots: on 132 SMs, runs of one and two roots, some of them across a row end
    assert _run(eng, 5, 64 * 12 + 32, 64 * 12, (-9, 12, -10, 7)) == 144


def test_walk_long_runs_8bit(eng):
    # 24 x 12 roots: runs of two and three roots, 8-bit planes
    assert _run(eng, 6, 64 * 24, 64 * 12, (-8, 8, -8, 8), bd=8) == 288


def test_walk_few_roots(eng):
    # fewer roots than SMs: one root per CTA
    _run(eng, 7, 64 * 3 + 32, 64 * 2, (-9, 12, -10, 7))


def test_walk_broken_quad_and_other_range_mid_row(eng):
    W, H = 64 * 24, 64 * 12

    def edit(blks):
        # root 30 (row 1): two 8x8 children swapped -> its whole tree is invalid, its neighbours restage and stay right
        b0 = blks[0]
        b0['x'][30 * 64 + 1], b0['x'][30 * 64 + 2] = b0['x'][30 * 64 + 2], b0['x'][30 * 64 + 1]
        b0['y'][30 * 64 + 1], b0['y'][30 * 64 + 2] = b0['y'][30 * 64 + 2], b0['y'][30 * 64 + 1]
        # root 53 (row 2): the same range size, shifted by one pel left and two up -> a window of its own
        for l in range(4):
            n = 1 << (2 * (3 - l))
            s = slice(53 * n, 54 * n)
            blks[l]['left'][s] -= 1; blks[l]['right'][s] -= 1; blks[l]['top'][s] -= 2; blks[l]['bottom'][s] -= 2
        return {30}
    _run(eng, 8, W, H, (-8, 8, -8, 8), edit=edit)


@pytest.mark.parametrize("left", [-31, -30])
def test_walk_window_alignment(eng, left):
    # odd window start: the 16-bit staging path, no carry; start 2 pels off a 16-byte boundary: 4-byte copies into the staging area
    _run(eng, 9, 64 * 12 + 32, 64 * 12, (left, left + 21, -10, 7))


@pytest.mark.parametrize("rng", [(-32, 32, -32, 32), (-32, 32, -35, 34)])
def test_walk_bench_range_and_no_staging(eng, rng):
    # +-32 (the staging area fits) and 65 x 70 positions (it does not: every root restages); the replay covers roots on both sides of run boundaries
    nRoots = 12 * 12
    check = [0, 1, 11, 12, 13, 23, 24, 25, 70, 71, 72, 143]
    assert _run(eng, 10, 64 * 12, 64 * 12, rng, check_roots=check) == nRoots
