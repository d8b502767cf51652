"""The 64x64 pyramid row walk at +-32, which runs an instantiation compiled for that geometry, next to the generic kernel on the same blocks.  A root
of a run takes its originals from a copy made behind the previous root's loop and finds its 32x32 tables cleared by the previous root's argmin pass.  Every level must equal an independent xPatternSearch replay (oracle), also around an invalid root inside a run and on
windows and originals off their 16-byte alignment, and on the benchmark picture it must equal the per-quad engine."""
import numpy as np
import pytest
from _libs import oracle, P, PO

pytestmark = pytest.mark.gpu

INVALID = (0, 0, 0xffffffff, 0xffffffffffffffff)
LAM = 61.5


@pytest.fixture(scope="module")
def eng():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def _runs(n_roots):
    """[first, end) of the run of roots each CTA of the 64x64 launch walks"""
    import torch
    g = min(n_roots, torch.cuda.get_device_properties(0).multi_processor_count)
    return [(b * n_roots // g, (b + 1) * n_roots // g) for b in range(g)]


def _run(eng, seed, W, H, rng, m=48, edit=None, check_roots=None):
    """rng = (left, right, top, bottom) of every block; the plane's first pel sits m pels into each row, so m sets the alignment of the originals and
    of the window rows; edit(blks) may change the lists and returns the roots whose trees must come back invalid"""
    import vvenc_b200 as V
    O = oracle()
    rs = np.random.RandomState(seed)
    S = W + 2 * m
    a = rs.randint(0, 1024, size=(H + 2 * m, S)).astype(np.int16)
    b = np.clip(np.roll(a, (3, -2), (0, 1)) + rs.randint(-12, 13, size=a.shape), 0, 1023).astype(np.int16)
    eng.upload_plane(0, a, W, H, m, 10); eng.upload_plane(1, b, W, H, m, 10)
    base = m * S + m
    blks = []
    for (xs, ys) in V.candidates.pyramid_lists(8, 4, W, H):
        bl = np.zeros(len(xs), dtype=V.BLOCK_DT)
        bl['x'] = xs; bl['y'] = ys; bl['left'], bl['right'], bl['top'], bl['bottom'] = rng
        bl['pred_hor'] = rs.randint(-40, 40, len(xs)); bl['pred_ver'] = rs.randint(-40, 40, len(xs))
        blks.append(bl)
    broken = edit(blks) if edit else set()
    nx, ny = rng[1] - rng[0] + 1, rng[3] - rng[2] + 1
    res = eng.sad_search_pyramid(0, 1, blks, 8, eng.me_par(LAM, 2, 0, 0), nx, ny)
    for l in range(4):
        n = 1 << (2 * (3 - l))
        idx = np.concatenate([np.arange(r * n, (r + 1) * n) for r in check_roots])
        ob = np.array([(blks[l]['x'][i], blks[l]['y'][i], 8 << l, 8 << l, blks[l]['left'][i], blks[l]['right'][i], blks[l]['top'][i],
                        blks[l]['bottom'][i], blks[l]['pred_hor'][i], blks[l]['pred_ver'][i]) for i in idx], dtype=np.int32).reshape(-1, 10)
        out = np.zeros((len(ob), 4), dtype=np.int32)
        O.orc_full_search(PO(a, base), S, PO(b, base), S, P(ob), len(ob), 0, LAM, 2, 0, P(out), None, 0)
        got = res[l]
        bad = []
        for k, i in enumerate(idx):
            g = (int(got['dx'][i]), int(got['dy'][i]), int(got['cost'][i]))
            if i // n in broken:
                if (g[0], g[1], int(got['sad'][i]), g[2]) != INVALID:
                    bad.append((i, 'invalid expected', g))
            elif g != (out[k][0], out[k][1], int(out[k][2]) & 0xffffffff):
                bad.append((i, g, tuple(out[k][:3])))
        assert bad == [], (W, H, rng, m, l, len(bad), bad[:4])
    return res


@pytest.mark.parametrize("rng", [(-32, 32, -32, 32), (-32, 32, -33, 32)])
def test_fixed_and_generic_geometry(eng, rng):
    # the same 12 x 12 roots (runs of one and two) at +-32 (fixed-geometry kernel) and at 65 x 66 positions (generic kernel)
    _run(eng, 21, 64 * 12, 64 * 12, rng, check_roots=[0, 1, 2, 11, 12, 13, 70, 71, 72, 143])


def test_fixed_invalid_root_between_carried(eng):
    # 40 x 20 roots: runs of six or seven.  Inside a run that stays on one row, the third root has two 8x8 children swapped: its tree is invalid, it skips
    # the candidate loop, and the roots around it (carried before it, restaged and then carried after it) must still find zeroed tables and their own originals
    W, H = 64 * 40, 64 * 20
    run = next((r0, r1) for r0, r1 in _runs(40 * 20) if r1 - r0 >= 5 and r0 // 40 == (r1 - 1) // 40)
    bad = run[0] + 2

    def edit(blks):
        b0 = blks[0]
        b0['x'][bad * 64 + 1], b0['x'][bad * 64 + 2] = b0['x'][bad * 64 + 2], b0['x'][bad * 64 + 1]
        b0['y'][bad * 64 + 1], b0['y'][bad * 64 + 2] = b0['y'][bad * 64 + 2], b0['y'][bad * 64 + 1]
        return {bad}
    _run(eng, 22, W, H, (-32, 32, -32, 32), edit=edit, check_roots=list(range(run[0], run[1])) + [run[1], 0, 40 * 20 - 1])


@pytest.mark.parametrize("left,m", [(-33, 48), (-32, 44)])
def test_fixed_misaligned(eng, left, m):
    # 65 x 65 positions whose windows start on an odd pel (16-bit staging, no carry), or 8 bytes off a 16-byte boundary together with the originals
    # (4-byte window copies, originals read in the staging phase)
    _run(eng, 23, 64 * 24, 64 * 12, (left, left + 64, -32, 32), m=m, check_roots=[0, 1, 2, 3, 23, 24, 25, 150, 151, 287])


def test_bench_picture_vs_engine0(eng):
    # the benchmark's 3840x2160 picture and block lists: every level of every block equals the per-quad engine's result bit for bit
    import bench as B
    import vvenc_b200 as V
    org, ref, S = B.synth_picture_pair(1234)
    eng.upload_plane(0, org, B.W, B.H, B.MARGIN, 10); eng.upload_plane(1, ref, B.W, B.H, B.MARGIN, 10)
    blks = []
    for n in B.SIZES:
        xs, ys = B.block_grid(n)
        bl = np.zeros(len(xs), dtype=V.BLOCK_DT)
        bl['x'] = xs; bl['y'] = ys; bl['left'] = -32; bl['right'] = 32; bl['top'] = -32; bl['bottom'] = 32
        blks.append(bl)
    me = eng.me_par(B.LAMBDA, 2, 0, 0, 1, 2)
    try:
        got = eng.sad_search_pyramid(0, 1, blks, 8, me, 65, 65)
        eng.set_pyramid_engine(0)
        exp = eng.sad_search_pyramid(0, 1, blks, 8, me, 65, 65)
    finally:
        eng.set_pyramid_engine(1)
    for l in range(4):
        for f in ('dx', 'dy', 'sad', 'cost'):
            assert np.array_equal(got[l][f], exp[l][f]), (l, f, int(np.count_nonzero(got[l][f] != exp[l][f])))
