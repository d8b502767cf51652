"""Hadamard refinement ring (had8_ring_kernel) against the CPU oracle on shapes the parity suite does not reach: whole-plane block lists (many blocks
per CTA), start vectors of both parities, a radius-8 pattern that reaches the plane margin, single-output calls, a 12-bit plane pair and pattern points
beyond the radius the caller states."""
import ctypes
import numpy as np
import pytest
import impls
from _libs import oracle, PO

pytestmark = pytest.mark.gpu

RING = [(0, 0)] + [(dx, dy) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dx or dy] + [(dx, dy) for dy in (-2, 0, 2) for dx in (-2, 0, 2) if dx or dy] + [(0, 0)]


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return impls.GpuImpl(0)


def _planes(rs, W, H, m, bd):
    S = W + 2 * m
    a = rs.randint(0, 1 << bd, size=(H + 2 * m, S)).astype(np.int16)
    b = np.clip(np.roll(a, (1, -2), (0, 1)) + rs.randint(-40, 41, size=a.shape), 0, (1 << bd) - 1).astype(np.int16)
    return np.ascontiguousarray(a), np.ascontiguousarray(b), S


def _pattern(V, pts):
    pat = np.zeros(len(pts), dtype=V.MV_DT); pat['dx'] = [p[0] for p in pts]; pat['dy'] = [p[1] for p in pts]
    return pat


def _tiling(V, rs, W, H, n, rng, start):
    xs, ys = np.meshgrid(np.arange(0, W - n + 1, n), np.arange(0, H - n + 1, n))
    blk = np.zeros(xs.size, dtype=V.BLOCK_DT)
    blk['x'] = xs.ravel(); blk['y'] = ys.ravel()
    blk['left'] = -rng; blk['right'] = rng; blk['top'] = -rng; blk['bottom'] = rng
    blk['pred_hor'] = rs.randint(-40, 40, len(blk)); blk['pred_ver'] = rs.randint(-40, 40, len(blk))
    blk['start_x'] = rs.randint(-start, start + 1, len(blk)); blk['start_y'] = rs.randint(-start, start + 1, len(blk))
    return blk


def _expect(O, a, b, S, m, blk, n, pat, lam):
    """oracle cost table (0xffffffff outside the search range) and (cost, dx, dy, sad) of the best point in list order"""
    base = m * S + m
    cost = np.zeros((len(blk), len(pat)), dtype=np.uint32); best = []
    for i in range(len(blk)):
        x, y = int(blk['x'][i]), int(blk['y'][i]); bc = None
        for k in range(len(pat)):
            mx = int(blk['start_x'][i]) + int(pat['dx'][k]); my = int(blk['start_y'][i]) + int(pat['dy'][k])
            if not (blk['left'][i] <= mx <= blk['right'][i] and blk['top'][i] <= my <= blk['bottom'][i]):
                cost[i, k] = 0xffffffff
                continue
            e = O.orc_had(PO(a, base + y * S + x), S, PO(b, base + (y + my) * S + x + mx), S, n, n, 0)
            cost[i, k] = e
            c = e + O.orc_mv_cost(lam, mx, my, int(blk['pred_hor'][i]), int(blk['pred_ver'][i]), 2, 0)
            if bc is None or c < bc[0]:
                bc = (c, mx, my, e)
        best.append(bc if bc is not None else (2 ** 64 - 1, 0, 0, 0xffffffff))
    return cost, best


def _check_best(best, exp):
    got = [(int(best['cost'][i]), int(best['dx'][i]), int(best['dy'][i]), int(best['sad'][i])) for i in range(len(best))]
    bad = [i for i in range(len(got)) if got[i] != exp[i]]
    assert not bad, (bad[:5], [got[i] for i in bad[:5]], [exp[i] for i in bad[:5]])


@pytest.mark.parametrize("n", [8, 16, 32, 64])
def test_had_ring_plane_tiling(gpu, n):
    """every block of a 256x192 plane at one size (the bench's ring at radius 2), odd and even start vectors, some points outside the range"""
    import vvenc_b200 as V
    O = oracle()
    rs = np.random.RandomState(4100 + n)
    W, H, m = 256, 192, 32
    a, b, S = _planes(rs, W, H, m, 10)
    gpu.eng.upload_plane(2, a, W, H, m); gpu.eng.upload_plane(3, b, W, H, m)
    blk = _tiling(V, rs, W, H, n, 11, 12)
    assert (blk['start_x'] % 2 == 1).any() and (blk['start_x'] % 2 == 0).any()
    pat = _pattern(V, RING)
    lam = 25.0
    cost, best = gpu.eng.cost_pattern(V.DF_HAD, 2, 3, blk, n, n, pat, gpu.eng.me_par(lam, 2, 0, 0))
    ec, eb = _expect(O, a, b, S, m, blk, n, pat, lam)
    assert (ec == 0xffffffff).any()
    assert np.array_equal(cost, ec), np.argwhere(cost != ec)[:5]
    _check_best(best, eb)


@pytest.mark.parametrize("n", [8, 16, 32, 64])
def test_had_ring_radius8_at_margin(gpu, n):
    """radius-8 pattern with points at +-8; blocks on the plane border whose start vectors put the window on the last margin pel"""
    import vvenc_b200 as V
    O = oracle()
    rs = np.random.RandomState(4200 + n)
    W, H, m = 192, 128, 16
    a, b, S = _planes(rs, W, H, m, 10)
    gpu.eng.upload_plane(2, a, W, H, m); gpu.eng.upload_plane(3, b, W, H, m)
    pts = [(0, 0), (8, 8), (-8, -8), (8, -8), (-8, 8), (-7, 3), (5, -6), (1, 0), (-1, 1), (0, -8), (8, 0), (-3, -3)]
    pat = _pattern(V, pts)
    rows = []
    for (x, sx) in ((0, -8), (W - n, 8), (0, -7), (W - n, 7)):
        for (y, sy) in ((0, -8), (H - n, 8), (n, 1)):
            rows.append((x, y, sx, sy))
    blk = np.zeros(len(rows), dtype=V.BLOCK_DT)
    for i, (x, y, sx, sy) in enumerate(rows):
        blk[i]['x'] = x; blk[i]['y'] = y; blk[i]['start_x'] = sx; blk[i]['start_y'] = sy
    blk['left'] = -m; blk['right'] = m; blk['top'] = -m; blk['bottom'] = m
    blk['pred_hor'] = rs.randint(-40, 40, len(blk)); blk['pred_ver'] = rs.randint(-40, 40, len(blk))
    lam = 12.0
    cost, best = gpu.eng.cost_pattern(V.DF_HAD, 2, 3, blk, n, n, pat, gpu.eng.me_par(lam, 2, 0, 0))
    ec, eb = _expect(O, a, b, S, m, blk, n, pat, lam)
    assert np.array_equal(cost, ec), np.argwhere(cost != ec)[:5]
    _check_best(best, eb)


def test_had_ring_single_outputs_and_12bit(gpu):
    """cost table only and best only give what the two-output call gives; a 12-bit pair takes the unpacked form"""
    import vvenc_b200 as V
    O = oracle()
    rs = np.random.RandomState(4300)
    W, H, m = 128, 128, 24
    pat = _pattern(V, RING)
    lam = 40.0
    for bd in (10, 12):
        a, b, S = _planes(rs, W, H, m, bd)
        gpu.eng.upload_plane(2, a, W, H, m, bd); gpu.eng.upload_plane(3, b, W, H, m, bd)
        for n in (8, 16, 32, 64):
            blk = _tiling(V, rs, W, H, n, 9, 9)
            par = gpu.eng.me_par(lam, 2, 0, 0)
            cost, best = gpu.eng.cost_pattern(V.DF_HAD, 2, 3, blk, n, n, pat, par)
            c1, _ = gpu.eng.cost_pattern(V.DF_HAD, 2, 3, blk, n, n, pat, par, want_best=False)
            _, b1 = gpu.eng.cost_pattern(V.DF_HAD, 2, 3, blk, n, n, pat, par, want_cost=False)
            assert np.array_equal(cost, c1) and np.array_equal(best, b1), (bd, n)
            ec, eb = _expect(O, a, b, S, m, blk, n, pat, lam)
            assert np.array_equal(cost, ec), (bd, n, np.argwhere(cost != ec)[:5])
            _check_best(best, eb)


def test_had_ring_points_beyond_stated_radius(gpu):
    """the device entry point takes pattern_radius from the caller: points beyond it are read from the plane, not from the staged window"""
    import torch
    import vvenc_b200 as V
    O = oracle()
    rs = np.random.RandomState(4400)
    W, H, m = 160, 128, 32
    a, b, S = _planes(rs, W, H, m, 10)
    gpu.eng.upload_plane(2, a, W, H, m); gpu.eng.upload_plane(3, b, W, H, m)
    pat = _pattern(V, RING[:9] + [(3, -5), (-9, 4), (12, 12), (0, 0)])
    lam = 18.0
    eng = gpu.eng
    for (n, radius) in ((8, 1), (16, 2), (32, 2), (64, 5)):
        blk = _tiling(V, rs, W, H, n, 14, 5)
        dev = lambda arr: torch.from_numpy(np.frombuffer(arr.tobytes(), dtype=np.uint8).copy()).cuda()
        d_blk, d_pat = dev(blk), dev(pat)
        d_cost = torch.zeros(len(blk) * len(pat), dtype=torch.int32, device='cuda'); d_best = torch.zeros(len(blk) * 16, dtype=torch.uint8, device='cuda')
        me = eng.me_par(lam, 2, 0, 0, 0, radius)
        rc = eng.lib.vvb_cost_pattern_dev(eng.h, V.DF_HAD, 2, 3, ctypes.c_void_p(d_blk.data_ptr()), len(blk), n, n, ctypes.c_void_p(d_pat.data_ptr()), len(pat),
                                          ctypes.byref(me), ctypes.c_void_p(d_cost.data_ptr()), ctypes.c_void_p(d_best.data_ptr()))
        assert rc == 0, eng.lib.vvb_last_error(eng.h)
        eng.synchronize()
        cost = d_cost.cpu().numpy().view(np.uint32).reshape(len(blk), len(pat))
        best = np.frombuffer(d_best.cpu().numpy().tobytes(), dtype=V.BEST_DT)
        ec, eb = _expect(O, a, b, S, m, blk, n, pat, lam)
        assert np.array_equal(cost, ec), (n, np.argwhere(cost != ec)[:5])
        _check_best(best, eb)
