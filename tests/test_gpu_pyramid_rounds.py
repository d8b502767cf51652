"""In-CTA SAD pyramid: range shapes where a warp holds both strip items and column items of the 64x64 roots (the item count of the strips is not a
multiple of 32), and a row count of 3 mod 4.  Every block of every level against the oracle's xPatternSearch replay and against the per-quad engine."""
import numpy as np
import pytest
import impls
from _libs import oracle
from test_gpu_parity import _pyramid_case, _check_pyramid

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return impls.GpuImpl(0)


@pytest.mark.parametrize("rng", [(-7, 7, -6, 6), (-20, 20, -13, 13)], ids=["15x13_mixed_warp", "41x27_rows_3mod4"])
def test_gpu_pyramid_in_cta_item_rounds(gpu, rng):
    O = oracle()
    rs = np.random.RandomState(21 + rng[1])
    lam = 43.1
    W, H, m = 192, 128, 40                                      # 3 x 2 roots of 64
    a, b, S, base, blks = _pyramid_case(gpu, rs, W, H, m, rng[0], rng[1], rng[2], rng[3], 4, lam)
    nx, ny = rng[1] - rng[0] + 1, rng[3] - rng[2] + 1
    par = gpu.eng.me_par(lam, 2, 0, 0)
    gpu.eng.set_pyramid_engine(1)
    res = gpu.eng.sad_search_pyramid(4, 5, blks, 8, par, nx, ny)
    _check_pyramid(O, a, b, S, base, blks, res, lam)
    gpu.eng.set_pyramid_engine(0)
    res0 = gpu.eng.sad_search_pyramid(4, 5, blks, 8, par, nx, ny)
    gpu.eng.set_pyramid_engine(1)
    for l in range(len(blks)):
        assert np.array_equal(res[l], res0[l]), (rng, l)
