"""The pel-pair identity behind sad_pyramid8_kernel's strip items, over every pair of 10-bit pels: read as fp16, a pel up to 1023 is a subnormal (or zero),
fma(o, -1, w) clamped at zero is exact there and its bits are the integer max(w - o, 0), and |a - b| = a - b + 2 max(b - a, 0).  32 such values per uint16
lane cannot carry into the next lane."""
import numpy as np


def test_relu_of_subnormal_pels_is_the_integer_clamp():
    v = np.arange(1024, dtype=np.uint16)
    o, w = np.meshgrid(v, v, indexing='ij')
    of, wf = o.view(np.float16).astype(np.float32), w.view(np.float16).astype(np.float32)
    d = np.maximum(of * np.float32(-1.0) + wf, np.float32(0.0)).astype(np.float16)     # exact in float32, so rounding once is the fused fma's result
    got = d.view(np.uint16).astype(np.int64)
    want = np.maximum(w.astype(np.int64) - o.astype(np.int64), 0)
    assert np.array_equal(got, want)
    a, b = o.astype(np.int64), w.astype(np.int64)
    assert np.array_equal(np.abs(a - b), a - b + 2 * want)
    assert 32 * int(want.max()) < 1 << 16
