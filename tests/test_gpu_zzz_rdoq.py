"""GPU parity (-m gpu) of the fast RDOQ (QuantRDOQ2::xRateDistOptQuant, Quant::m_RDOQ == 2; SURVEY 8f rank 4) through the C ABI (vvb_rdoq):
golden vectors from the unmodified reference, picture-sized batches against the CPU build of the same restatement, the reference-side binding next to the member
on the real library, and whole-encoder bitstream identity with the RDOQ seam routed through the GPU.  Sorted last in the suite on purpose: the entry point is the
newest one of the library."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import cases as C
import impls
from _libs import have_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


# Tests written after the GPU budget of the round was spent: their subjects are pinned on the CPU (shared host / device text against the reference's members, whole-encoder
# identity on the oracle-backed mock), the kernels under them have the shape of rdoq_kernel, which ran green on hardware -- but these tests themselves have not run on a GPU
# yet.  Non-strict xfail states exactly that: the round-end suite reports XPASS when they pass, and a first-run failure does not mask the verified tests.
first_hardware_run = pytest.mark.xfail(strict=False, reason='first hardware run (written after the GPU budget of the round was spent); pinned on the CPU')


@pytest.fixture(scope="module")
def gpu():
    return impls.GpuImpl(0)          # vvb_create fails loudly without a CUDA device; no torch needed on this path


def test_gpu_rdoq_golden(gpu, golden_rdoq):
    """every row of cases.rdoq_cases() against what the reference produced (tests/golden/golden_v6_rdoq.npz): levels, absSum, lastPos; the constants the library
    derives (quantiser scale / shift, error scale, thresholds, bin budget) against the reference's"""
    import ctypes
    import vvenc_b200._lib as L
    g = golden_rdoq
    rows = C.rdoq_cases()
    assert np.array_equal(rows, g['cases'])
    nonzero = 0
    for i, row in enumerate(rows):
        w, h, bd, qp, lam1000, scale, decay10, comp, lf, sbt, intra, sh, cb, thr, init_id, seed = [int(v) for v in row]
        coef = C.rdoq_inputs(row)[None]
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, sign_hiding=bool(sh), lfnst_idx=lf, is_chroma=comp > 0)
        rq = L.vvb_rdoq_par(lam1000 / 1000.0, thr, sbt)
        k = np.zeros(7, dtype=np.int32)
        assert gpu.eng.lib.vvb_rdoq_constants(ctypes.byref(par), ctypes.byref(rq), k.ctypes.data_as(ctypes.c_void_p)) == 0
        assert np.array_equal(k, g['consts'][i]), i
        r = gpu.eng.rdoq(par, gpu.eng.rdoq_rates(g['rates'][i]), coef, lam1000 / 1000.0, thr, sbt)
        assert np.array_equal(r['q'][0], g['q_%d' % i]), (i, [int(v) for v in row])
        assert (int(r['abs_sum'][0]), int(r['last_pos'][0])) == tuple(int(v) for v in g['meta'][i]), (i, [int(v) for v in row])
        nonzero += int(r['last_pos'][0] >= 0)
    assert nonzero > 100


def test_gpu_rdoq_batches_vs_oracle(gpu, golden_rdoq):
    """a picture's worth of TUs per launch (more TUs than resident threads for the small shapes: the threads stride over the list), the need_rdoq mask of
    useSelectiveRdoq, luma and chroma, hiding on and off, against the CPU build of the restatement on the same inputs; fractional bits of a reference CABAC state"""
    from _libs import dq_oracle, P
    O = dq_oracle()
    g = golden_rdoq
    rs = np.random.RandomState(78)
    chroma_rows = [i for i, r in enumerate(g['cases']) if int(r[7]) > 0]
    luma_rows = [i for i, r in enumerate(g['cases']) if int(r[7]) == 0]
    for (w, h, n, qp, lam, sbt, lf, sh, chroma) in ((4, 4, 90000, 32, 57.3, 0, 0, 1, 0), (8, 8, 30000, 27, 30.0, 0, 1, 0, 0), (16, 16, 6000, 37, 120.0, 0, 0, 1, 0), (32, 32, 1500, 32, 57.3, 1, 0, 1, 0),
                                                   (64, 64, 300, 22, 11.7, 0, 0, 0, 0), (32, 8, 3000, 42, 800.0, 0, 0, 1, 1), (16, 64, 500, 32, 30.0, 0, 2, 1, 0), (8, 8, 20000, 30, 40.0, 0, 0, 1, 1)):
        scale = rs.choice([3, 10, 40, 150, 600, 2500], size=(n, 1, 1))
        coef = rs.laplace(0, 1.0, size=(n, h, w)) * scale * (1.0 / (1 + np.add.outer(np.arange(h), np.arange(w))) ** 0.7)
        coef = np.clip(coef, -32768, 32767).astype(np.int32)
        coef[:, :, 32:] = 0; coef[:, 32:, :] = 0
        pick = chroma_rows if chroma else luma_rows
        rates_flat = np.ascontiguousarray(g['rates'][pick[int(rs.randint(len(pick)))]])
        mask = (rs.randint(0, 8, size=n) > 0).astype(np.uint8)
        par = gpu.eng.tu_par(w, h, 0, 0, 10, qp, sign_hiding=bool(sh), lfnst_idx=lf, is_chroma=bool(chroma))
        r = gpu.eng.rdoq(par, gpu.eng.rdoq_rates(rates_flat), coef, lam, 8, sbt, need_rdoq=mask)
        q = np.zeros((n, h, w), dtype=np.int16); s = np.zeros(n, dtype=np.int32); l = np.zeros(n, dtype=np.int32)
        assert O.orc_rdoq(w, h, 10, qp, chroma, lf, sbt, sh, lam, 8, P(rates_flat), P(coef), n, P(q), P(s), P(l)) == 0
        q[mask == 0] = 0; s[mask == 0] = 0; l[mask == 0] = -1
        assert np.array_equal(r['q'], q), (w, h, int((r['q'] != q).any(axis=(1, 2)).sum()))
        assert np.array_equal(r['abs_sum'], s) and np.array_equal(r['last_pos'], l), (w, h)
        assert (l >= 0).sum() > n // 8, (w, h, int((l >= 0).sum()))


def test_gpu_rdoq_rejects_what_stays_on_the_host(gpu, golden_rdoq):
    import vvenc_b200 as V
    coef = np.zeros((1, 8, 8), dtype=np.int32)
    rates = gpu.eng.rdoq_rates(golden_rdoq['rates'][0])
    with pytest.raises(V.VvbError):
        gpu.eng.rdoq(gpu.eng.tu_par(8, 8, 0, 0, 10, 30, transform_skip=True), rates, coef, 30.0)          # rateDistOptQuantTS
    with pytest.raises(V.VvbError):
        gpu.eng.rdoq(gpu.eng.tu_par(8, 8, 0, 0, 10, 30), rates, coef, 0.0)                                  # lambda


@pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
def test_rdoq_binding_on_the_real_library():
    """xRateDistOptQuantB200 (integration/TrQuantB200.h) bound to libvvenc_b200.so next to QuantRDOQ2::xRateDistOptQuant called as a member"""
    import vvenc_b200._lib as VL
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', '_integration_host_run.py'), VL.LIB_PATH, 'rdoq'], capture_output=True, text=True, timeout=400)
    assert out.returncode == 0, out.stderr[-3000:]
    r = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith('RESULT ')][-1][len('RESULT '):])['rdoq']
    assert r['cases'] == 224 and r['non_empty'] > 100 and r['non_empty_with_hiding'] > 40 and r['bad'] == [], r


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'enc_identity')), reason='oracle/_ref/enc_identity not built')
@pytest.mark.parametrize("W,H,F,preset,qp", [(80, 44, 4, 0, 37), (176, 144, 3, 0, 27), (416, 240, 8, 0, 37)])       # the last one is BASELINE configs[0]
def test_bitstream_identity_with_the_rdoq_seam_on_the_gpu(tmp_path, W, H, F, preset, qp):
    import vvenc_b200._lib as VL
    from test_encoder_identity import _identity_rdoq
    kb = _identity_rdoq(tmp_path, W, H, F, preset, qp, VL.LIB_PATH, timeout=1500)
    print('encoder identity with the RDOQ seam on the GPU:', W, H, F, preset, kb)


@first_hardware_run
@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'enc_identity')), reason='oracle/_ref/enc_identity not built')
@pytest.mark.parametrize("W,H,F,preset,qp", [(80, 44, 3, 2, 37), (176, 144, 2, 1, 32)])
def test_bitstream_identity_with_the_widest_tu_seam_on_the_gpu(tmp_path, W, H, F, preset, qp):
    """the widest routing of the TU seam (LFNST on separate-tree chroma and ISP luma TUs, joint Cb-Cr TUs, single-tree chroma of LFNST CUs) with the kernels answering:
    the same kernels as the narrower routing, fed with the chroma / ISP parameter combinations"""
    import vvenc_b200._lib as VL
    from test_encoder_identity import _identity_widest
    kb = _identity_widest(tmp_path, W, H, F, preset, qp, VL.LIB_PATH, timeout=1500)
    print('encoder identity with the widest TU seam on the GPU:', W, H, F, preset, kb)


@first_hardware_run
@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'enc_identity')), reason='oracle/_ref/enc_identity not built')
@pytest.mark.parametrize("W,H,F,preset,qp", [(80, 44, 9, 2, 37), (176, 144, 9, 0, 32)])
def test_bitstream_identity_with_the_mctf_errors_on_the_gpu(tmp_path, W, H, F, preset, qp):
    """the MCTF error pointers answered per call by mctf_error_packed_kernel (two small plane uploads + one candidate per call) under the unmodified motion search of the
    pre-analysis, together with the distortion tables and the widest TU seam: the whole encoder, nine frames"""
    import vvenc_b200._lib as VL
    from test_encoder_identity import _identity_mctf
    kb = _identity_mctf(tmp_path, W, H, F, preset, qp, VL.LIB_PATH, timeout=1500)
    print('encoder identity with the MCTF errors on the GPU:', W, H, F, preset, kb)


# ---- transform-skipped TUs: QuantRDOQ::rateDistOptQuantTS (vvb_rdoq_ts)
def test_gpu_rdoq_ts_golden(gpu, golden_rdoq):
    g = golden_rdoq
    rows = C.rdoq_ts_cases()
    assert np.array_equal(rows, g['ts_cases'])
    nonzero = 0
    for i, row in enumerate(rows):
        w, h, bd, qp, lam1000, amp, kind, comp, intra, delta, init_id, seed = [int(v) for v in row]
        coef = C.rdoq_ts_inputs(row)[None]
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, transform_skip=True, input_bit_depth_delta=delta, is_chroma=comp > 0)
        r = gpu.eng.rdoq_ts(par, gpu.eng.rdoq_ts_rates(g['ts_rates'][i]), coef, lam1000 / 1000.0)
        assert np.array_equal(r['q'][0], g['tsq_%d' % i]) and int(r['abs_sum'][0]) == int(g['ts_abs_sum'][i]), (i, [int(v) for v in row])
        nonzero += int(r['abs_sum'][0] > 0)
    assert nonzero > 80


def test_gpu_rdoq_ts_batches_vs_oracle(gpu, golden_rdoq):
    from _libs import dq_oracle, P
    O = dq_oracle()
    g = golden_rdoq
    rs = np.random.RandomState(79)
    for (w, h, n, qp, lam, bd) in ((4, 4, 60000, 32, 57.3, 10), (8, 8, 20000, 27, 30.0, 10), (16, 16, 5000, 37, 120.0, 10), (32, 32, 1200, 22, 11.7, 10), (32, 8, 3000, 42, 800.0, 8), (4, 16, 8000, 30, 40.0, 10)):
        amp = rs.choice([2, 6, 20, 60, 200, 1023], size=(n, 1, 1))
        resi = (rs.laplace(0, 1.0, size=(n, h, w)) * amp / 3.0).astype(np.int64)
        resi[rs.rand(n, h, w) < 0.4] = 0
        lim = (1 << bd) - 1
        shift = max(0, 15 - bd - ((int(np.log2(w)) + int(np.log2(h))) >> 1))
        coef = np.clip(resi, -lim, lim).astype(np.int32); coef[::2] <<= shift          # unscaled as xTransformSkip leaves them, every second TU scaled up (large levels)
        rates_flat = np.ascontiguousarray(g['ts_rates'][int(rs.randint(len(g['ts_rates'])))])
        mask = (rs.randint(0, 8, size=n) > 0).astype(np.uint8)
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, transform_skip=True)
        r = gpu.eng.rdoq_ts(par, gpu.eng.rdoq_ts_rates(rates_flat), coef, lam, need_rdoq=mask)
        q = np.zeros((n, h, w), dtype=np.int16); s = np.zeros(n, dtype=np.int32)
        assert O.orc_rdoq_ts(w, h, bd, qp, 0, lam, P(rates_flat), P(coef), n, P(q), P(s)) == 0
        q[mask == 0] = 0; s[mask == 0] = 0
        assert np.array_equal(r['q'], q), (w, h, int((r['q'] != q).any(axis=(1, 2)).sum()))
        assert np.array_equal(r['abs_sum'], s) and (s > 0).sum() > n // 8, (w, h, int((s > 0).sum()))


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'enc_identity')), reason='oracle/_ref/enc_identity not built')
@pytest.mark.parametrize("W,H,F,preset,qp,min_ts", [(80, 44, 4, 0, 32, 40), (176, 144, 3, 0, 27, 1000)])
def test_bitstream_identity_with_transform_skip_rdoq_on_the_gpu(tmp_path, W, H, F, preset, qp, min_ts):
    import vvenc_b200._lib as VL
    from test_encoder_identity import _identity_ts
    kb = _identity_ts(tmp_path, W, H, F, preset, qp, VL.LIB_PATH, min_ts, timeout=1500)
    print('encoder identity with the transform-skip RDOQ on the GPU:', W, H, F, preset, kb)


@pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
def test_rdoq_ts_binding_on_the_real_library():
    """rateDistOptQuantTSB200 (integration/TrQuantB200.h) bound to libvvenc_b200.so next to QuantRDOQ::rateDistOptQuantTS called as a member"""
    import vvenc_b200._lib as VL
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', '_integration_host_run.py'), VL.LIB_PATH, 'rdoq'], capture_output=True, text=True, timeout=400)
    assert out.returncode == 0, out.stderr[-3000:]
    t = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith('RESULT ')][-1][len('RESULT '):])['rdoq_ts']
    assert t['cases'] == 140 and t['non_empty'] > 80 and t['bad'] == [], t


# ---- BDPCM TUs: QuantRDOQ::forwardRDPCM (vvb_rdoq_bdpcm); inverse side = host running sums + vvb_inv_trquant of skipped transforms (verified kernel)
def test_gpu_rdoq_bdpcm_golden(gpu, golden_rdoq):
    g = golden_rdoq
    rows = C.rdoq_ts_cases()
    nonzero = 0
    for i, row in enumerate(rows):
        w, h, bd, qp, lam1000, amp, kind, comp, intra, delta, init_id, seed = [int(v) for v in row]
        coef = C.rdoq_ts_inputs(row)[None]
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, transform_skip=True, input_bit_depth_delta=delta, is_chroma=comp > 0)
        r = gpu.eng.rdoq_bdpcm(par, gpu.eng.rdoq_ts_rates(g['ts_rates'][i]), coef, lam1000 / 1000.0, 1 + (seed & 1))
        assert np.array_equal(r['q'][0], g['bdq_%d' % i]) and int(r['abs_sum'][0]) == int(g['bd_abs_sum'][i]), (i, [int(v) for v in row])
        nonzero += int(r['abs_sum'][0] > 0)
    assert nonzero > 70


def test_gpu_rdoq_bdpcm_batches_vs_oracle(gpu, golden_rdoq):
    from _libs import dq_oracle, P
    O = dq_oracle()
    g = golden_rdoq
    rs = np.random.RandomState(80)
    for (w, h, n, qp, lam, bd, dm) in ((4, 4, 40000, 32, 57.3, 10, 1), (8, 8, 20000, 27, 30.0, 10, 2), (16, 16, 5000, 37, 120.0, 10, 1), (32, 32, 1200, 22, 11.7, 10, 2), (32, 8, 3000, 42, 800.0, 8, 1)):
        amp = rs.choice([2, 6, 20, 60, 200, 1023], size=(n, 1, 1))
        resi = (rs.laplace(0, 1.0, size=(n, h, w)) * amp / 3.0).astype(np.int64)
        resi[rs.rand(n, h, w) < 0.4] = 0
        lim = (1 << bd) - 1
        coef = np.clip(resi, -lim, lim).astype(np.int32)
        rates_flat = np.ascontiguousarray(g['ts_rates'][int(rs.randint(len(g['ts_rates'])))])
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, transform_skip=True)
        r = gpu.eng.rdoq_bdpcm(par, gpu.eng.rdoq_ts_rates(rates_flat), coef, lam, dm)
        q = np.zeros((n, h, w), dtype=np.int16); s = np.zeros(n, dtype=np.int32)
        assert O.orc_rdoq_bdpcm(w, h, bd, qp, 0, dm, lam, P(rates_flat), P(coef), n, P(q), P(s)) == 0
        assert np.array_equal(r['q'], q), (w, h, int((r['q'] != q).any(axis=(1, 2)).sum()))
        assert np.array_equal(r['abs_sum'], s) and (s > 0).sum() > n // 10, (w, h, int((s > 0).sum()))


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'enc_identity')), reason='oracle/_ref/enc_identity not built')
@pytest.mark.parametrize("W,H,F,preset,qp,min_bdpcm", [(80, 44, 4, 0, 32, 100), (176, 144, 3, 0, 27, 2000)])
def test_bitstream_identity_with_bdpcm_on_the_gpu(tmp_path, W, H, F, preset, qp, min_bdpcm):
    import vvenc_b200._lib as VL
    from test_encoder_identity import _identity_bdpcm
    kb = _identity_bdpcm(tmp_path, W, H, F, preset, qp, VL.LIB_PATH, min_bdpcm, timeout=1500)
    print('encoder identity with BDPCM on the GPU:', W, H, F, preset, kb)


@pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')
def test_rdoq_bdpcm_binding_on_the_real_library():
    """forwardRDPCMB200 next to QuantRDOQ::forwardRDPCM, and the inverse path of the BDPCM levels through invTransformNxNB200 next to TrQuant::invTransformNxN"""
    import vvenc_b200._lib as VL
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', '_integration_host_run.py'), VL.LIB_PATH, 'rdoq'], capture_output=True, text=True, timeout=400)
    assert out.returncode == 0, out.stderr[-3000:]
    b = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith('RESULT ')][-1][len('RESULT '):])['rdoq_bdpcm']
    assert b['cases'] == 140 and b['non_empty'] > 70 and b['bad'] == [], b


# ---- second engine of vvb_rdoq (vvb_set_rdoq_engine 2: accumulated templates + cost tables; rq_quant_tu_v2 is pinned on the CPU against the member like the first engine)
def test_gpu_rdoq_second_engine_vs_golden_and_first_engine(gpu, golden_rdoq):
    from _libs import dq_oracle, P
    O = dq_oracle()
    g = golden_rdoq
    gpu.eng.set_rdoq_engine(2)
    try:
        nonzero = 0
        for i, row in enumerate(C.rdoq_cases()):
            w, h, bd, qp, lam1000, scale, decay10, comp, lf, sbt, intra, sh, cb, thr, init_id, seed = [int(v) for v in row]
            par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, sign_hiding=bool(sh), lfnst_idx=lf, is_chroma=comp > 0)
            r = gpu.eng.rdoq(par, gpu.eng.rdoq_rates(g['rates'][i]), C.rdoq_inputs(row)[None], lam1000 / 1000.0, thr, sbt)
            assert np.array_equal(r['q'][0], g['q_%d' % i]) and (int(r['abs_sum'][0]), int(r['last_pos'][0])) == tuple(int(v) for v in g['meta'][i]), (i, [int(v) for v in row])
            nonzero += int(r['last_pos'][0] >= 0)
        assert nonzero > 100
        rs = np.random.RandomState(81)
        luma_rows = [i for i, r in enumerate(g['cases']) if int(r[7]) == 0]
        for (w, h, n, qp, lam, sbt, lf, sh) in ((4, 4, 60000, 32, 57.3, 0, 0, 1), (8, 8, 30000, 27, 30.0, 0, 1, 0), (16, 16, 6000, 37, 120.0, 0, 0, 1), (32, 32, 1500, 32, 57.3, 1, 0, 1), (64, 64, 300, 22, 11.7, 0, 0, 0), (16, 64, 500, 32, 30.0, 0, 2, 1)):
            scale = rs.choice([3, 10, 40, 150, 600, 2500], size=(n, 1, 1))
            coef = rs.laplace(0, 1.0, size=(n, h, w)) * scale * (1.0 / (1 + np.add.outer(np.arange(h), np.arange(w))) ** 0.7)
            coef = np.clip(coef, -32768, 32767).astype(np.int32)
            coef[:, :, 32:] = 0; coef[:, 32:, :] = 0
            rates_flat = np.ascontiguousarray(g['rates'][luma_rows[int(rs.randint(len(luma_rows)))]])
            par = gpu.eng.tu_par(w, h, 0, 0, 10, qp, sign_hiding=bool(sh), lfnst_idx=lf)
            r2 = gpu.eng.rdoq(par, gpu.eng.rdoq_rates(rates_flat), coef, lam, 8, sbt)
            q = np.zeros((n, h, w), dtype=np.int16); s = np.zeros(n, dtype=np.int32); l = np.zeros(n, dtype=np.int32)
            assert O.orc_rdoq(w, h, 10, qp, 0, lf, sbt, sh, lam, 8, P(rates_flat), P(coef), n, P(q), P(s), P(l)) == 0
            assert np.array_equal(r2['q'], q) and np.array_equal(r2['abs_sum'], s) and np.array_equal(r2['last_pos'], l), (w, h, int((r2['q'] != q).any(axis=(1, 2)).sum()))
    finally:
        gpu.eng.set_rdoq_engine(1)
