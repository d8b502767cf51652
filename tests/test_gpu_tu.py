"""GPU parity (-m gpu) of the inverse TU path and the fused TU round trip (SURVEY 8f rank 1), through the C ABI:
golden vectors from the unmodified reference, oracle comparison on seeded batches (compact pools and resident planes),
and algebraic properties at full picture size."""
import numpy as np
import pytest
import cases as C
import impls

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return impls.GpuImpl(0)


def test_gpu_inverse_path_golden(gpu, golden_tu):
    assert impls.run_itq(gpu, golden_tu['itq_rows'], golden_tu['itq_coef'], golden_tu['itq_resi']) == []


def test_gpu_tu_roundtrip_golden(gpu, golden_tu):
    assert impls.run_rt(gpu, golden_tu['rt_rows'], golden_tu['rt_q'], golden_tu['rt_reco'], golden_tu['rt_meta']) == []


SHAPES = ((4, 4, 0, 0), (8, 8, 2, 2), (16, 16, 0, 0), (16, 16, 2, 1), (32, 32, 1, 2), (32, 32, 0, 0), (64, 64, 0, 0), (4, 16, 2, 1), (64, 8, 0, 0),
          (16, 64, 0, 0), (32, 4, 2, 2), (8, 32, 0, 0), (64, 32, 0, 0))


def test_gpu_inverse_batch_vs_oracle(gpu):
    O = impls.OracleImpl()
    rs = np.random.RandomState(808)
    for (w, h, th, tv) in SHAPES:
        n = 67 if w * h < 4096 else 35                       # not a multiple of the teams per CTA: tail teams idle
        amp = np.array([32767, 3000, 60, 3])[rs.randint(0, 4, n)]
        q = (rs.randint(-1000, 1001, size=(n, h, w)) * amp[:, None, None] // 1000).astype(np.int16)
        q[rs.rand(n, h, w) < 0.6] = 0
        q[0] = 32767; q[1] = -32768; q[2] = 0
        for bd, qp in ((10, int(rs.randint(0, 64))), (8, int(rs.randint(0, 64))), (12, int(rs.randint(-20, 64)))):
            par = gpu.eng.tu_par(w, h, th, tv, bd, qp, False, False)
            r = gpu.eng.inv_trquant(par, q)
            for i in range(n):
                _, e = O.inv_transform_quant(th, tv, np.ascontiguousarray(q[i]), w, h, bd, qp, w)
                assert np.array_equal(r[i], e), (w, h, th, tv, bd, qp, i)


def _pool(rs, n, w, h, bd=10):
    mx = (1 << bd) - 1
    org = rs.randint(0, mx + 1, size=(n, h, w))
    amp = np.array([mx, 300, 40, 6, 0])[rs.randint(0, 5, n)]
    noise = rs.randint(-1000, 1001, size=(n, h, w)) * amp[:, None, None] // 1000
    pred = np.clip(org + noise, 0, mx)
    pred[0] = mx - org[0]                                     # large residuals of both signs
    return org.astype(np.int16), pred.astype(np.int16)


def test_gpu_tu_roundtrip_batch_vs_oracle(gpu):
    O = impls.OracleImpl()
    rs = np.random.RandomState(909)
    for (w, h, th, tv) in SHAPES:
        n = 67 if w * h < 4096 else 35
        for bd in (10, 8):
            org, pred = _pool(rs, n, w, h, bd)
            qp = int(rs.randint(8, 52)); irap = int(rs.randint(0, 2))
            par = gpu.eng.tu_par(w, h, th, tv, bd, qp, bool(irap), False)
            r = gpu.eng.tu_roundtrip(par, org, pred)
            zeros = 0
            for i in range(n):
                q, reco, m = O.tu_roundtrip(th, tv, np.ascontiguousarray(org[i]), w, np.ascontiguousarray(pred[i]), w, w, h, bd, qp, irap)
                x = r['res'][i]
                got = [int(x['dist_reco']), int(x['dist_resi']), int(x['dist_zero']), int(x['abs_sum']), int(x['last_pos'])]
                assert np.array_equal(r['q'][i], q) and np.array_equal(r['reco'][i], reco) and got == m, (w, h, th, tv, bd, qp, i, got, m)
                zeros += m[3] == 0
            assert 0 < zeros < n, (w, h, zeros)               # both branches (inverse / zero residual) are exercised


def test_gpu_tu_roundtrip_planes_vs_pool(gpu):
    """plane-addressed variant == pool variant on the same pels (odd prediction displacements included)"""
    rs = np.random.RandomState(1001)
    W, H, m = 256, 128, 16
    S = W + 2 * m
    base = rs.randint(0, 1024, size=(H + 2 * m, S)).astype(np.int16)
    pred_pl = np.clip(base.astype(np.int32) + rs.randint(-30, 31, size=base.shape), 0, 1023).astype(np.int16)
    gpu.eng.upload_plane(0, base, W, H, m, 10)
    gpu.eng.upload_plane(1, pred_pl, W, H, m, 10)
    for (w, h, th, tv) in ((8, 8, 0, 0), (16, 16, 2, 2), (32, 32, 0, 0), (64, 64, 0, 0), (16, 4, 1, 2)):
        xs = np.arange(0, W - w + 1, w); ys = np.arange(0, H - h + 1, h)
        B = np.zeros(len(xs) * len(ys), dtype=gpu.V.BLOCK_DT)
        k = 0
        for y in ys:
            for x in xs:
                B[k] = (x, y, 0, 0, 0, 0, 0, 0, int(rs.randint(-5, 6)), int(rs.randint(-5, 6))); k += 1
        par = gpu.eng.tu_par(w, h, th, tv, 10, 30, False, False)
        a = gpu.eng.tu_roundtrip_planes(par, 0, 1, B)
        org = np.stack([base[m + b['y']:m + b['y'] + h, m + b['x']:m + b['x'] + w] for b in B])
        pred = np.stack([pred_pl[m + b['y'] + b['start_y']:m + b['y'] + b['start_y'] + h, m + b['x'] + b['start_x']:m + b['x'] + b['start_x'] + w] for b in B])
        b_ = gpu.eng.tu_roundtrip(par, org, pred)
        assert np.array_equal(a['q'], b_['q']) and np.array_equal(a['reco'], b_['reco']) and np.array_equal(a['res'], b_['res']), (w, h)


def test_gpu_tu_roundtrip_properties_full_size(gpu):
    """3840x2160 worth of 16x16 TUs: (1) pred == org -> all-zero levels, reco == org, all distortions 0;
    (2) fused levels == vvb_fwd_trquant levels and fused reco == clip(pred + vvb_inv_trquant(levels)) -- the fused kernel agrees with the
    separately tested pieces on 32400 TUs; (3) dist_zero == sum (org-pred)^2 computed in numpy."""
    rs = np.random.RandomState(2002)
    w = h = 16; n = (3840 // w) * (2160 // h)
    org = rs.randint(0, 1024, size=(n, h, w)).astype(np.int16)
    par = gpu.eng.tu_par(w, h, 0, 0, 10, 27, False, False)
    r = gpu.eng.tu_roundtrip(par, org, org)
    assert not r['q'].any() and np.array_equal(r['reco'], org)
    assert not r['res']['dist_reco'].any() and not r['res']['dist_resi'].any() and not r['res']['dist_zero'].any() and not r['res']['abs_sum'].any()
    pred = np.clip(org.astype(np.int32) + rs.randint(-50, 51, size=org.shape), 0, 1023).astype(np.int16)
    r = gpu.eng.tu_roundtrip(par, org, pred)
    resi = (org.astype(np.int32) - pred).astype(np.int16)
    f = gpu.eng.fwd_trquant(par, resi, want_coef=False)
    assert np.array_equal(f['q'], r['q']) and np.array_equal(f['abs_sum'], r['res']['abs_sum']) and np.array_equal(f['last_pos'], r['res']['last_pos'])
    rec = gpu.eng.inv_trquant(par, r['q']).astype(np.int32)
    rec[r['res']['abs_sum'] == 0] = 0
    reco = np.clip(pred.astype(np.int32) + rec, 0, 1023)
    assert np.array_equal(reco.astype(np.int16), r['reco'])
    d = org.astype(np.int64) - pred
    assert np.array_equal((d * d).sum(axis=(1, 2)).astype(np.uint64), r['res']['dist_zero'])
    e = org.astype(np.int64) - reco
    assert np.array_equal((e * e).sum(axis=(1, 2)).astype(np.uint64), r['res']['dist_reco'])
    g = d - rec
    assert np.array_equal((g * g).sum(axis=(1, 2)).astype(np.uint64), r['res']['dist_resi'])


# ------------------------------------------------------------------------------------------ MCTF apply stage (SURVEY 8f rank 3)
def test_gpu_mctf_apply_golden(gpu, golden_mctf_apply):
    """xFinalizeBlkLine for whole small pictures: motion compensation with the 6/4-tap filters, planar correction, bilateral blend -- equal to the
    reference's output (float arithmetic included), 8 and 10 bit, unit sizes 8/16/32, 2..8 references, clipped edge blocks"""
    O = impls.OracleImpl()
    for k, (seed, W, H, refs, bs, bd, tap4, planar) in enumerate(C.MCTF_APPLY_CASES):
        case = C.mctf_apply_case(seed, W, H, 24, refs, bs, bd)
        m = case['margin']
        gpu.eng.upload_plane(0, case['org'], W, H, m, bd)
        for r in range(refs):
            gpu.eng.upload_plane(1 + r, case['refs'][r], W, H, m, bd)
        mv = np.zeros(case['mvs'].shape[:2], dtype=gpu.V.MCTF_MV_DT)
        mv['x'] = case['mvs'][..., 0]; mv['y'] = case['mvs'][..., 1]; mv['error'] = case['mvs'][..., 2]; mv['rmsme'] = case['mvs'][..., 3]
        got = gpu.eng.mctf_apply(0, list(range(1, 1 + refs)), mv, bs, case['strengths'], case['ws'], case['sigma'], W, H, planar=bool(planar), low_res_filter=bool(tap4))
        exp = golden_mctf_apply['apply_%d' % k]
        assert np.array_equal(got, exp), (seed, int(np.abs(got.astype(int) - exp).max()), np.argwhere(got != exp)[:4])
        assert np.array_equal(impls.mctf_apply_expected(O.L, 'orc', case, tap4, planar), exp)


def test_gpu_mctf_calc_var_golden(gpu, golden_mctf_apply):
    plane = golden_mctf_apply['var_plane']
    H, W = plane.shape
    gpu.eng.upload_plane(0, np.ascontiguousarray(plane), W, H, 0, 10)
    blocks = np.zeros(len(golden_mctf_apply['var_blocks']), dtype=gpu.V.MCTF_DT)
    b = golden_mctf_apply['var_blocks']
    blocks['x'] = b[:, 0]; blocks['y'] = b[:, 1]; blocks['w'] = b[:, 2]; blocks['h'] = b[:, 3]
    assert np.array_equal(gpu.eng.mctf_calc_var(0, blocks), golden_mctf_apply['var_expect'])


# ------------------------------------------------------------------------------------------ fractional-pel refinement grid (SURVEY 8f rank 2)
def test_gpu_frac_cost_grid_golden(gpu, golden_frac):
    """every quarter-pel offset (-3..3)^2 around integer vectors of mixed alignment: two-pass 8-tap interpolation + SAD / SATD equal to the
    reference's filterHor/filterVer + distFunc results (8 and 10 bit, blocks 8..64, extreme content)"""
    for ci, (seed, bd) in enumerate(C.FRAC_CASES):
        case = C.frac_case(seed, bit_depth=bd)
        gpu.eng.upload_plane(0, case['org'], case['W'], case['H'], case['margin'], bd)
        gpu.eng.upload_plane(1, case['ref'], case['W'], case['H'], case['margin'], bd)
        for li, (fam, w, h, b) in enumerate(case['lists']):
            blk = np.zeros(len(b), dtype=gpu.V.BLOCK_DT)
            blk['x'] = b[:, 0]; blk['y'] = b[:, 1]; blk['start_x'] = b[:, 4]; blk['start_y'] = b[:, 5]
            rt, alt = C.frac_filter_of(li)
            got = gpu.eng.frac_cost_grid(gpu.V.DF_SAD if fam == 1 else gpu.V.DF_HAD, 0, 1, blk, w, h, rt, alt)
            exp = golden_frac['c%d_l%d' % (ci, li)]
            assert np.array_equal(got, exp), (seed, fam, w, h, np.argwhere(got != exp)[:5], got[got != exp][:4], exp[got != exp][:4])


def test_gpu_frac_grid_centre_equals_integer_distortion(gpu):
    """property at full picture size: the centre entry of the table (offset 0,0: both passes with the single tap 64) is the integer-pel SAD / SATD"""
    rs = np.random.RandomState(77)
    W, H, m = 3840, 2160, 16
    S = W + 2 * m
    org = rs.randint(0, 1024, size=(H + 2 * m, S)).astype(np.int16)
    ref = np.clip(org.astype(np.int32) + rs.randint(-20, 21, size=org.shape), 0, 1023).astype(np.int16)
    gpu.eng.upload_plane(0, org, W, H, m, 10); gpu.eng.upload_plane(1, ref, W, H, m, 10)
    xs, ys = np.meshgrid(np.arange(0, W, 16), np.arange(0, H, 16))
    blk = np.zeros(xs.size, dtype=gpu.V.BLOCK_DT)
    blk['x'] = xs.ravel(); blk['y'] = ys.ravel(); blk['start_x'] = rs.randint(-3, 4, size=xs.size); blk['start_y'] = rs.randint(-3, 4, size=xs.size)
    blk['left'] = -8; blk['right'] = 8; blk['top'] = -8; blk['bottom'] = 8
    t = gpu.eng.frac_cost_grid(gpu.V.DF_HAD, 0, 1, blk, 16, 16, 2, False)
    pat = np.zeros(1, dtype=gpu.V.MV_DT)
    cost, _ = gpu.eng.cost_pattern(gpu.V.DF_HAD, 0, 1, blk, 16, 16, pat, gpu.eng.me_par(0.0), want_best=False)
    assert np.array_equal(t[:, 3, 3], cost[:, 0])


@pytest.mark.parametrize("bd", [10, 8])
def test_gpu_frac_cost_grid_generic_shapes_vs_oracle(gpu, bd):
    """the rest of xPatternRefinement's shapes (frac_grid_generic_kernel): rectangular PUs on 16x8 / 8x16 / 8x4 / 4x8 Hadamard tiles (fp64 normalisation), 4-pel sides,
    DF_HAD_fast with its 16x16_fast tiles, SAD on all of them; every entry of the 7x7 table against the oracle (which equals the reference member, CPU suite)"""
    from _libs import oracle, P, PO
    O = oracle()
    case = C.frac_case(9090 + bd, bit_depth=bd)
    S = case['stride']; base = case['margin'] * S + case['margin']
    gpu.eng.upload_plane(0, case['org'], case['W'], case['H'], case['margin'], bd)
    gpu.eng.upload_plane(1, case['ref'], case['W'], case['H'], case['margin'], bd)
    rs = np.random.RandomState(3 + bd)
    fams = {1: gpu.V.DF_SAD, 2: gpu.V.DF_HAD, 3: gpu.V.DF_HAD_FAST}
    shapes = [(2, 16, 8), (2, 8, 16), (2, 32, 16), (2, 16, 32), (2, 8, 4), (2, 4, 8), (2, 4, 4), (2, 64, 32), (2, 32, 64), (2, 4, 16), (2, 16, 4), (2, 64, 16), (2, 8, 64),
              (3, 32, 32), (3, 64, 64), (3, 16, 16), (3, 8, 8), (3, 32, 16),
              (1, 4, 8), (1, 8, 4), (1, 4, 4), (1, 64, 32), (1, 16, 64)]
    for li, (fam, w, h) in enumerate(shapes):
        n = 5
        b = np.zeros((n, 6), dtype=np.int32)
        for k in range(n):
            b[k] = (int(rs.randint(0, case['W'] - w + 1)), int(rs.randint(0, case['H'] - h + 1)), w, h, int(rs.randint(-9, 10)), int(rs.randint(-9, 10)))
        b[0, :2] = 0
        blk = np.zeros(n, dtype=gpu.V.BLOCK_DT)
        blk['x'] = b[:, 0]; blk['y'] = b[:, 1]; blk['start_x'] = b[:, 4]; blk['start_y'] = b[:, 5]
        rt, alt = ((2, 0), (2, 0), (0, 0), (1, 0), (2, 1))[li % 5]
        if w * h == 16 and rt != 2:
            rt = 2
        got = gpu.eng.frac_cost_grid(fams[fam], 0, 1, blk, w, h, rt, alt)
        exp = np.zeros((n, 7, 7), dtype=np.uint32)
        O.orc_frac_cost_grid(PO(case['org'], base), S, PO(case['ref'], base), S, P(np.ascontiguousarray(b)), n, fam, bd, rt, alt, P(exp))
        assert np.array_equal(got, exp), (bd, fam, w, h, rt, alt, np.argwhere(got != exp)[:5], got[got != exp][:4], exp[got != exp][:4])


def test_gpu_sign_bit_hiding_vs_oracle(gpu):
    """vvb_tu_par.sign_hiding: the levels leave the device as Quant::quant leaves them after xSignBitHidingHDQ (Quant.cpp:377-518) -- forward call (CUDA-core
    kernels: the tensor engine has no sign-bit hiding) and the fused TU round trip (the hidden levels are the ones dequantised); every TU against the oracle, which
    equals the reference (CPU suite)"""
    import ctypes
    from _libs import oracle, P
    O = oracle()
    rs = np.random.RandomState(909)
    changed = 0
    for (w, h, th, tv) in ((4, 4, 0, 0), (8, 8, 2, 2), (16, 16, 0, 0), (16, 16, 2, 1), (32, 32, 1, 2), (32, 32, 0, 0), (64, 64, 0, 0), (4, 16, 2, 1), (64, 8, 0, 0), (16, 64, 0, 0), (32, 4, 2, 2), (8, 32, 0, 0)):
        n = 48 if w * h < 4096 else 20
        amp = np.array([1023, 300, 40, 8])[rs.randint(0, 4, n)]
        resi = (rs.randint(-1000, 1001, size=(n, h, w)) * amp[:, None, None] // 1000).astype(np.int16)
        qp = int(rs.randint(14, 46)); irap = int(rs.randint(0, 2))
        par = gpu.eng.tu_par(w, h, th, tv, 10, qp, bool(irap), False, True)
        r = gpu.eng.fwd_trquant(par, resi)
        plain = gpu.eng.fwd_trquant(gpu.eng.tu_par(w, h, th, tv, 10, qp, bool(irap), False, False), resi)
        for i in range(n):
            coef = np.zeros((h, w), dtype=np.int32); q = np.zeros((h, w), dtype=np.int16); s = ctypes.c_int32(); lp = ctypes.c_int32()
            assert O.orc_transform_quant_ex(th, tv, P(np.ascontiguousarray(resi[i])), w, w, h, 10, qp, irap, 1, P(coef), P(q), ctypes.byref(s), ctypes.byref(lp)) == 0
            assert np.array_equal(r['q'][i], q) and int(r['abs_sum'][i]) == s.value and int(r['last_pos'][i]) == lp.value, (w, h, th, tv, i, qp, int((r['q'][i] != q).sum()))
            changed += int(not np.array_equal(plain['q'][i], q))
        # fused round trip with hiding
        org = rs.randint(0, 1024, size=(8, h, w)).astype(np.int16); pred = np.clip(org + rs.randint(-120, 121, size=org.shape), 0, 1023).astype(np.int16)
        rt = gpu.eng.tu_roundtrip(par, org, pred)
        for i in range(8):
            q2 = np.zeros((h, w), dtype=np.int16); rc2 = np.zeros((h, w), dtype=np.int16); o4 = np.zeros(4, dtype=np.uint64)
            O.orc_tu_roundtrip_ex(th, tv, P(np.ascontiguousarray(org[i])), w, P(np.ascontiguousarray(pred[i])), w, w, h, 10, qp, irap, 1, P(q2), P(rc2), w, P(o4))
            assert np.array_equal(rt['q'][i], q2) and np.array_equal(rt['reco'][i], rc2) and int(rt['res'][i]['dist_reco']) == int(o4[0]), (w, h, i)
    assert changed > 60


def test_gpu_lfnst_forward_vs_oracle(gpu):
    """vvb_tu_par.lfnst_*: transform zero-out + LFNST kernel + quantiser on coefficient group 0 (TrQuant::xFwdLfnst, TrQuant.cpp:942-1048) for every TU shape that can
    carry LFNST, all kernel sets, both indices, transposed and not, with and without sign hiding; coefficients, levels, absSum, lastPos and the RDOQ flag equal
    the oracle (= the reference, CPU suite)"""
    import ctypes
    import vvenc_b200 as V
    from _libs import oracle, P
    O = oracle()
    rs = np.random.RandomState(4321)
    for (w, h) in ((4, 4), (8, 8), (4, 8), (8, 4), (16, 16), (4, 16), (16, 4), (8, 16), (32, 32), (32, 8), (64, 64), (16, 64), (64, 4)):
        for (st, idx, tr) in ((0, 1, 0), (1, 2, 0), (2, 1, 1), (3, 2, 1), (1, 1, 1), (3, 1, 0)):
            n = 24
            amp = np.array([1023, 300, 40])[rs.randint(0, 3, n)]
            resi = (rs.randint(-1000, 1001, size=(n, h, w)) * amp[:, None, None] // 1000).astype(np.int16)
            qp = int(rs.randint(16, 46)); irap = int(rs.randint(0, 2)); sh = int(rs.randint(0, 2)); dq = int(rs.randint(0, 2))
            par = gpu.eng.tu_par(w, h, V.DCT2, V.DCT2, 10, qp, bool(irap), bool(dq), bool(sh), idx, st, bool(tr))
            r = gpu.eng.fwd_trquant(par, resi)
            for i in range(n):
                coef = np.zeros((h, w), dtype=np.int32); q = np.zeros((h, w), dtype=np.int16); s = ctypes.c_int32(); lp = ctypes.c_int32()
                assert O.orc_transform_quant_lfnst(P(np.ascontiguousarray(resi[i])), w, w, h, 10, qp, irap, sh, st, idx, tr, P(coef), P(q), ctypes.byref(s), ctypes.byref(lp)) == 0
                assert np.array_equal(r['coef'][i], coef), (w, h, st, idx, tr, i, np.argwhere(r['coef'][i] != coef)[:4])
                assert np.array_equal(r['q'][i], q) and int(r['abs_sum'][i]) == s.value and int(r['last_pos'][i]) == lp.value, (w, h, st, idx, tr, i, qp, sh)
                assert int(r['need_rdoq'][i]) == O.orc_need_rdoq(P(coef), w, h, 10, qp, dq), (w, h, i)


@pytest.mark.parametrize("engine", [1, 0])
def test_gpu_dep_quant_golden(gpu, golden_depquant, engine):
    """DepQuant::xQuantDQ on the device against what the reference produced (tests/golden/golden_v5_depquant.npz): every row of cases.dq_cases(), scalar and x86
    member semantics, the Quantizer constants derived inside the library against the reference's"""
    import ctypes
    import vvenc_b200._lib as L
    g = golden_depquant
    gpu.eng.set_depquant_engine(engine)           # 1: four lanes per TU, 0: one thread per TU
    rows = C.dq_cases()
    assert np.array_equal(rows, g['cases'])
    nonzero = 0
    for i, row in enumerate(rows):
        w, h, bd, qp, lam1000, scale, decay10, mts, lf, sbt, intra, init_id, seed = [int(v) for v in row]
        coef = C.dq_inputs(row)[None]
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, lfnst_idx=lf)
        rates = gpu.eng.dq_rates(g['rates'][i])
        dq = L.vvb_dq_par(lam1000 / 1000.0, 8, C.dq_zero_out(row), 0, 0)
        k = np.zeros(9, dtype=np.int64)
        assert gpu.eng.lib.vvb_dep_quant_constants(ctypes.byref(par), ctypes.byref(dq), k.ctypes.data_as(ctypes.c_void_p)) == 0
        assert np.array_equal(k, g['consts'][i]), i
        for scalar in (1, 0):
            r = gpu.eng.dep_quant(par, rates, coef, lam1000 / 1000.0, 8, C.dq_zero_out(row), scalar_members=bool(scalar))
            name = 'q_x86_%d' % i
            want = g['q_scalar_%d' % i] if (scalar or name not in g) else g[name]
            assert np.array_equal(r['q'][0], want), (i, scalar, [int(v) for v in row])
            assert (int(r['abs_sum'][0]), int(r['last_pos'][0])) == tuple(int(v) for v in g['meta'][i, 0 if scalar else 1]), (i, scalar)
        nonzero += int(r['last_pos'][0] >= 0)
    gpu.eng.set_depquant_engine(1)
    assert nonzero > 100


@pytest.mark.parametrize("engine", [1, 0])
def test_gpu_dep_quant_batches_vs_oracle(gpu, golden_depquant, engine):
    """a picture's worth of TUs per launch (more TUs than resident threads for the small shapes: the threads stride over the list and reuse their arena slot),
    the need_rdoq mask of useSelectiveRdoq, against the CPU build of the restatement on the same inputs; rate tables of a reference CABAC state"""
    import ctypes
    from _libs import dq_oracle, P
    O = dq_oracle()
    g = golden_depquant
    gpu.eng.set_depquant_engine(engine)
    rs = np.random.RandomState(77)
    for (w, h, n, qp, lam, zo, lf) in ((4, 4, 90000, 32, 57.3, 0, 0), (8, 8, 30000, 27, 30.0, 0, 1), (16, 16, 6000, 37, 120.0, 0, 0), (32, 32, 1500, 32, 57.3, 1, 0),
                                       (64, 64, 300, 22, 11.7, 0, 0), (32, 8, 3000, 42, 800.0, 0, 0), (16, 64, 500, 32, 30.0, 0, 2)):
        scale = rs.choice([3, 10, 40, 150, 600, 2500], size=(n, 1, 1))
        coef = rs.laplace(0, 1.0, size=(n, h, w)) * scale * (1.0 / (1 + np.add.outer(np.arange(h), np.arange(w))) ** 0.7)
        coef = np.clip(coef, -32768, 32767).astype(np.int32)
        coef[:, :, 32:] = 0; coef[:, 32:, :] = 0
        rates_flat = np.ascontiguousarray(g['rates'][int(rs.randint(len(g['rates'])))])
        mask = (rs.randint(0, 8, size=n) > 0).astype(np.uint8)
        par = gpu.eng.tu_par(w, h, 0, 0, 10, qp, lfnst_idx=lf)
        r = gpu.eng.dep_quant(par, gpu.eng.dq_rates(rates_flat), coef, lam, 8, zo, need_rdoq=mask)
        q = np.zeros((n, h, w), dtype=np.int16); s = np.zeros(n, dtype=np.int32); l = np.zeros(n, dtype=np.int32)
        assert O.orc_dep_quant(w, h, 10, qp, lam, 8, zo, 1 if lf else 0, 0, P(rates_flat), P(coef), n, P(q), P(s), P(l)) == 0
        q[mask == 0] = 0; s[mask == 0] = 0; l[mask == 0] = -1
        assert np.array_equal(r['q'], q), (w, h, int((r['q'] != q).any(axis=(1, 2)).sum()))
        assert np.array_equal(r['abs_sum'], s) and np.array_equal(r['last_pos'], l), (w, h)
        assert (l >= 0).sum() > n // 4, (w, h, int((l >= 0).sum()))
    gpu.eng.set_depquant_engine(1)


def test_gpu_transform_skip_and_chroma_vs_oracle(gpu):
    """vvb_tu_par.transform_skip / input_bit_depth_delta / is_chroma: forward (xTransformSkip + quantiser at the transform-skip QP, xNeedRDOQ with its chroma constant),
    inverse (dequant without the transform shift + xITransformSkip) and the fused round trip against the oracle restatements that tests/test_oracle_vs_reference.py pins
    to the reference members; batches per case row so that the EXT instantiations run with full CTAs"""
    import ctypes
    from _libs import oracle, P
    O = oracle()
    I32 = ctypes.c_int32
    nfwd = 0; ninv = 0; nrt = 0
    for row in C.ts_cases():
        w, h, st, bd, amp, qp, irap, sh, dq, ts, delta, comp, seed = [int(v) for v in row]
        rs = np.random.RandomState(seed)
        n = 40
        resi = rs.randint(-amp, amp + 1, size=(n, h, w)).astype(np.int16)
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, bool(irap), bool(dq), bool(sh), transform_skip=bool(ts), input_bit_depth_delta=delta, is_chroma=bool(comp))
        r = gpu.eng.fwd_trquant(par, resi)
        for i in range(n):
            cO = np.zeros((h, w), np.int32); qO = np.zeros((h, w), np.int16); sO = I32(); lO = I32()
            if ts:
                assert O.orc_transform_quant_ts(P(resi[i]), w, w, h, bd, qp, irap, sh, delta, P(cO), P(qO), ctypes.byref(sO), ctypes.byref(lO)) == 0
            else:
                assert O.orc_transform_quant_ex(0, 0, P(resi[i]), w, w, h, bd, qp, irap, sh, P(cO), P(qO), ctypes.byref(sO), ctypes.byref(lO)) == 0
            assert np.array_equal(r['coef'][i], cO) and np.array_equal(r['q'][i], qO), ([int(v) for v in row], i)
            assert int(r['abs_sum'][i]) == sO.value and int(r['last_pos'][i]) == lO.value, ([int(v) for v in row], i)
            assert int(r['need_rdoq'][i]) == O.orc_need_rdoq_ex(P(cO), w, h, bd, qp, dq, ts, delta, comp), ([int(v) for v in row], i)
        nfwd += n
        if ts:
            got = gpu.eng.inv_trquant(par, r['q'])
            for i in range(0, n, 5):
                dO = np.zeros((h, w), np.int32); rO = np.zeros((h, w), np.int16)
                assert O.orc_inv_transform_quant_ts(P(np.ascontiguousarray(r['q'][i])), w, h, bd, qp, delta, P(dO), P(rO), w) == 0
                assert np.array_equal(got[i], rO), ([int(v) for v in row], i)
                ninv += 1
            # fused round trip: residual = org - pred -> skip "transform" -> quant -> dequant -> reconstruct; the levels must equal the separate forward call and
            # the reconstruction pred + residual' clipped to the bit depth
            org = rs.randint(0, 1 << bd, size=(n, h, w)).astype(np.int16)
            pred = np.clip(org.astype(np.int32) - resi, 0, (1 << bd) - 1).astype(np.int16)
            rr = gpu.eng.tu_roundtrip(par, org, pred)
            f2 = gpu.eng.fwd_trquant(par, (org.astype(np.int32) - pred).astype(np.int16))
            assert np.array_equal(rr['q'], f2['q'])
            rec_resi = gpu.eng.inv_trquant(par, f2['q'])
            exp = np.clip(pred.astype(np.int32) + np.where((f2['abs_sum'] > 0)[:, None, None], rec_resi.astype(np.int32), 0), 0, (1 << bd) - 1).astype(np.int16)
            assert np.array_equal(rr['reco'], exp), [int(v) for v in row]
            nrt += n
    assert nfwd == 220 * 40 and ninv > 300 and nrt > 2000, (nfwd, ninv, nrt)


@pytest.mark.parametrize("engine", [1, 0])
def test_gpu_dep_quant_chroma_golden(gpu, golden_depquant, engine):
    """vvb_dep_quant with vvb_tu_par.is_chroma: the chroma scan-table set on the device against the levels the reference produced for Cb components"""
    g = golden_depquant
    gpu.eng.set_depquant_engine(engine)
    rows = C.dq_chroma_cases()
    assert np.array_equal(rows, g['chroma_cases'])
    for i, row in enumerate(rows):
        w, h, bd, qp, lam1000, scale, decay10, lf, intra, init_id, seed = [int(v) for v in row]
        coef = C.dq_chroma_inputs(row)[None]
        par = gpu.eng.tu_par(w, h, 0, 0, bd, qp, lfnst_idx=lf, is_chroma=True)
        r = gpu.eng.dep_quant(par, gpu.eng.dq_rates(g['chroma_rates'][i]), coef, lam1000 / 1000.0, 8, False)
        assert np.array_equal(r['q'][0], g['cq_%d' % i]), (i, [int(v) for v in row])
        assert (int(r['abs_sum'][0]), int(r['last_pos'][0])) == tuple(int(v) for v in g['chroma_meta'][i]), i
    gpu.eng.set_depquant_engine(1)


def test_gpu_dep_quant_dequantiser_vs_oracle(gpu):
    """vvb_inv_trquant with vvb_tu_par.dep_quant: DepQuant::dequant's state machine (levels -> qIdx by one warp per TU with a shuffle scan of the state maps) + the
    inverse transform, batches of TUs with random last positions, against the oracle restatement pinned to the reference member"""
    from _libs import oracle, P
    O = oracle()
    for row in C.dqd_cases():
        th, tv, w, h, bd, qp, amp, seed = [int(v) for v in row]
        so = np.zeros(1024, np.int32); O.orc_scan_order(w, h, P(so))
        n = 24
        qs = np.zeros((n, h, w), dtype=np.int16)
        for i in range(n):
            r2 = row.copy(); r2[7] = seed * 31 + i
            qs[i], _ = C.dqd_inputs(r2, so)
        par = gpu.eng.tu_par(w, h, th, tv, bd, qp, False, True)
        got = gpu.eng.inv_trquant(par, qs)
        for i in range(n):
            cO = np.zeros((h, w), np.int32); rO = np.zeros((h, w), np.int16)
            assert O.orc_inv_transform_quant_dq(th, tv, P(np.ascontiguousarray(qs[i])), w, h, bd, qp, P(cO), P(rO), w) == 0
            assert np.array_equal(got[i], rO), ([int(v) for v in row], i)


def test_gpu_lfnst_inverse_and_roundtrip_vs_oracle(gpu):
    """vvb_inv_trquant / vvb_tu_roundtrip with vvb_tu_par.lfnst_*: dequantiser (plain or DepQuant's), TrQuant::xInvLfnst on the first 16 scan positions, xIT over the
    top-left 8x8 / 4x4, for every TU shape that can carry LFNST, all kernel sets, both indices, transposed and not, against the oracle restatement that
    tests/test_oracle_vs_reference.py pins to the reference member; then the fused round trip of LFNST TUs (forward LFNST -> levels -> inverse LFNST -> reconstruction ->
    distortions) against the separate calls"""
    import ctypes
    import vvenc_b200 as V
    from _libs import oracle, P
    O = oracle()
    rs = np.random.RandomState(977)
    ninv = 0; nrt = 0; live = 0
    for (w, h) in ((4, 4), (8, 8), (4, 8), (8, 4), (16, 16), (4, 16), (16, 4), (8, 16), (32, 32), (32, 8), (64, 64), (16, 64), (64, 4)):
        so = np.zeros(1024, np.int32); O.orc_scan_order(w, h, P(so))
        for (st, idx, tr) in ((0, 1, 0), (1, 2, 0), (2, 1, 1), (3, 2, 1), (1, 1, 1), (3, 1, 0)):
            for dq in (0, 1):
                n = 24; bd = int(rs.choice([8, 10])); qp = int(rs.randint(-6 * (bd - 8), 64))
                qs = np.zeros((n, h, w), dtype=np.int16)
                for i in range(n):
                    qs[i], _ = C.ilf_inputs(np.array([w, h, bd, qp, 0, idx, dq, int(rs.choice([2, 20, 300, 5000])), int(rs.randint(1 << 30))]), so)
                par = gpu.eng.tu_par(w, h, V.DCT2, V.DCT2, bd, qp, False, bool(dq), False, idx, st, bool(tr))
                got = gpu.eng.inv_trquant(par, qs)
                for i in range(n):
                    cO = np.zeros((h, w), np.int32); rO = np.zeros((h, w), np.int16)
                    assert O.orc_inv_transform_quant_lfnst(P(np.ascontiguousarray(qs[i])), w, h, bd, qp, dq, st, idx, tr, P(cO), P(rO), w) == 0
                    assert np.array_equal(got[i], rO), (w, h, st, idx, tr, dq, bd, qp, i)
                    ninv += 1
            # fused round trip (plain quantiser)
            n = 40; bd = 10; qp = int(rs.randint(12, 40)); irap = int(rs.randint(0, 2)); sh = int(rs.randint(0, 2))
            org = rs.randint(0, 1 << bd, size=(n, h, w)).astype(np.int16)
            amp = np.array([600, 120, 20])[rs.randint(0, 3, n)]
            pred = np.clip(org.astype(np.int32) - (rs.randint(-1000, 1001, size=(n, h, w)) * amp[:, None, None] // 1000), 0, (1 << bd) - 1).astype(np.int16)
            par = gpu.eng.tu_par(w, h, V.DCT2, V.DCT2, bd, qp, bool(irap), False, bool(sh), idx, st, bool(tr))
            rr = gpu.eng.tu_roundtrip(par, org, pred)
            resi = (org.astype(np.int32) - pred).astype(np.int16)
            f2 = gpu.eng.fwd_trquant(par, resi)
            assert np.array_equal(rr['q'], f2['q']) and np.array_equal(rr['res']['abs_sum'], f2['abs_sum']) and np.array_equal(rr['res']['last_pos'], f2['last_pos'])
            assert np.array_equal(rr['need_rdoq'], f2['need_rdoq'])
            rec_resi = np.where((f2['abs_sum'] > 0)[:, None, None], gpu.eng.inv_trquant(par, f2['q']).astype(np.int32), 0)
            for i in range(0, n, 8):
                cO = np.zeros((h, w), np.int32); rO = np.zeros((h, w), np.int16)
                assert O.orc_inv_transform_quant_lfnst(P(np.ascontiguousarray(f2['q'][i])), w, h, bd, qp, 0, st, idx, tr, P(cO), P(rO), w) == 0
                assert np.array_equal(rec_resi[i], rO if f2['abs_sum'][i] > 0 else 0 * rO), (w, h, st, idx, tr, i)
            exp = np.clip(pred.astype(np.int32) + rec_resi, 0, (1 << bd) - 1)
            assert np.array_equal(rr['reco'], exp.astype(np.int16)), (w, h, st, idx, tr)
            d = org.astype(np.int64) - exp
            assert np.array_equal(rr['res']['dist_reco'], (d * d).sum(axis=(1, 2)).astype(np.uint64))
            d = resi.astype(np.int64) - rec_resi
            assert np.array_equal(rr['res']['dist_resi'], (d * d).sum(axis=(1, 2)).astype(np.uint64))
            nrt += n; live += int((f2['abs_sum'] > 0).sum())
    assert ninv == 13 * 6 * 2 * 24 and nrt == 13 * 6 * 40 and live > nrt // 2, (ninv, nrt, live)


def test_gpu_raw_byte_tensor_engine_vs_cuda_core_engine_and_oracle(gpu):
    """vvb_set_tensor_transform(3): the wgmma engine whose MMA operands are the raw bytes of the residual / the stage-1 values (trquant_tc2_kernels.cuh), square TUs
    8..64: compact pools and residuals formed from planes (every pel alignment of org and pred), all transform pairs, 8/10/12 bit, tails that do not fill a tile,
    int16 extremes (the full input domain is exact), with and without the coefficient output -- levels, coefficients, absSum, lastPos and the RDOQ flag equal the
    CUDA-core engine on everything and the oracle on a sample"""
    import vvenc_b200 as V
    O = impls.OracleImpl()
    rs = np.random.RandomState(8086)
    checked = 0
    try:
        for (N, pairs) in ((8, ((0, 0), (2, 2), (1, 2))), (16, ((0, 0), (2, 1))), (32, ((0, 0), (1, 2), (2, 2))), (64, ((0, 0),))):
            for (th, tv) in pairs:
                for bd in (8, 10, 12):
                    n = int(rs.choice([1, 3, 37, 130, 1000])) if N < 64 else int(rs.choice([1, 3, 37, 130]))
                    lim = 1 << bd
                    amp = np.array([lim - 1, lim // 3, 40, 5, 0])[rs.randint(0, 5, n)]
                    resi = (rs.randint(-1000, 1001, size=(n, N, N)) * amp[:, None, None] // 1000).astype(np.int16)
                    resi[0] = np.where((np.arange(N)[None, :] + np.arange(N)[:, None]) % 2 == 0, lim - 1, -(lim - 1))
                    if n > 2:
                        resi[1] = rs.randint(-32768, 32768, size=(N, N))          # any int16 input
                        resi[2] = rs.choice([-32768, 32767], size=(N, N))
                    qp = int(rs.randint(-6 * (bd - 8), 58)); irap = int(rs.randint(0, 2)); dq = int(rs.randint(0, 2))
                    par = gpu.eng.tu_par(N, N, th, tv, bd, qp, bool(irap), bool(dq))
                    gpu.eng.set_tensor_transform(0); a = gpu.eng.fwd_trquant(par, resi)
                    gpu.eng.set_tensor_transform(3); b = gpu.eng.fwd_trquant(par, resi); c = gpu.eng.fwd_trquant(par, resi, want_coef=False)
                    for k in ('coef', 'q', 'abs_sum', 'last_pos', 'need_rdoq'):
                        assert np.array_equal(a[k], b[k]), (N, th, tv, bd, qp, n, k, np.argwhere(a[k] != b[k])[:4])
                        if k != 'coef':
                            assert np.array_equal(a[k], c[k]), (N, th, tv, bd, k)
                    for i in (0, n - 1):
                        if np.abs(resi[i].astype(np.int32)).max() < lim:
                            co, q, s, lp, nr = O.transform_quant(th, tv, np.ascontiguousarray(resi[i]), N, N, N, bd, qp, irap, dq)
                            assert np.array_equal(b['coef'][i], co) and np.array_equal(b['q'][i], q) and (int(b['abs_sum'][i]), int(b['last_pos'][i]), int(b['need_rdoq'][i])) == (s, lp, nr)
                            checked += 1
        # residual from planes: org and pred at every pel alignment
        W, H, m = 320, 192, 16
        a_, b_, S = _tc2_planes(rs, W, H, m)
        po, pp = 0, 1
        gpu.eng.upload_plane(po, a_, W, H, m, 10); gpu.eng.upload_plane(pp, b_, W, H, m, 10)
        for N in (8, 16, 32, 64):
            n = 333 if N < 64 else 45
            blocks = np.zeros(n, dtype=gpu.V.BLOCK_DT)
            blocks['x'] = rs.randint(0, W - N + 1, n); blocks['y'] = rs.randint(0, H - N + 1, n)
            blocks['x'][: n // 2] &= ~7                                           # half of the TUs on the 8-pel grid the encoder uses, the rest anywhere
            blocks['start_x'] = rs.randint(-m, m + 1, n); blocks['start_y'] = rs.randint(-m, m + 1, n)
            par = gpu.eng.tu_par(N, N, 0, 0, 10, int(rs.randint(20, 40)), False, False)
            gpu.eng.set_tensor_transform(0); a = gpu.eng.fwd_trquant_planes(par, po, pp, blocks, want_coef=True)
            gpu.eng.set_tensor_transform(3); b = gpu.eng.fwd_trquant_planes(par, po, pp, blocks, want_coef=True)
            for k in ('coef', 'q', 'abs_sum', 'last_pos', 'need_rdoq'):
                assert np.array_equal(a[k], b[k]), (N, k, np.argwhere(a[k] != b[k])[:4])
            assert (a['abs_sum'] > 0).sum() > n // 2
    finally:
        gpu.eng.set_tensor_transform(3)
    assert checked > 30


def _tc2_planes(rs, W, H, m, bd=10):
    S = W + 2 * m
    a = rs.randint(0, 1 << bd, size=(H + 2 * m, S)).astype(np.int16)
    b = np.clip(np.roll(a, (2, -3), (0, 1)) + rs.randint(-40, 41, size=a.shape), 0, (1 << bd) - 1).astype(np.int16)
    return np.ascontiguousarray(a), np.ascontiguousarray(b), S


def test_gpu_inverse_tensor_engine_vs_cuda_core_engine(gpu):
    """vvb_set_tensor_transform(3) also routes vvb_inv_trquant and the second half of vvb_tu_roundtrip of square 8 / 16 / 32 / 64 TUs through the wgmma inverse engine
    (itrquant_tc_kernels.cuh: dequantised coefficients and first-pass outputs as raw int16 bytes): residuals, reconstructions and the three distortions equal the
    CUDA-core engine for every transform pair, 8 / 10 / 12 bit, plain and DepQuant dequantiser, levels up to the int16 extremes, tails that do not fill a tile, and
    resident-plane addressing with any prediction displacement"""
    rs = np.random.RandomState(4004)
    try:
        for (N, pairs) in ((8, ((0, 0), (2, 2), (1, 2))), (16, ((0, 0), (2, 1))), (32, ((0, 0), (1, 2), (2, 2))), (64, ((0, 0),))):
            for (th, tv) in pairs:
                for bd in (8, 10, 12):
                    for dq in (0, 1):
                        n = int(rs.choice([1, 5, 37, 130, 700]))
                        amp = np.array([32767, 2000, 60, 3, 0])[rs.randint(0, 5, n)]
                        q = (rs.randint(-1000, 1001, size=(n, N, N)) * amp[:, None, None] // 1000).astype(np.int16)
                        q[rs.randint(0, 3, size=q.shape) > 0] = 0
                        if n > 2:
                            q[1] = rs.choice([-32768, 32767], size=(N, N))
                        qp = int(rs.randint(-6 * (bd - 8), 64))
                        par = gpu.eng.tu_par(N, N, th, tv, bd, qp, False, bool(dq))
                        gpu.eng.set_tensor_transform(0); a = gpu.eng.inv_trquant(par, q)
                        gpu.eng.set_tensor_transform(3); b = gpu.eng.inv_trquant(par, q)
                        assert np.array_equal(a, b), (N, th, tv, bd, dq, qp, n, np.argwhere(a != b)[:4])
                    # fused round trip, pools
                    n = int(rs.choice([3, 37, 500])); lim = 1 << bd
                    org = rs.randint(0, lim, size=(n, N, N)).astype(np.int16)
                    amp = np.array([lim // 2, 60, 8, 0])[rs.randint(0, 4, n)]
                    pred = np.clip(org.astype(np.int32) - (rs.randint(-1000, 1001, size=(n, N, N)) * amp[:, None, None] // 1000), 0, lim - 1).astype(np.int16)
                    par = gpu.eng.tu_par(N, N, th, tv, bd, int(rs.randint(0, 50)), bool(rs.randint(0, 2)), False)
                    gpu.eng.set_tensor_transform(0); a = gpu.eng.tu_roundtrip(par, org, pred)
                    gpu.eng.set_tensor_transform(3); b = gpu.eng.tu_roundtrip(par, org, pred); c = gpu.eng.tu_roundtrip(par, org, pred, want_reco=False)
                    for k in ('q', 'reco', 'need_rdoq'):
                        assert np.array_equal(a[k], b[k]), (N, th, tv, bd, k)
                    assert np.array_equal(a['res'], b['res']) and np.array_equal(a['res'], c['res']) and np.array_equal(a['q'], c['q']), (N, th, tv, bd)
                    assert (a['res']['abs_sum'] == 0).any() or n < 30
        W, H, m = 320, 192, 16
        a_, b_, S = _tc2_planes(rs, W, H, m)
        gpu.eng.upload_plane(0, a_, W, H, m, 10); gpu.eng.upload_plane(1, b_, W, H, m, 10)
        for N in (8, 16, 32, 64):
            n = 301 if N < 64 else 40
            blocks = np.zeros(n, dtype=gpu.V.BLOCK_DT)
            blocks['x'] = rs.randint(0, W - N + 1, n); blocks['y'] = rs.randint(0, H - N + 1, n)
            blocks['start_x'] = rs.randint(-m, m + 1, n); blocks['start_y'] = rs.randint(-m, m + 1, n)
            par = gpu.eng.tu_par(N, N, 0, 0, 10, int(rs.randint(20, 40)), False, False)
            gpu.eng.set_tensor_transform(0); a = gpu.eng.tu_roundtrip_planes(par, 0, 1, blocks)
            gpu.eng.set_tensor_transform(3); b = gpu.eng.tu_roundtrip_planes(par, 0, 1, blocks)
            assert np.array_equal(a['q'], b['q']) and np.array_equal(a['reco'], b['reco']) and np.array_equal(a['res'], b['res']) and np.array_equal(a['need_rdoq'], b['need_rdoq']), N
    finally:
        gpu.eng.set_tensor_transform(3)


def test_gpu_tensor_engines_run_at_every_square_size(gpu):
    """with vvb_set_tensor_transform on (any non-zero value: 3 and 1 here) the raw-byte wgmma kernels themselves run for square 8 / 16 / 32 / 64 TUs:
    fwd_trquant_tc2_kernel for vvb_fwd_trquant, inv_trquant_tc_kernel for vvb_inv_trquant, both for vvb_tu_roundtrip -- the kernel names in a torch.profiler
    trace of each call"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    rs = np.random.RandomState(77)

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events()]

    def count(names, kernel, N):
        return sum(1 for e in names if '%s<%d,' % (kernel, N) in e or '%sILi%dE' % (kernel, N) in e)

    for tensor in (3, 1):
        gpu.eng.set_tensor_transform(tensor)
        for N in (8, 16, 32, 64):
            par = gpu.eng.tu_par(N, N, 0, 0, 10, 30, False, False)
            resi = rs.randint(-300, 301, size=(5, N, N)).astype(np.int16)
            org = rs.randint(0, 1024, size=(5, N, N)).astype(np.int16)
            pred = np.clip(org + rs.randint(-60, 61, size=org.shape), 0, 1023).astype(np.int16)
            q = gpu.eng.fwd_trquant(par, resi)['q']
            fwd = kernels(lambda: gpu.eng.fwd_trquant(par, resi))
            inv = kernels(lambda: gpu.eng.inv_trquant(par, q))
            rt = kernels(lambda: gpu.eng.tu_roundtrip(par, org, pred))
            assert count(fwd, 'fwd_trquant_tc2_kernel', N) == 1, (tensor, N, sorted(set(fwd)))
            assert count(inv, 'inv_trquant_tc_kernel', N) == 1, (tensor, N, sorted(set(inv)))
            assert count(rt, 'fwd_trquant_tc2_kernel', N) == 1 and count(rt, 'inv_trquant_tc_kernel', N) == 1, (tensor, N, sorted(set(rt)))
