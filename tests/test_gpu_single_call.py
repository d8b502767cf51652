"""The single-call helpers on borrowed host blocks (vvb_dist_block, vvb_sad_mask_block, vvb_sad_x5_block, vvb_fix_wsse_block, vvb_affine_sobel,
vvb_affine_equal_coeff), which the encoder integration installs in RdCost and AffineGradientSearch:
  * each distortion helper, on strided host blocks, equals its descriptor-list form over the same pels bound as resident planes, and the oracle;
  * the affine helpers equal vvb_affine_eq_batch's derivatives and sums, and the oracle; vvb_affine_equal_coeff adds to the caller's sums;
  * in asynchronous mode every helper returns with its results in place (page-locked outputs, no vvb_synchronize);
  * each distortion helper runs the kernel of its list form and nothing else."""
import ctypes
import os
import re
import numpy as np
import pytest
from _libs import oracle, P, PO

pytestmark = pytest.mark.gpu

W, H, M = 320, 256, 16
S = W + 2 * M
BASE = M * S + M
MS, MH = 160, 136                                # mask table: one GEO-like mask of MH rows of MS weights


@pytest.fixture(scope="module")
def eng():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def _pictures(seed):
    """org and cur, 10-bit, with a margin of M samples, resident as planes 0 and 1 of eng by _upload"""
    rs = np.random.RandomState(seed)
    org = rs.randint(0, 1024, size=(H + 2 * M, S)).astype(np.int16)
    cur = np.clip(org + rs.randint(-40, 41, size=org.shape), 0, 1023).astype(np.int16)
    return rs, org, cur


def _upload(eng, org, cur):
    eng.upload_plane(0, org, W, H, M); eng.upload_plane(1, cur, W, H, M)


def _cand(dt, w, h, ox, oy, cx, cy, sub_shift=0):
    c = np.zeros(1, dtype=dt)
    c['org_plane'] = 0; c['cur_plane'] = 1; c['w'] = w; c['h'] = h; c['sub_shift'] = sub_shift
    c['org_x'] = ox; c['org_y'] = oy; c['cur_x'] = cx; c['cur_y'] = cy
    return c


# ---------------------------------------------------------------------------------------------------- distortions
def test_fix_wsse_block_equals_list_form_and_oracle(eng):
    import vvenc_b200._lib as L
    O = oracle()
    rs, org, cur = _pictures(11)
    _upload(eng, org, cur)
    for (w, h) in ((1, 1), (1, 8), (2, 2), (2, 32), (8, 8), (128, 128)):
        ox, oy = int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1)); cx, cy = int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1))
        o, c = BASE + oy * S + ox, BASE + cy * S + cx
        wt = int(rs.randint(0, 1 << 17))
        got = eng.fix_wsse_block(org.reshape(-1)[o:], S, cur.reshape(-1)[c:], S, w, h, wt)
        lst = int(eng.fix_wsse_batch(_cand(L.CAND_DT, w, h, ox, oy, cx, cy), np.array([wt], dtype=np.uint32))[0])
        exp = O.orc_fix_wsse(PO(org, o), S, PO(cur, c), S, w, h, wt)
        assert got == lst == exp, (w, h, got, lst, exp)


def test_sad_mask_block_equals_list_form_and_oracle(eng):
    import vvenc_b200._lib as L
    O = oracle()
    rs, org, cur = _pictures(12)
    _upload(eng, org, cur)
    table = rs.randint(0, 9, size=(MH, MS)).astype(np.int16)
    eng.mask_upload(table)
    flat = table.reshape(-1)
    for (w, h) in ((8, 8), (16, 16), (32, 64), (64, 8), (128, 128)):
        for step_x in (1, -1):
            for ss in (0, 1):
                ox, oy = int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1)); cx, cy = int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1))
                o, c = BASE + oy * S + ox, BASE + cy * S + cx
                start = int(rs.randint(0, MH - h + 1)) * MS + int(rs.randint(0, MS - w + 1)) + (w - 1 if step_x < 0 else 0)
                got = eng.sad_mask_block(org.reshape(-1)[o:], S, cur.reshape(-1)[c:], S, w, h, flat, start, MS, step_x, -w * step_x, ss)
                d = _cand(L.MASK_CAND_DT, w, h, ox, oy, cx, cy, ss)
                d['mask_offset'] = start; d['mask_stride'] = MS; d['step_x'] = step_x; d['mask_stride2'] = -w * step_x
                lst = int(eng.sad_mask_batch(d)[0])          # after the helper: its call leaves the uploaded table as it was
                exp = O.orc_sad_mask(PO(org, o), S, PO(cur, c), S, w, h, PO(flat, start), MS, step_x, -w * step_x, ss)
                assert got == lst == exp, (w, h, step_x, ss, got, lst, exp)


def test_sad_x5_block_equals_list_form_and_oracle(eng):
    import vvenc_b200._lib as L
    O = oracle()
    rs, org, cur = _pictures(13)
    _upload(eng, org, cur)
    for w in (8, 16):
        for h in (2, 8, 16, 64, 128):
            for ss in (0, 1):
                ox, oy = int(rs.randint(0, W - w - 4 + 1)), int(rs.randint(0, H - h + 1)); cx, cy = int(rs.randint(4, W - w + 1)), int(rs.randint(0, H - h + 1))
                o, c = BASE + oy * S + ox, BASE + cy * S + cx
                lst = eng.sad_x5_batch(_cand(L.CAND_DT, w, h, ox, oy, cx, cy, ss))[0]
                for cc in (0, 1):
                    got = eng.sad_x5_block(org.reshape(-1), o, S, cur.reshape(-1), c, S, w, h, ss, bool(cc))
                    exp = np.zeros(5, dtype=np.uint64)
                    O.orc_sad_x5(PO(org, o), S, PO(cur, c), S, w, h, ss, cc, P(exp))
                    assert np.array_equal(got, exp), (w, h, ss, cc, got, exp)
                    want = lst.copy()
                    if not cc:
                        want[2] = 0                           # the centre stays as the caller had it
                    assert np.array_equal(got, want), (w, h, ss, cc, got, lst)


def test_dist_block_equals_list_form_and_oracle(eng):
    import vvenc_b200 as V
    import vvenc_b200._lib as L
    O = oracle()
    rs, org, cur = _pictures(14)
    _upload(eng, org, cur)
    for dfunc in (V.DF_SSE, V.DF_SAD, V.DF_HAD, V.DF_HAD_FAST, V.DF_HAD_2SAD):
        for (w, h) in ((8, 8), (16, 16), (64, 64), (4, 16), (32, 8)):
            ox, oy = int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1)); cx, cy = int(rs.randint(0, W - w + 1)), int(rs.randint(0, H - h + 1))
            o, c = BASE + oy * S + ox, BASE + cy * S + cx
            got = eng.dist_block(dfunc, org.reshape(-1)[o:], S, cur.reshape(-1)[c:], S, w, h)
            d = _cand(L.CAND_DT, w, h, ox, oy, cx, cy); d['dfunc'] = dfunc
            assert got == int(eng.dist_batch(d)[0]) == O.orc_dist(dfunc, PO(org, o), S, PO(cur, c), S, w, h, 0), (dfunc, w, h)


# ---------------------------------------------------------------------------------------------------- affine
@pytest.mark.parametrize("w,h", [(4, 4), (8, 4), (4, 16), (16, 16), (32, 8), (64, 64), (128, 128)])
def test_affine_helpers_equal_eq_batch_and_oracle(eng, w, h):
    O = oracle()
    rs = np.random.RandomState(w * 1000 + h)
    ps, rstr, ds = w + 5, w + 3, w + 7
    pred = rs.randint(0, 1024, size=(h, ps)).astype(np.int16)
    resi = rs.randint(-300, 301, size=(h, rstr)).astype(np.int16)
    eqb, bx, by = eng.affine_eq_batch(0, np.ascontiguousarray(pred[:, :w])[None], np.ascontiguousarray(resi[:, :w])[None], want_derivs=True)
    eqb6 = eng.affine_eq_batch(1, np.ascontiguousarray(pred[:, :w])[None], np.ascontiguousarray(resi[:, :w])[None])
    gx = eng.affine_sobel(0, pred, ps, ds, w, h); gy = eng.affine_sobel(1, pred, ps, ds, w, h)
    for vert, g, b in ((0, gx, bx[0]), (1, gy, by[0])):
        e = np.zeros((h, ds), dtype=np.int16)
        O.orc_sobel(vert, P(pred), ps, P(e), ds, w, h)
        assert np.array_equal(g[:, :w], b) and np.array_equal(g[:, :w], e[:, :w]), (w, h, vert)
        assert not g[:, w:].any()                               # samples right of the block stay untouched
    for six, batch in ((0, eqb[0]), (1, eqb6[0])):
        e = np.zeros(49, dtype=np.int64)
        O.orc_equal_coeff(six, P(resi), rstr, P(gx), P(gy), ds, w, h, P(e))
        assert np.array_equal(batch.reshape(-1), e), (w, h, six)
        start = rs.randint(-1 << 40, 1 << 40, size=49).astype(np.int64)
        acc = start.copy()
        for _ in range(2):
            eng.affine_equal_coeff(six, resi, rstr, gx, gy, ds, w, h, acc)
        assert np.array_equal(acc, start + 2 * e), (w, h, six)


# ---------------------------------------------------------------------------------------------------- asynchronous mode
def test_helpers_block_in_async_mode(eng):
    """vvb_set_async(1) and page-locked buffers: every helper returns with its results in place, without vvb_synchronize"""
    import torch
    O = oracle()
    lib, hnd = eng.lib, eng.h
    rs, org, cur = _pictures(15)
    w, h = 16, 16

    def pinned(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        return t, t.data_ptr()

    o, po = pinned(org[M:M + h + 4, M:M + w + 8]); c, pc = pinned(cur[M:M + h, M:M + w + 8])
    so, sc = w + 8, w + 8
    on, cn = o.numpy(), c.numpy()
    msk = rs.randint(0, 9, size=(h, w)).astype(np.int16)
    m, pm = pinned(msk)
    d5, p5 = pinned(np.full(5, 7, dtype=np.int64))
    dv, pdv = pinned(np.full((h, w + 2), -1, dtype=np.int16))
    eq, peq = pinned(np.zeros(49, dtype=np.int64))
    err = ctypes.c_int(-1)
    eng.set_async(True)
    try:
        v = lib.vvb_dist_block(hnd, 1, po, so, pc, sc, w, h, 10, 0, ctypes.byref(err))
        assert err.value == 0 and v == O.orc_dist(1, P(on), so, P(cn), sc, w, h, 0)
        v = lib.vvb_sad_mask_block(hnd, po, so, pc, sc, w, h, pm, w, 1, -w, 0, ctypes.byref(err))
        assert err.value == 0 and v == O.orc_sad_mask(P(on), so, P(cn), sc, w, h, P(msk), w, 1, -w, 0)
        v = lib.vvb_fix_wsse_block(hnd, po, so, pc, sc, w, h, 40000, ctypes.byref(err))
        assert err.value == 0 and v == O.orc_fix_wsse(P(on), so, P(cn), sc, w, h, 40000)
        assert lib.vvb_sad_x5_block(hnd, po, so, pc + 8, sc, w, h, 1, 1, p5) == 0
        e5 = np.zeros(5, dtype=np.uint64); O.orc_sad_x5(P(on), so, PO(cn, 4), sc, w, h, 1, 1, P(e5))
        assert np.array_equal(d5.numpy(), e5.astype(np.int64))
        assert lib.vvb_affine_sobel(hnd, 0, po, so, pdv, w + 2, w, h) == 0
        ex = np.zeros((h, w + 2), dtype=np.int16); O.orc_sobel(0, P(on), so, P(ex), w + 2, w, h)
        assert np.array_equal(dv.numpy()[:, :w], ex[:, :w])
        gx = np.ascontiguousarray(dv.numpy())
        assert lib.vvb_affine_equal_coeff(hnd, 1, pc, sc, pdv, pdv, w + 2, w, h, peq) == 0
        ee = np.zeros(49, dtype=np.int64); O.orc_equal_coeff(1, P(cn), sc, P(gx), P(gx), w + 2, w, h, P(ee))
        assert np.array_equal(eq.numpy(), ee)
    finally:
        eng.set_async(False)


# ---------------------------------------------------------------------------------------------------- which kernels run
def kernel_selection_cases():
    """[(label, setup)] for tests/_kernel_selection_run.py: each distortion helper launches the kernel of its descriptor-list form and no other kernel"""
    import vvenc_b200 as V
    rs = np.random.RandomState(16)
    o = rs.randint(0, 1024, size=(24, 40)).astype(np.int16); c = rs.randint(0, 1024, size=(24, 40)).astype(np.int16)
    msk = rs.randint(0, 9, size=(16, 16)).astype(np.int16)
    calls = (('dist_block', 'dist_list_kernel', lambda e: e.dist_block(V.DF_HAD, o, 40, c, 40, 16, 16)),
             ('sad_mask_block', 'sad_mask_batch_kernel', lambda e: e.sad_mask_block(o, 40, c, 40, 16, 16, msk, 0, 16, 1, -16)),
             ('sad_x5_block', 'sad_x5_batch_kernel', lambda e: e.sad_x5_block(o, 0, 40, c, 4, 40, 16, 16)),
             ('fix_wsse_block', 'fix_wsse_batch_kernel', lambda e: e.fix_wsse_block(o, 40, c, 40, 16, 16, 40000)))
    cases = []
    for name, kernel, call in calls:
        def setup(eng, kernel=kernel, call=call):
            return (lambda: call(eng)), (lambda names: len(names) == 1 and re.search(r'\b%s\b' % kernel, names[0]) is not None)
        cases.append(('%s: %s only' % (name, kernel), setup))
    return cases


def test_kernel_selection():
    import json, subprocess, sys
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_kernel_selection_run.py')
    out = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [script, 'test_gpu_single_call'], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]
    assert [r['case'] for r in rows] == [label for label, _ in kernel_selection_cases()]
    assert [r for r in rows if not r['ok']] == [], rows
