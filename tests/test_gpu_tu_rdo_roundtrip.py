"""vvb_tu_roundtrip_rdo* on the GPU: the TU candidate round trip with fast RDOQ or dependent quantisation between the forward and the inverse transform.
Every result is compared bit for bit: with the golden vectors of the reference, with the same chain made of the separate device calls (vvb_fwd_trquant ->
vvb_rdoq / vvb_dep_quant -> vvb_inv_trquant, reconstruction and SSE in numpy) and with the CPU oracle composition (tests/tu_rdo_cases.py).  The oracle's
quantisers are the library's own restatements (rdoq_core.h, depquant_core.h) compiled for the CPU, so for the levels that leg checks the device build and the
chaining, not the algorithm; the golden rows, taken from the reference's members, are what pins the quantisers themselves."""
import ctypes, os
import numpy as np
import pytest
import tu_rdo_cases as T

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v8_tu_rdo.npz')


@pytest.fixture(scope='module')
def golden_v8():
    return np.load(GOLDEN)


@pytest.fixture(scope='module')
def eng():
    import vvenc_b200 as V
    e = V.CostEngine(0)
    yield e
    e.close()


def rates_for(g, quantiser, comp, k=0):
    """rate tables the reference read for a golden row of this quantiser and component (the k-th such row)"""
    idx = [i for i, r in enumerate(g['cases']) if int(r[0]) == quantiser and int(r[7]) == comp]
    return np.ascontiguousarray(g['rates_%d' % idx[k % len(idx)]])


def par_of(eng, c, lfnst_st=(0, 0)):
    return eng.tu_par(c['w'], c['h'], c['th'], c['tv'], c['bd'], c['qp'], bool(c['irap']), c['quantiser'] == 2, bool(c['sh']), c['lfnst'], lfnst_st[0], bool(lfnst_st[1]),
                      False, 0, bool(c['comp']))


def call(eng, c, org, pred, rates, **kw):
    return eng.tu_roundtrip_rdo(par_of(eng, c, kw.pop('lfnst_st', (0, 0))), org, pred, c['quantiser'], rates, c['lam1000'] / 1000.0, zero_out=T.zero_out(c),
                                selective=bool(c['sel']), **kw)


def chain(eng, c, org, pred, rates, lfnst_st=(0, 0)):
    """the same TUs through the separate device calls, reconstruction and SSE in numpy"""
    par = par_of(eng, c, lfnst_st)
    lam = c['lam1000'] / 1000.0
    resi = (org.astype(np.int32) - pred.astype(np.int32)).astype(np.int16)
    f = eng.fwd_trquant(par, resi)
    nr = f['need_rdoq'] if c['sel'] else None
    if c['quantiser'] == 2:
        r = eng.dep_quant(par, eng.dq_rates(rates), f['coef'], lam, zero_out=T.zero_out(c), need_rdoq=nr)
    else:
        r = eng.rdoq(par, eng.rdoq_rates(rates), f['coef'], lam, need_rdoq=nr)
    rec = eng.inv_trquant(par, r['q']).astype(np.int32)
    rec[r['abs_sum'] == 0] = 0
    reco = np.clip(pred.astype(np.int32) + rec, 0, (1 << c['bd']) - 1).astype(np.int16)
    d = resi.astype(np.int64)
    sse = lambda x: (x.astype(np.int64) ** 2).reshape(len(x), -1).sum(1)
    res = np.stack([sse(org.astype(np.int64) - reco), sse(d - rec), sse(d), r['abs_sum'], r['last_pos']], 1)
    return r['q'], reco, res, f['need_rdoq']


def res_rows(res):
    return np.stack([res['dist_reco'].astype(np.int64), res['dist_resi'].astype(np.int64), res['dist_zero'].astype(np.int64), res['abs_sum'], res['last_pos']], 1)


def same(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))


def batch_inputs(c, n, seed):
    """n TUs of one shape with residual amplitudes from flat to full scale, so that both branches and both need_rdoq outcomes occur"""
    rs = np.random.RandomState(seed)
    mx = (1 << c['bd']) - 1
    pred = rs.randint(0, mx + 1, size=(n, c['h'], c['w']))
    amp = np.array([0, 2, 6, 30, 150, mx])[rs.randint(6, size=n)][:, None, None]
    org = np.clip(pred + np.round((rs.rand(n, c['h'], c['w']) * 2 - 1) * amp), 0, mx)
    return org.astype(np.int16), pred.astype(np.int16)


def case(quantiser, w, h, comp, bd, qp=32, sel=1, sh=0, th=0, tv=0, lfnst=0, lam=57.3, irap=0):
    return dict(quantiser=quantiser, w=w, h=h, th=th, tv=tv, lfnst=lfnst, mode=0, comp=comp, bd=bd, qp=qp, irap=irap, sh=sh, sel=sel, lam1000=int(lam * 1000),
                amp=0, init_id=0, seed=0)


def test_golden_v8(eng, golden_v8):
    bad = []
    for i, row in enumerate(golden_v8['cases']):
        c = T.row_dict(row)
        org, pred = T.inputs(row)
        assert T.inputs_crc(org[0], pred[0]) == int(golden_v8['inputs_crc'][i]), i
        st = tuple(int(v) for v in golden_v8['lfnst'][i])
        r = call(eng, c, org, pred, golden_v8['rates_%d' % i], lfnst_st=st)
        m = [int(v) for v in golden_v8['meta'][i]]
        ok = (np.array_equal(r['q'][0], golden_v8['q_%d' % i]) and np.array_equal(r['reco'][0], pred[0] + golden_v8['dreco_%d' % i])
              and res_rows(r['res'])[0].tolist() == m[:5] and int(r['need_rdoq'][0]) == m[5])
        if not ok:
            bad.append((i, c))
    assert bad == [], (len(bad), bad[:3])


@pytest.mark.parametrize('quantiser', [1, 2])
def test_every_shape_against_chain_and_oracle(eng, golden_v8, quantiser):
    seen = {'inv': 0, 'zero': 0, 'need0': 0, 'need1': 0}
    bad = []
    k = 0
    for (w, h) in T.SHAPES:
        for comp in (0, 1):
            for bd in (8, 10):
                k += 1
                c = case(quantiser, w, h, comp, bd, qp=[22, 27, 32, 37][k % 4], sel=k % 3 != 0, sh=int(quantiser == 1 and k % 2), lam=[11.7, 57.3, 120.0][k % 3])
                rates = rates_for(golden_v8, quantiser, comp, k)
                n = 37 + (k % 5) * 26                          # never a multiple of the TUs per CTA
                org, pred = batch_inputs(c, n, 100 * k + quantiser)
                r = call(eng, c, org, pred, rates)
                q, reco, res, need = chain(eng, c, org, pred, rates)
                if not same((r['q'], r['reco'], res_rows(r['res']), r['need_rdoq']), (q, reco, res, need)):
                    bad.append(('chain', c))
                for i in (0, n // 2, n - 1):
                    oq, oreco, om, oneed = T.oracle_roundtrip_rdo([c[k2] for k2 in T.COLS], org[i], pred[i], rates)
                    if not same((r['q'][i], r['reco'][i], res_rows(r['res'])[i], [int(r['need_rdoq'][i])]), (oq, oreco, om, [oneed])):
                        bad.append(('oracle', c, i))
                seen['inv'] += int((r['res']['abs_sum'] > 0).sum()); seen['zero'] += int((r['res']['abs_sum'] == 0).sum())
                seen['need0'] += int((r['need_rdoq'] == 0).sum()); seen['need1'] += int((r['need_rdoq'] == 1).sum())
    assert bad == [], (len(bad), bad[:3])
    assert all(v > 0 for v in seen.values()), seen


def test_lfnst_and_mts(eng, golden_v8):
    bad = []
    for quantiser in (1, 2):
        for (w, h, th, tv, lf, st) in ((4, 4, 0, 0, 1, (0, 0)), (8, 8, 0, 0, 2, (3, 1)), (16, 16, 0, 0, 1, (2, 1)), (16, 16, 2, 2, 0, (0, 0)), (32, 8, 1, 2, 0, (0, 0)),
                                       (4, 32, 2, 1, 0, (0, 0)), (32, 32, 1, 1, 0, (0, 0))):
            c = case(quantiser, w, h, 0, 10, qp=27, th=th, tv=tv, lfnst=lf)
            rates = rates_for(golden_v8, quantiser, 0, w + lf)
            org, pred = batch_inputs(c, 45, 7 * w + lf)
            r = call(eng, c, org, pred, rates, lfnst_st=st)
            if not same((r['q'], r['reco'], res_rows(r['res']), r['need_rdoq']), chain(eng, c, org, pred, rates, st)):
                bad.append(('chain', c))
            for i in (0, 44):
                oq, oreco, om, oneed = T.oracle_roundtrip_rdo([c[k] for k in T.COLS], org[i], pred[i], rates, st)
                if not same((r['q'][i], r['reco'][i], res_rows(r['res'])[i]), (oq, oreco, om)):
                    bad.append(('oracle', c, i))
    assert bad == [], bad[:3]


class DevBufs:
    """device buffers of a _dev call, each `off` bytes into its allocation"""

    def __init__(self, n, w, h, off):
        import torch
        self.off = off; self.n = n; self.area = w * h
        self.t = {k: torch.zeros(b + 64, dtype=torch.uint8, device='cuda') for k, b in
                  (('org', n * w * h * 2), ('pred', n * w * h * 2), ('q', n * w * h * 2), ('reco', n * w * h * 2), ('res', n * 32), ('nr', n))}

    def ptr(self, k):
        return self.t[k].data_ptr() + self.off

    def put(self, k, a):
        import torch
        b = np.frombuffer(np.ascontiguousarray(a).tobytes(), dtype=np.uint8)
        self.t[k][self.off:self.off + len(b)] = torch.from_numpy(b.copy()).cuda()

    def get(self, k, dtype, shape):
        b = self.t[k][self.off:self.off + int(np.prod(shape)) * np.dtype(dtype).itemsize].cpu().numpy()
        return np.frombuffer(b.tobytes(), dtype=dtype).reshape(shape)


def dev_call(eng, c, org, pred, rates, off):
    import vvenc_b200 as V
    n = len(org)
    B = DevBufs(n, c['w'], c['h'], off)
    B.put('org', org); B.put('pred', pred)
    tq, keep = eng._tu_quant(c['quantiser'], rates, c['lam1000'] / 1000.0, 8, False, 8, T.zero_out(c), False, bool(c['sel']))
    eng._chk(eng.lib.vvb_tu_roundtrip_rdo_dev(eng.h, ctypes.byref(par_of(eng, c)), ctypes.byref(tq), B.ptr('org'), B.ptr('pred'), n, B.ptr('q'), B.ptr('reco'),
                                              B.ptr('res'), B.ptr('nr')))
    eng.synchronize()
    return (B.get('q', np.int16, org.shape), B.get('reco', np.int16, org.shape), res_rows(B.get('res', V.TU_RESULT_DT, (n,))), B.get('nr', np.uint8, (n,)))


def test_tensor_engines_and_alignment(eng, golden_v8):
    bad = []
    for quantiser in (1, 2):
        for (w, h) in ((8, 8), (16, 16), (32, 32), (64, 64), (4, 4), (16, 4)):
            c = case(quantiser, w, h, 0, 10, qp=27, sel=1)
            rates = rates_for(golden_v8, quantiser, 0, w)
            org, pred = batch_inputs(c, 29, 3 * w + h)
            outs = []
            for tensor in (1, 0):
                eng.set_tensor_transform(tensor)
                for off in (0, 8):
                    outs.append(dev_call(eng, c, org, pred, rates, off))
            eng.set_tensor_transform(1)
            if not all(same(o, outs[0]) for o in outs[1:]) or not same(outs[0], chain(eng, c, org, pred, rates)):
                bad.append(c)
    assert bad == [], bad


def test_engines_agree(eng, golden_v8):
    bad = []
    for quantiser, engines, setter in ((1, (1, 2), 'set_rdoq_engine'), (2, (1, 0), 'set_depquant_engine')):
        for (w, h) in ((4, 4), (16, 16), (64, 64), (32, 8)):
            c = case(quantiser, w, h, (w // 4) & 1, 8, qp=32, sel=0)
            rates = rates_for(golden_v8, quantiser, c['comp'], h)
            org, pred = batch_inputs(c, 41, w * h)
            outs = []
            for e in engines:
                getattr(eng, setter)(e)
                r = call(eng, c, org, pred, rates)
                outs.append((r['q'], r['reco'], res_rows(r['res']), r['need_rdoq']))
            getattr(eng, setter)(engines[0])
            if not same(outs[0], outs[1]):
                bad.append(c)
    assert bad == [], bad


def test_planes_against_pools(eng, golden_v8):
    import vvenc_b200 as V
    W, H, m = 192, 128, 16
    S = W + 2 * m
    bad = []
    for quantiser in (1, 2):
        rs = np.random.RandomState(40 + quantiser)
        orgp = rs.randint(0, 1024, size=(H + 2 * m, S)).astype(np.int16)
        prdp = np.clip(orgp + rs.randint(-60, 61, size=orgp.shape), 0, 1023).astype(np.int16)
        eng.upload_plane(20, orgp, W, H, m, 10); eng.upload_plane(21, prdp, W, H, m, 10)
        for (w, h) in ((8, 8), (16, 16), (32, 32), (4, 8), (16, 4)):
            c = case(quantiser, w, h, 0, 10, qp=27, sel=1)
            rates = rates_for(golden_v8, quantiser, 0, w)
            xs, ys = np.meshgrid(np.arange(0, W - w + 1, w), np.arange(0, H - h + 1, h))
            blk = np.zeros(xs.size, dtype=V.BLOCK_DT)
            blk['x'] = xs.ravel(); blk['y'] = ys.ravel()
            blk['start_x'] = rs.randint(-7, 8, size=xs.size) | 1; blk['start_y'] = rs.randint(-7, 8, size=xs.size) | 1   # odd displacements
            r = eng.tu_roundtrip_rdo_planes(par_of(eng, c), 20, 21, blk, quantiser, rates, c['lam1000'] / 1000.0, selective=True)
            org = np.stack([orgp[m + b['y']:m + b['y'] + h, m + b['x']:m + b['x'] + w] for b in blk])
            pred = np.stack([prdp[m + b['y'] + b['start_y']:m + b['y'] + b['start_y'] + h, m + b['x'] + b['start_x']:m + b['x'] + b['start_x'] + w] for b in blk])
            p = call(eng, c, org, pred, rates)
            if not same((r['q'], r['reco'], res_rows(r['res']), r['need_rdoq']), (p['q'], p['reco'], res_rows(p['res']), p['need_rdoq'])):
                bad.append(c)
    assert bad == [], bad


def test_extremes(eng, golden_v8):
    bad = []
    for quantiser in (1, 2):
        for (w, h, bd) in ((4, 4, 8), (16, 16, 10), (32, 32, 8), (64, 64, 10), (64, 16, 10)):
            for qp in (17, 51):
                c = case(quantiser, w, h, 0, bd, qp=qp, sel=1, lam=30.0)
                rates = rates_for(golden_v8, quantiser, 0, qp)
                mx = (1 << bd) - 1
                rs = np.random.RandomState(w + h + qp)
                sign = rs.rand(6, 1, 1) < 0.5
                org = np.where(sign, mx, 0) * np.ones((6, h, w)); pred = mx - org          # full-scale residuals of both signs
                org[4:] = np.where(rs.rand(2, h, w) < 0.5, 0, mx); pred[4:] = mx - org[4:]
                org = org.astype(np.int16); pred = pred.astype(np.int16)
                r = call(eng, c, org, pred, rates)
                if not same((r['q'], r['reco'], res_rows(r['res']), r['need_rdoq']), chain(eng, c, org, pred, rates)):
                    bad.append(('chain', c))
                for i in (0, 5):
                    oq, oreco, om, oneed = T.oracle_roundtrip_rdo([c[k] for k in T.COLS], org[i], pred[i], rates)
                    if not same((r['q'][i], r['reco'][i], res_rows(r['res'])[i]), (oq, oreco, om)):
                        bad.append(('oracle', c, i))
                if w * h == 4096 and bd == 10:
                    assert int(r['res']['dist_zero'].max()) == 4096 * mx * mx > 2 ** 31     # beyond 32-bit signed sums
    assert bad == [], bad[:3]


def test_rejections(eng, golden_v8):
    import vvenc_b200 as V
    L = V._lib
    org = np.zeros((2, 8, 8), dtype=np.int16); pred = org.copy()
    rq, dq = rates_for(golden_v8, 1, 0), rates_for(golden_v8, 2, 0)

    def code(par, quantiser, rates, lam=57.3, n=None, **kw):
        o = org if n is None else org[:n]
        try:
            eng.tu_roundtrip_rdo(par, o, pred[:len(o)], quantiser, rates, lam, **kw)
            return L.VVB_OK
        except V.VvbError as e:
            return e.code
    p = lambda **kw: eng.tu_par(8, 8, **kw)
    assert code(p(), 1, rq) == L.VVB_OK and code(p(dep_quant=True), 2, dq) == L.VVB_OK
    assert code(p(), 1, rq, n=0) == L.VVB_OK and code(p(dep_quant=True), 2, dq, n=0) == L.VVB_OK
    for quantiser in (0, 3, -1):
        assert code(p(), quantiser, rq) == L.VVB_ERR_ARG
    assert code(p(dep_quant=True), 1, rq) == L.VVB_ERR_ARG and code(p(), 2, dq) == L.VVB_ERR_ARG
    assert code(p(dep_quant=True, sign_hiding=True), 2, dq) == L.VVB_ERR_ARG
    assert code(p(), 1, rq, lam=0.0) == L.VVB_ERR_ARG and code(p(dep_quant=True), 2, dq, lam=-1.0) == L.VVB_ERR_ARG
    assert code(p(), 1, rq, thr_val=0) == L.VVB_ERR_ARG and code(p(), 1, rq, thr_val=65) == L.VVB_ERR_ARG
    assert code(p(transform_skip=True), 1, rq) == L.VVB_ERR_UNSUPPORTED and code(p(transform_skip=True, dep_quant=True), 2, dq) == L.VVB_ERR_UNSUPPORTED
    for bd in (9, 12):
        assert code(p(bit_depth=bd), 1, rq) == L.VVB_ERR_UNSUPPORTED and code(p(bit_depth=bd, dep_quant=True), 2, dq) == L.VVB_ERR_UNSUPPORTED
    # null quantiser parameters: the structure with the other quantiser's half only
    tq, keep = eng._tu_quant(2, dq, 57.3, 8, False, 8, False, False, True)
    tq.quantiser = 1
    res = np.zeros(2, dtype=V.TU_RESULT_DT); q = np.zeros_like(org)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert eng.lib.vvb_tu_roundtrip_rdo(eng.h, ctypes.byref(p()), ctypes.byref(tq), P(org), P(pred), 2, P(q), None, P(res), None) == L.VVB_ERR_ARG
    assert eng.lib.vvb_tu_roundtrip_rdo(eng.h, ctypes.byref(p()), None, P(org), P(pred), 2, P(q), None, P(res), None) == L.VVB_ERR_ARG


def test_large_dq_batch_after_small_one(golden_v8):
    """the work arena grows (and is reallocated) between two calls of one context; the second call must equal a fresh context's"""
    import vvenc_b200 as V
    c = case(2, 32, 32, 0, 10, qp=27, sel=1)
    rates = rates_for(golden_v8, 2, 0, 5)
    small = batch_inputs(c, 3, 1); big = batch_inputs(c, 3001, 2)
    e1 = V.CostEngine(0)
    call(e1, c, *small, rates)
    a = call(e1, c, *big, rates)
    e1.close()
    e2 = V.CostEngine(0)
    b = call(e2, c, *big, rates)
    e2.close()
    assert same((a['q'], a['reco'], res_rows(a['res']), a['need_rdoq']), (b['q'], b['reco'], res_rows(b['res']), b['need_rdoq']))


def kernel_selection_cases():
    """[(label, setup)] for tests/_kernel_selection_run.py: with the tensor engines on, square 8..64 TUs on 16-byte aligned buffers run the raw-byte forward and
    inverse engines, on buffers 8 bytes off (and with the engines off, and for 4 x 4 and rectangular TUs) the CUDA-core kernels; the quantiser kernel of the
    slice and, for dependent quantisation, its dequantiser run between them"""
    from test_gpu_format_limits import ran
    g = np.load(GOLDEN)
    cases = []
    for quantiser in (1, 2):
        for (w, h, tensor, off) in ((16, 16, 1, 0), (64, 64, 1, 0), (16, 16, 1, 8), (32, 32, 0, 0), (4, 4, 1, 0), (8, 32, 1, 0)):
            tc = tensor and off == 0 and w == h and w >= 8

            def setup(eng, quantiser=quantiser, w=w, h=h, tensor=tensor, off=off, tc=tc):
                c = case(quantiser, w, h, 0, 10, qp=27, sel=1)
                rates = rates_for(g, quantiser, 0)
                org, pred = batch_inputs(c, 33, w)
                eng.set_tensor_transform(tensor)
                tc_k, core_k = ['fwd_trquant_tc2_kernel', 'inv_trquant_tc_kernel'], ['fwd_trquant_kernel', 'inv_trquant_kernel']
                want, other = (tc_k, core_k) if tc else (core_k, tc_k)
                want = want + (['rdoq_kernel'] if quantiser == 1 else ['dep_quant_quad_kernel', 'dq_dequant_levels_kernel'])
                return (lambda: dev_call(eng, c, org, pred, rates, off)), \
                    (lambda names: all(ran(names, k) for k in want) and not any(ran(names, k) for k in other + ['tu_roundtrip_kernel']))
            cases.append(('quantiser %d %dx%d tensor %d offset %d: %s engines' % (quantiser, w, h, tensor, off, 'raw-byte' if tc else 'CUDA-core'), setup))
    return cases


def test_kernel_selection():
    import json, subprocess, sys
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_kernel_selection_run.py')
    out = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [script, 'test_gpu_tu_rdo_roundtrip'], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]
    assert [r['case'] for r in rows] == [label for label, _ in kernel_selection_cases()]
    assert [r for r in rows if not r['ok']] == [], rows
