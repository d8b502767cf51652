#!/usr/bin/env python3
"""Times the TU round trip with the slice's quantiser on the device: vvb_tu_roundtrip_rdo_dev (one call) against the three-call chain it replaces
(vvb_fwd_trquant_dev -> vvb_rdoq_dev / vvb_dep_quant_dev -> vvb_inv_trquant_dev, plus the reconstruction and SSE the caller then does, here one torch expression)
on the same resident inputs, per shape and quantiser.  CUDA events on the context stream, after a warm-up of every shape; the outputs of the two are compared bit
for bit (levels, and the reconstruction against the chain's clip(pred + residual)).  Beside it, where oracle/_ref exists, the reference's own AVX2 members composed
the same way (tests/tu_rdo_cases.py) in one process per usable host thread, over a small sample: one probe call per member and TU, so the per-TU rig set-up and the
Python glue are in that number.  Prints the card name and power limit of the run, then one JSON line.
usage: python tools/tu_rdo_bench.py [reps] [TUs per launch, default 2160p's worth]"""
import ctypes, json, multiprocessing, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))

SHAPES = ((8, 8), (16, 16), (32, 32), (64, 64), (4, 16), (32, 8))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # the number is still the device's; say that the card could not be read
        return 'unknown (%s)' % e


def usable_threads():
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count() or 1


def _ref_chunk(work):
    """the reference's members on a list of (row, org, pred), in a worker process of its own"""
    import tu_rdo_cases as T
    for row, org, pred in work:
        T.ref_roundtrip_rdo(row, org, pred, b'AVX2')
    return len(work)


def main():
    import torch
    import vvenc_b200 as V
    from _libs import have_ref
    assert torch.cuda.is_available(), 'needs cuda:0'
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    tus = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    print('card:', card(), flush=True)
    eng = V.CostEngine(0)
    ext = torch.cuda.ExternalStream(eng.stream, device=torch.device('cuda', 0))
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'golden_v8_tu_rdo.npz'))
    lam = 57.3
    cp = lambda t: ctypes.c_void_p(t.data_ptr())
    out = {'card': card(), 'reps': reps, 'rows': []}
    threads, pool = usable_threads(), None
    for quantiser in (1, 2):
        rates_flat = np.ascontiguousarray(g['rates_%d' % [i for i, r in enumerate(g['cases']) if int(r[0]) == quantiser and int(r[7]) == 0][0]])
        for (w, h) in SHAPES:
            n = tus or (3840 // w) * (2160 // h)
            rs = np.random.RandomState(w * 100 + h + quantiser)
            pred = rs.randint(0, 1024, size=(n, h, w))
            amp = np.array([2, 6, 30, 150])[rs.randint(4, size=n)][:, None, None]
            org = np.clip(pred + np.round((rs.rand(n, h, w) * 2 - 1) * amp), 0, 1023).astype(np.int16); pred = pred.astype(np.int16)
            par = eng.tu_par(w, h, 0, 0, 10, 32, dep_quant=quantiser == 2)
            tq, keep = eng._tu_quant(quantiser, rates_flat, lam, 8, False, 8, False, False, True)
            d_org = torch.from_numpy(org).cuda(); d_pred = torch.from_numpy(pred).cuda()
            d_q = torch.zeros((n, h, w), dtype=torch.int16, device='cuda'); d_reco = torch.zeros_like(d_q)
            d_res = torch.zeros(n * 32, dtype=torch.uint8, device='cuda'); d_nr = torch.zeros(n, dtype=torch.uint8, device='cuda')
            # the chain's buffers
            d_resi = (d_org.int() - d_pred.int()).short()
            d_coef = torch.zeros((n, h, w), dtype=torch.int32, device='cuda'); d_q2 = torch.zeros_like(d_q); d_r2 = torch.zeros_like(d_q)
            d_sum = torch.zeros(n, dtype=torch.int32, device='cuda'); d_last = torch.zeros_like(d_sum); d_nr2 = torch.zeros_like(d_nr)
            rq = V._lib.vvb_rdoq_par(lam, 8, 0); dq = V._lib.vvb_dq_par(lam, 8, 0, 0, 0)
            r_rq = eng.rdoq_rates(rates_flat) if quantiser == 1 else None; r_dq = eng.dq_rates(rates_flat) if quantiser == 2 else None

            def one():
                eng._chk(eng.lib.vvb_tu_roundtrip_rdo_dev(eng.h, ctypes.byref(par), ctypes.byref(tq), cp(d_org), cp(d_pred), n, cp(d_q), cp(d_reco), cp(d_res), cp(d_nr)))

            def three():
                # the residual is formed by the caller before the chain as well; it is not timed on either side
                eng._chk(eng.lib.vvb_fwd_trquant_dev(eng.h, ctypes.byref(par), cp(d_resi), n, cp(d_coef), cp(d_q2), None, None, cp(d_nr2)))
                if quantiser == 1:
                    eng._chk(eng.lib.vvb_rdoq_dev(eng.h, ctypes.byref(par), ctypes.byref(rq), ctypes.byref(r_rq), cp(d_coef), cp(d_nr2), n, cp(d_q2), cp(d_sum), cp(d_last)))
                else:
                    eng._chk(eng.lib.vvb_dep_quant_dev(eng.h, ctypes.byref(par), ctypes.byref(dq), ctypes.byref(r_dq), cp(d_coef), cp(d_nr2), n, cp(d_q2), cp(d_sum), cp(d_last)))
                eng._chk(eng.lib.vvb_inv_trquant_dev(eng.h, ctypes.byref(par), cp(d_q2), n, cp(d_r2)))
                with torch.cuda.stream(ext):                       # what the caller then does: zero residual where abs_sum is 0, reconstruct, three SSEs
                    r = torch.where((d_sum > 0)[:, None, None], d_r2.int(), 0)
                    reco = (d_pred.int() + r).clamp(0, 1023)
                    e = (d_org.int() - reco).long(); z = (d_org.int() - d_pred.int()).long(); x = z - r.long()
                    return reco, (e * e).sum((1, 2)), (x * x).sum((1, 2)), (z * z).sum((1, 2))

            def timed(fn):
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(ext):
                    e0.record(ext)
                    for _ in range(reps):
                        fn()
                    e1.record(ext)
                eng.synchronize(); torch.cuda.synchronize()
                return e0.elapsed_time(e1) / reps

            for _ in range(3):
                one(); three()
            eng.synchronize(); torch.cuda.synchronize()
            t1, t3, t1b, t3b = timed(one), timed(three), timed(one), timed(three)       # alternated, twice
            one(); reco3, dr, dd, dz = three(); eng.synchronize(); torch.cuda.synchronize()
            res = np.frombuffer(d_res.cpu().numpy().tobytes(), dtype=V.TU_RESULT_DT)
            equal = bool(torch.equal(d_q, d_q2) and torch.equal(d_reco.int(), reco3) and torch.equal(d_nr, d_nr2)
                         and np.array_equal(res['abs_sum'], d_sum.cpu().numpy()) and np.array_equal(res['last_pos'], d_last.cpu().numpy())
                         and np.array_equal(res['dist_reco'].astype(np.int64), dr.cpu().numpy()) and np.array_equal(res['dist_resi'].astype(np.int64), dd.cpu().numpy())
                         and np.array_equal(res['dist_zero'].astype(np.int64), dz.cpu().numpy()))
            row = {'quantiser': {1: 'fast RDOQ', 2: 'DepQuant'}[quantiser], 'shape': '%dx%d' % (w, h), 'tus': n,
                   'one_call_ms': round(min(t1, t1b), 4), 'three_calls_ms': round(min(t3, t3b), 4), 'one_over_three': round(min(t1, t1b) / min(t3, t3b), 3),
                   'one_call_Mtus_s': round(n / min(t1, t1b) / 1e3, 2), 'bit_exact': equal, 'nonzero_tus': int((res['abs_sum'] > 0).sum())}
            if have_ref():
                # the members are called one TU at a time through the probe's ctypes entry points (rig set-up and the Python glue between the calls
                # included), so this is an upper bound of what the reference's own code needs; a small sample, extrapolated to the launch.  One process
                # per host thread: the probe keeps process-wide state (the SIMD selection among it), so it is not driven from several threads of one process
                if pool is None:
                    pool = multiprocessing.get_context('spawn').Pool(threads)
                    pool.map(_ref_chunk, [[]] * threads)                 # start-up (interpreter, probe load) outside the timed window
                m = min(n, 8 * threads)
                rows = [[quantiser, w, h, 0, 0, 0, 0, 0, 10, 32, 0, 0, 1, int(lam * 1000), 0, 0, 0]] * m
                work = [(rows[i], org[i], pred[i]) for i in range(m)]
                t0 = time.perf_counter()
                pool.map(_ref_chunk, [work[k::threads] for k in range(threads)])
                row['reference_avx2_members_ms_per_launch_%d_processes' % threads] = round((time.perf_counter() - t0) / m * n * 1e3, 1)
            out['rows'].append(row)
            print(json.dumps(row), flush=True)
            del d_org, d_pred, d_q, d_reco, d_res, d_nr, d_resi, d_coef, d_q2, d_r2, d_sum, d_last, d_nr2
            torch.cuda.empty_cache()
    slower = [r['quantiser'] + ' ' + r['shape'] for r in out['rows'] if r['one_over_three'] > 1.0]
    out['slower_in_one_call'] = slower
    if pool is not None:
        pool.close(); pool.join()
    eng.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
