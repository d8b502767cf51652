#!/usr/bin/env python3
"""Component timing of the TU kernels on pools larger than L2: forward (tensor engine on / off), inverse, fused round trip.
usage: python tools/tu_bench.py [noise_amp [WxH ...]]   (GPU box)"""
import ctypes, sys, os
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vvenc_b200 as V

amp = int(sys.argv[1]) if len(sys.argv) > 1 else 200
eng = V.CostEngine(0); lib = eng.lib
P_ = ctypes.c_void_p
ext = torch.cuda.ExternalStream(eng.stream)


def chk(rc):
    if rc: raise RuntimeError(lib.vvb_last_error(eng.h).decode())


def tl(fn, reps=3):
    fn(); eng.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(ext):
        e0.record(ext)
        for _ in range(reps): fn()
        e1.record(ext)
    eng.synchronize(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


shapes = [(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (32, 8), (64, 16)]
if len(sys.argv) > 2:
    shapes = [tuple(int(v) for v in a.split('x')) for a in sys.argv[2:]]
for (w, h) in shapes:
    ntu = (256 << 20) // (8 * w * h)
    par = eng.tu_par(w, h, 0, 0, 10, 32, False, False)
    d_o = torch.randint(0, 1024, (ntu * w * h,), dtype=torch.int16, device='cuda')
    d_p = (d_o + torch.randint(-amp, amp + 1, (ntu * w * h,), dtype=torch.int16, device='cuda')).clamp_(0, 1023)
    d_r = d_o - d_p
    d_q = torch.empty_like(d_o); d_rc = torch.empty_like(d_o); d_rs = torch.empty(ntu * 32, dtype=torch.uint8, device='cuda')
    d_sum = torch.empty(ntu, dtype=torch.int32, device='cuda'); d_last = torch.empty_like(d_sum); d_nr = torch.empty(ntu, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    res = {}
    for (name, tens) in (('fwd_tensor', 1), ('fwd_cudacore', 0)):
        eng.set_tensor_transform(tens)
        res[name] = tl(lambda: chk(lib.vvb_fwd_trquant_dev(eng.h, ctypes.byref(par), P_(d_r.data_ptr()), ntu, None, P_(d_q.data_ptr()), P_(d_sum.data_ptr()),
                                                        P_(d_last.data_ptr()), P_(d_nr.data_ptr()))))
    eng.set_tensor_transform(1)
    res['inv'] = tl(lambda: chk(lib.vvb_inv_trquant_dev(eng.h, ctypes.byref(par), P_(d_q.data_ptr()), ntu, P_(d_rc.data_ptr()))))
    res['roundtrip'] = tl(lambda: chk(lib.vvb_tu_roundtrip_dev(eng.h, ctypes.byref(par), P_(d_o.data_ptr()), P_(d_p.data_ptr()), ntu, P_(d_q.data_ptr()), P_(d_rc.data_ptr()),
                                                               P_(d_rs.data_ptr()), None)))
    nz = int((d_sum > 0).sum())
    gb = {'fwd': ntu * (4 * w * h + 9), 'inv': ntu * 4 * w * h, 'roundtrip': ntu * (8 * w * h + 32)}
    print('%2dx%-2d ntu %8d nz %5.1f%% |' % (w, h, ntu, 100.0 * nz / ntu), ' '.join('%s %.3f ms (%4.0f GB/s)' % (k, v, gb[k.split('_')[0]] / v / 1e6) for k, v in res.items()), flush=True)
    del d_o, d_p, d_r, d_q, d_rc, d_rs
eng.close()
