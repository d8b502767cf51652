"""What the motion-search picture benchmarks (tz_bench.py, frac_bench.py, bipred_bench.py) share: the card they run on, their seeded 3840x2160 10-bit
pictures and CUDA-event timing."""
import subprocess

import numpy as np

PW, PH = 3840, 2160


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in q.split(',')]
        return name, plim
    except Exception as e:                    # noqa: BLE001
        return 'unknown (%s)' % e, 'unknown'


def pictures(margin, third=False):
    """org, cur (and with `third` a second reference, drawn after them from the same RandomState, so org and cur do not change), then the stride S"""
    rs = np.random.RandomState(2160)
    S = PW + 2 * margin
    b = rs.randint(0, 1024, size=(PH + 2 * margin + 8, S + 8))
    sm = (b + np.roll(b, 1, 0) + np.roll(b, 1, 1) + np.roll(b, (1, 1), (0, 1))) // 4
    org = np.ascontiguousarray(sm[4:4 + PH + 2 * margin, 4:4 + S], dtype=np.int16)
    cur = np.ascontiguousarray(np.clip(sm[1:1 + PH + 2 * margin, 7:7 + S] + rs.randint(-9, 10, size=org.shape), 0, 1023), dtype=np.int16)
    if not third:
        return org, cur, S
    oth = np.ascontiguousarray(np.clip(sm[6:6 + PH + 2 * margin, 2:2 + S] + rs.randint(-9, 10, size=org.shape), 0, 1023), dtype=np.int16)
    return org, cur, oth, S


def timed(eng, stream, fn, reps):
    """ms per call of fn on the engine's stream: one warm-up call, then CUDA events around `reps` calls"""
    import torch
    fn(); eng.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for _ in range(reps):
        fn()
    t1.record(stream); t1.synchronize()
    return t0.elapsed_time(t1) / reps
