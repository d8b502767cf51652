#!/usr/bin/env python3
"""issue-rate probe of the SAD pyramid's instruction mixes on register operands (alu_probe_kernel, vvb_alu_probe_dev):
  mode 1: VIMNMX.S16x2 + IDP.2A per packed word (the pair the CUDA-core SAD kernels use)
  mode 2: per 4 words 2 VIMNMX.S16x2 + 2 HFMA2.RELU + 1 HMMA.16816.F32 (the SAD pyramid's pel sums on the tensor cores, DESIGN §5)
  mode 3: per 4 words 4 VIMNMX.S16x2 + 1 HMMA.16816.F32 (every minimum on the alu pipe)
  mode 4: the HMMA.16816.F32 alone (mma.sync m16n8k16, f16 operands, f32 accumulators): the tensor pipe's own rate
Prints the card, its power limit and SM clock limit, and pel differences per second and per lane and cycle for each mode.
usage: python tools/mma_probe.py [iters]"""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import vvenc_b200 as V


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(', ')
        return {'name': q[0], 'power_limit_w': float(q[1]), 'sm_max_mhz': float(q[2]), 'sm_mhz_now': float(q[3])}
    except Exception as e:                      # the numbers below still stand; the card line says why it is missing
        return {'name': torch.cuda.get_device_name(0), 'nvidia_smi': repr(e)}


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
    eng = V.CostEngine(0)
    lib = eng.lib
    ext = torch.cuda.ExternalStream(eng.stream)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = sms * 8
    diffs = ctas * 256 * iters * 16

    def once(mode):
        assert lib.vvb_alu_probe_dev(eng.h, ctas, iters, mode) == 0, lib.vvb_last_error(eng.h)

    def timed(mode, reps=5):
        once(mode)
        eng.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(ext):
            e0.record(ext)
            for _ in range(reps):
                once(mode)
            e1.record(ext)
        eng.synchronize(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps
    c = card()
    mhz = c.get('sm_max_mhz') or 1980.0
    out = {'card': c, 'ctas': ctas, 'iters': iters, 'modes': {}}
    for rnd in range(2):                         # two alternating rounds: the spread between them is the noise of the numbers
        for mode in (1, 2, 3, 4):
            ms = timed(mode)
            rate = diffs / (ms * 1e-3)
            out['modes'].setdefault(str(mode), []).append({'ms': round(ms, 4), 'Tpel_diff_s': round(rate / 1e12, 3),
                                                           'per_lane_cycle_at_max_clock': round(rate / (sms * 128 * mhz * 1e6), 3)})
    best = {m: max(r['Tpel_diff_s'] for r in v) for m, v in out['modes'].items()}
    out['mode2_over_mode1'] = round(best['2'] / best['1'], 3)
    out['mode3_over_mode1'] = round(best['3'] / best['1'], 3)
    out['mode4_over_mode1'] = round(best['4'] / best['1'], 3)
    hmma = ctas * 8 * iters * 2                  # warps x iterations x 2 HMMA steps
    ms4 = min(r['ms'] for r in out['modes']['4'])
    out['mma_sync_m16n8k16_TFLOPs'] = round(hmma * 2 * 16 * 8 * 16 / (ms4 * 1e-3) / 1e12, 1)
    out['mma_sync_cycles_per_hmma_per_scheduler'] = round(sms * 4 * mhz * 1e6 * ms4 * 1e-3 / hmma, 2)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
