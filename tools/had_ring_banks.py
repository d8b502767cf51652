#!/usr/bin/env python3
"""shared-memory bank check of had8_ring_kernel (search_kernels.cuh): evaluates the kernel's window address formula for every lane of every warp and
reports the worst number of lanes that hit one bank in a single LDS, per block size, staged radius RC, CTA size and pattern point.
The window starts at the exact pel x + start_x - RC, so the parity of start_x does not enter the read addresses; it only decides which staging
thread writes a word.  usage: python tools/had_ring_banks.py"""
import sys


def shape(W, RC):                         # HadRingShape<W, RC>
    TX = W // 8; T = TX * TX; ROWS = W + 2 * RC; WPR = W // 2 + RC
    PITCH = WPR + (1 if (TX == 4 and WPR % 4 == 0) else 0)
    WIN1 = ROWS * PITCH
    S = ((2 * WIN1 + 3) & ~7) + 4
    return dict(TX=TX, T=T, ROWS=ROWS, WPR=WPR, PITCH=PITCH, WIN1=WIN1, S=S)


def lanes(W, RC, threads):
    """per thread: laneBase and the word order x-or xr, as the kernel computes them (xr = rank among the warp's lanes with equal laneBase / 4 mod 8)"""
    s = shape(W, RC)
    out = []
    for warp in range(threads // 32):
        base = []
        for lane in range(32):
            tid = warp * 32 + lane
            slot, t = tid // s['T'], tid % s['T']
            tx, ty = t % s['TX'], t // s['TX']
            base.append(slot * s['S'] + 8 * ty * s['PITCH'] + 4 * tx)
        cls = [(b >> 2) & 7 for b in base]
        xr = [sum(1 for l2 in range(l) if cls[l2] == cls[l]) & 3 for l in range(32)]
        out.append(list(zip(base, xr)))
    return out


def worst(W, RC, threads, R):
    s = shape(W, RC)
    w = 0
    for warp in lanes(W, RC, threads):
        for dy in range(-R, R + 1):
            for dx in range(-R, R + 1):
                cx = dx + RC
                off = (dy + RC) * s['PITCH'] + (cx >> 1) + (cx & 1) * s['WIN1']
                for r in range(8):
                    for i in range(4):
                        banks = {}
                        for base, xr in warp:
                            b = (base + (i ^ xr) + off + r * s['PITCH']) % 32
                            banks[b] = banks.get(b, 0) + 1
                        w = max(w, max(banks.values()))
    return w


def main():
    bad = 0
    print('%4s %3s %7s %6s %6s %6s  %s' % ('W', 'RC', 'threads', 'pitch', 'S', 'words', 'worst lanes per bank per LDS'))
    for W in (16, 32, 64):             # 8x8 blocks take had8_direct_kernel
        for RC in (2, 8):
            s = shape(W, RC)
            for threads in (32, 64, 128):
                if threads < s['T']:
                    continue
                m = worst(W, RC, threads, RC)
                bad += m > 1
                print('%4d %3d %7d %6d %6d %6d  %d' % (W, RC, threads, s['PITCH'], s['S'], 2 * s['WIN1'], m))
    return 1 if bad else 0


if __name__ == '__main__':
    sys.exit(main())
