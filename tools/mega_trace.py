"""Summarise a GGML_B200_MEGA_TRACE dump of the persistent dataflow decode kernel (csrc/decode_flow.cu).

Per phase and CTA the kernel stamps the globaltimer at: 0 phase entered, 1 input vector arrived (all of its tagged slots valid),
2 activation quantised and in registers, 3 all of the CTA's rows done.  A phase has no barrier, so "time of a phase" is defined by
the dependency it sits on: from the moment the LAST producer CTA of the previous phase finished (max of stamp 3 of the previous
phase) to the moment the last CTA of this phase finished.  CTAs without rows in a phase leave no stamps 1..3."""
import collections
import json
import os
import struct
import sys

import numpy as np


def hbm_peak() -> float:
    """GB/s: the measured peak when MEASURED_PEAKS.json exists, else the H100 SXM data sheet's 3.35 TB/s (as bench.py)"""
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"])
    return 3350.0


raw = open(sys.argv[1], "rb").read()
n, grid = struct.unpack("ii", raw[:8])
rec = np.frombuffer(raw[8:8 + 16 * n], np.int32).reshape(n, 4)
body = np.frombuffer(raw[8 + 16 * n:], np.uint64)
TN = body.size // (n * 160)            # words per phase and CTA (decode_flow.cuh FLOW_TRACE_N; 6 in older dumps)
t = body.reshape(-1, TN, 160)[:n, :, :grid].astype(np.float64)
FINE = TN >= 11 and (t[:, 8] > 0).any()
KN = {0: "MATVEC", 1: "ATTN", 2: "COPY", 3: "ADD"}
BB = {12: 144, 13: 176, 14: 210}
PEAK = hbm_peak()


def bytes_of(r):
    if r[0] != 0:
        return 0
    K, M, ty = int(r[1]), int(r[2]), int(r[3])
    return M * (K // 256) * BB.get(ty % 100, 0)     # (mixed-type phases: counted with the first matrix's type -- close enough for a summary)


ts = t[:, :4]                          # the four globaltimer stamps (slots 4, 5 are cycle counters)
t0 = ts[ts > 0].min()
end_prev = t0
agg = collections.OrderedDict()
fine = {}
total_span = 0.0
for i in range(n):
    done = t[i, 3]
    have = done > 0
    if rec[i, 0] != 0 or not have.any():
        # attention / copy phases: no stamp 3; use the next phase's input-arrival time as their end
        if i + 1 < n and (t[i + 1, 1] > 0).any():
            end = t[i + 1, 1][t[i + 1, 1] > 0].max()
        else:
            continue
        span = end - end_prev
        key = (KN.get(int(rec[i, 0]), "?"), int(rec[i, 1]), int(rec[i, 2]), int(rec[i, 3]))
        a = agg.setdefault(key, [0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
        a[0] += 1; a[1] += span
        total_span += span
        end_prev = end
        continue
    end = done[have].max()
    span = end - end_prev
    arrive = (t[i, 1][have] - end_prev)
    quant = (t[i, 2][have] - t[i, 1][have])
    stream = (done[have] - t[i, 2][have])
    key = (KN[0], int(rec[i, 1]), int(rec[i, 2]), int(rec[i, 3]))
    a = agg.setdefault(key, [0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
    a[0] += 1; a[1] += span; a[2] += arrive.mean(); a[3] += quant.mean(); a[4] += stream.mean(); a[5] += (done[have].max() - done[have].min())
    a[6] += t[i, 4][have].mean(); a[7] += t[i, 5][have].mean()
    if FINE:
        f = fine.setdefault(key, [0.0] * 6)
        h6 = have & (t[i, 6] > 0)
        f[0] += (t[i, 6][h6] - end_prev).mean() if h6.any() else 0.0          # first chunk valid
        f[1] += (t[i, 1][h6] - t[i, 6][h6]).mean() if h6.any() else 0.0       # batch rounds until pass 1 resolved
        h7 = have & (t[i, 7] > 0)
        f[2] += (t[i, 7][h7] - t[i, 1][h7]).mean() if h7.any() else 0.0       # norm reduction
        f[3] += (t[i, 8][have] - np.where(t[i, 7][have] > 0, t[i, 7][have], t[i, 1][have])).mean()   # quantise (+ later passes)
        f[4] += (t[i, 2][have] - t[i, 8][have]).mean()                        # CTA barrier + registers
        h10 = have & (t[i, 10] > 0)
        f[5] += (t[i, 10][h10].max() - end_prev) if h10.any() else 0.0        # last warp of the last CTA done
    total_span += span
    end_prev = end
print(f"{n} phases, grid {grid}; token span {(ts[ts > 0].max() - t0) / 1e3:.1f} us; sum of phase spans {total_span / 1e3:.1f} us; ideal = weight bytes / {PEAK:.0f} GB/s")
print(f"{'phase (kind, K, sum M, type)':42s} {'n':>4s} {'span us':>8s} {'ideal us':>8s} {'x-arrive':>8s} {'quantise':>8s} {'stream':>8s} {'skew':>6s} {'w0 wait kcyc':>12s} {'w0 comp kcyc':>12s}")
for key, (c, span, arr, qd, strm, skew, tw, tc) in agg.items():
    ideal = bytes_of((0 if key[0] == "MATVEC" else 1, key[1], key[2], key[3])) / PEAK / 1e3
    print(f"{str(key):42s} {c:4d} {span / c / 1e3:8.2f} {ideal:8.2f} {arr / c / 1e3:8.2f} {qd / c / 1e3:8.2f} {strm / c / 1e3:8.2f} {skew / c / 1e3:6.2f} {tw / c / 1e3:12.2f} {tc / c / 1e3:12.2f}")

if FINE:
    print()
    print("fine stamps (thread 0 of every CTA, mean over CTAs, us after the previous phase's last warp-0 finish):")
    print(f"{'phase':42s} {'first chunk':>11s} {'+rounds':>8s} {'+norm':>8s} {'+quant':>8s} {'+bar/regs':>9s} {'last warp':>9s}")
    for key, f in fine.items():
        c = agg[key][0]
        print(f"{str(key):42s} {f[0] / c / 1e3:11.2f} {f[1] / c / 1e3:8.2f} {f[2] / c / 1e3:8.2f} {f[3] / c / 1e3:8.2f} {f[4] / c / 1e3:9.2f} {f[5] / c / 1e3:9.2f}")
