#!/usr/bin/env python3
"""bench_freqmap.py -- device-resident time per step of ONE batch whose streams have their own frequency-map tables.

Workload: batch 1024 stereo, 48 kHz presetDefault, 0.8x time-stretch, 32 blocks per process() call, input and output in
device memory.  Every table has 2049 points (setFreqMap's default tabulation).  The mixes:
  engine        one table for the engine (b200s_set_freq_map_table), on every stream
  same_each     that table set on every stream through b200s_set_freq_map_table_per_stream (one pooled table)
  distinct64    64 distinct tables, stream s takes table s % 64
  own_each      every stream its own table (1024 tables)
  half_plain    64 distinct tables on the even streams; the odd streams plain
  formants      distinct64 with formant compensation at a 200 Hz formant base
The question is whether per-stream tables cost anything next to the engine's one table: the same kernels run, and only
the table each stream's binary search reads differs.
Per mix: warm-up steps, then CUDA-event timing of the timed steps, then one profiled step (per-kernel times of
profile_end()).  Then the host time of one b200s_set_freq_map_table_per_stream call that gives 1024 streams 1024
distinct tables (taken on a pool already that large, and on a fresh engine, where the pool is allocated).  Prints one
JSON line per mix and one for the set call; the card's name and power limit are read in the same run.

    python bench_freqmap.py [--steps 20] [--warmup 5] [--batch 1024] [--mix engine,same_each,...]
"""
import argparse
import ctypes
import json
import sys
import time

import numpy as np

from bench_mixed import card

SR = 48000.0
RATIO = 0.8
POINTS = 2049
MIXES = ("engine", "same_each", "distinct64", "own_each", "half_plain", "formants")


def table(k):
    """Map k: a transposition between -6 and +6 semitones with a gentle curve, tabulated on [0, 0.5]."""
    fin = np.linspace(0.0, 0.5, POINTS).astype(np.float32)
    st = -6 + 12 * ((k * 37) % 1024) / 1023.0
    fout = (fin * 2 ** (st / 12) * (1 + 0.05 * np.sin(20 * fin + k))).astype(np.float32)
    return fin, fout


def set_tables(e, streams, tabs):
    """b200s_set_freq_map_table_per_stream with ready arrays: (host seconds of the call)."""
    ip, fp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float)
    s = np.ascontiguousarray(streams, np.int32)
    pts = np.array([len(t[0]) for t in tabs], np.int32)
    fin = np.ascontiguousarray(np.concatenate([t[0] for t in tabs]), np.float32)
    fout = np.ascontiguousarray(np.concatenate([t[1] for t in tabs]), np.float32)
    t0 = time.perf_counter()
    e._ck(e._lib.b200s_set_freq_map_table_per_stream(e._h, s.ctypes.data_as(ip), len(s), pts.ctypes.data_as(ip),
                                                      fin.ctypes.data_as(fp), fout.ctypes.data_as(fp)))
    return time.perf_counter() - t0


def apply_mix(e, mix, S):
    """Returns the number of streams on the mapped path."""
    if mix == "engine":
        e.setFreqMapTable(*table(0))
    elif mix == "same_each":
        set_tables(e, range(S), [table(0)] * S)
    elif mix in ("distinct64", "formants"):
        set_tables(e, range(S), [table(s % 64) for s in range(S)])
        if mix == "formants":
            e.setFormantFactor(1.0, True)
            e.setFormantBase(200 / SR)
    elif mix == "own_each":
        set_tables(e, range(S), [table(s) for s in range(S)])
    elif mix == "half_plain":
        set_tables(e, range(0, S, 2), [table(s % 64) for s in range(0, S, 2)])
    else:
        raise ValueError(mix)
    return (S + 1) // 2 if mix == "half_plain" else S


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--mix", default=",".join(MIXES))
    a = ap.parse_args()
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    name, limit = card()
    S, C = a.batch, 2
    for mix in a.mix.split(","):
        e = BatchStretch(S)
        e.presetDefault(C, SR)
        H = e.intervalSamples()
        n_out = a.blocks * H
        n_in = int(round(n_out / RATIO))
        mapped = apply_mix(e, mix, S)
        e.reserve(n_in, n_out)
        # four distinct input chunks, used in turn (the time only depends on the schedule, which every chunk shares)
        t = torch.arange(4 * n_in, dtype=torch.float32, device="cuda") / SR
        f0 = 110.0 * (1 + torch.arange(S, dtype=torch.float32, device="cuda") % 17 / 8.0)
        x = torch.empty((S, C, 4 * n_in), dtype=torch.float32, device="cuda")
        for c in range(C):
            x[:, c] = 0.3 * torch.sin(2 * np.pi * f0[:, None] * t[None, :]) + 0.1 * torch.sin(2 * np.pi * 3.01 * f0[:, None] * t[None, :] + c)
        chunks = [x[:, :, k * n_in:(k + 1) * n_in].contiguous() for k in range(4)]
        del x, t
        out = torch.empty((S, C, n_out), dtype=torch.float32, device="cuda")
        for k in range(a.warmup):
            e.process(chunks[k % 4], n_out, out=out)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for k in range(a.warmup, a.warmup + a.steps):
            e.process(chunks[k % 4], n_out, out=out)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / a.steps
        e.profile_begin()
        e.process(chunks[0], n_out, out=out)
        prof = e.profile_end()
        assert bool(torch.isfinite(out).all())
        print(json.dumps({
            "mix": mix, "batch": S, "channels": C, "blocks_per_step": a.blocks, "ratio": RATIO, "mapped_streams": mapped,
            "ms_per_step": round(ms, 3), "profile_ms": {k: round(v[0], 3) for k, v in prof.items()},
            "profile_launches": {k: v[1] for k, v in prof.items()}, "gpu": name, "power_limit": limit,
        }))
        sys.stdout.flush()
        del e, chunks, out
        torch.cuda.empty_cache()
    # one set call of 1024 distinct tables: on a fresh engine (the pool is allocated), then again on that pool
    tabs = [table(s) for s in range(S)]
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    first = set_tables(e, range(S), tabs)
    again = [set_tables(e, range(S), tabs[k:] + tabs[:k]) for k in (1, 2, 3)]
    print(json.dumps({"set_call": "b200s_set_freq_map_table_per_stream", "streams": S, "distinct_tables": S, "points": POINTS,
                      "ms_first": round(first * 1e3, 3), "ms_within_capacity": [round(v * 1e3, 3) for v in again],
                      "gpu": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
