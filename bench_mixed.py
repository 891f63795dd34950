#!/usr/bin/env python3
"""bench_mixed.py -- device-resident time per step of ONE batch whose streams have different parameters.

Workload: batch 1024 stereo, 48 kHz presetDefault, 0.8x time-stretch, 32 blocks per process() call, input and output in
device memory.  The parameter mixes (per stream, through the per-stream setters):
  plain      every stream a pure time-stretch (the plain kernels only)
  all_7st    every stream +7 semitones with an 8 kHz tonality limit (the mapped kernels only)
  half_7st   every other stream +7 st, 8 kHz tonality limit
  tenth_7st  every tenth stream +7 st, 8 kHz tonality limit
  random     semitones drawn from [-12, 12] with a fixed seed, 10 % of the streams at 0 (plain), 10 % with formant
             compensation at a 200 Hz formant base
Per mix: warm-up steps, then CUDA-event timing of the timed steps, then one profiled step (per-kernel times of
profile_end()).  Prints one JSON line per mix; the card's name and power limit are read in the same run.

    python bench_mixed.py [--steps 20] [--warmup 5] [--batch 1024] [--mix plain,all_7st,...]
"""
import argparse
import json
import subprocess
import sys

import numpy as np

SR = 48000.0
RATIO = 0.8
MIXES = ("plain", "all_7st", "half_7st", "tenth_7st", "random")


def mix_parameters(mix, S, seed=1234):
    """Per-stream (semitones, tonality limit, formant compensation, formant base) of a mix; frequencies / sample rate."""
    semis = np.zeros(S, np.float32)
    ton = np.full(S, 8000 / SR, np.float32)
    comp = np.zeros(S, np.int32)
    base = np.zeros(S, np.float32)
    if mix == "all_7st":
        semis[:] = 7
    elif mix == "half_7st":
        semis[1::2] = 7
    elif mix == "tenth_7st":
        semis[::10] = 7
    elif mix == "random":
        rng = np.random.default_rng(seed)
        semis[:] = rng.uniform(-12, 12, S)
        order = rng.permutation(S)
        n10 = S // 10
        semis[order[:n10]] = 0
        comp[order[n10:2 * n10]] = 1
        base[order[n10:2 * n10]] = 200 / SR
    elif mix != "plain":
        raise ValueError(mix)
    return semis, ton, comp, base


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:  # (read-only query)
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        limit = "unknown (%s)" % ex
    return name, limit


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
        semis, ton, comp, base = mix_parameters(mix, S)
        e.setTransposeSemitones(semis, ton)
        e.setFormantFactor(np.ones(S, np.float32), comp)
        e.setFormantBase(base)
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
        print(json.dumps({
            "mix": mix, "batch": S, "channels": C, "blocks_per_step": a.blocks, "ratio": RATIO,
            "mapped_streams": int(np.count_nonzero((semis != 0) | (comp != 0))),
            "ms_per_step": round(ms, 3), "profile_ms": {k: round(v[0], 3) for k, v in prof.items()},
            "profile_launches": {k: v[1] for k, v in prof.items()}, "gpu": name, "power_limit": limit,
        }))
        sys.stdout.flush()
        del e, chunks, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
