#!/usr/bin/env python3
"""bench_ragged.py -- device-resident time per step of ONE batch whose streams have their own input and output lengths
(b200s_process_per_stream_device).

Workload: batch 1024 stereo, 48 kHz presetDefault, up to 32 blocks per process() call, input and output in device memory.
The length mixes (per stream):
  uniform          every stream 0.8x, 32 blocks, through b200s_process_device (the reference point)
  per_stream_same  the same lengths through b200s_process_per_stream_device
  ratios           ratios drawn from {0.55, 0.67, 0.8, 1.0, 1.25, 1.5, 1.8} with a fixed seed, every stream 32 blocks out
  half_idle        every other slot idle with (0, 0), the others 0.8x, 32 blocks
  out_lengths      output lengths drawn from [8, 32] blocks with a fixed seed, 0.8x
Per mix: warm-up steps, then CUDA-event timing of the timed steps, then one profiled step (per-kernel times of
profile_end()).  Prints one JSON line per mix; the card's name and power limit are read in the same run.

--pinned also times the host-buffer pipeline on pinned memory: chained b200s_process_per_stream_async calls whose lengths
change every call (0.8x, outputs drawn from [24, 32] blocks) against uniform b200s_process_async calls at the same strides.

    python bench_ragged.py [--steps 20] [--warmup 5] [--batch 1024] [--mix uniform,ratios,...] [--pinned]
"""
import argparse
import json
import sys

import numpy as np

from bench_mixed import card

SR = 48000.0
RATIO = 0.8
MIXES = ("uniform", "per_stream_same", "ratios", "half_idle", "out_lengths")
RATIOS = (0.55, 0.67, 0.8, 1.0, 1.25, 1.5, 1.8)


def mix_lengths(mix, S, H, blocks, seed=1234):
    """Per-stream (input samples, output samples) of a mix."""
    rng = np.random.default_rng(seed)
    n_out = np.full(S, blocks * H, np.int64)
    ratio = np.full(S, RATIO)
    if mix == "ratios":
        ratio = np.array(RATIOS)[rng.integers(0, len(RATIOS), S)]
    elif mix == "out_lengths":
        n_out = rng.integers(8, blocks + 1, S) * H
    elif mix not in ("uniform", "per_stream_same", "half_idle"):
        raise ValueError(mix)
    n_in = np.round(n_out / ratio).astype(np.int64)
    if mix == "half_idle":
        n_in[1::2] = 0
        n_out[1::2] = 0
    return n_in.astype(np.int32), n_out.astype(np.int32)


def signal(S, C, n, device="cuda"):
    import torch

    t = torch.arange(n, dtype=torch.float32, device=device) / SR
    f0 = 110.0 * (1 + torch.arange(S, dtype=torch.float32, device=device) % 17 / 8.0)
    x = torch.empty((S, C, n), dtype=torch.float32, device=device)
    for c in range(C):
        x[:, c] = 0.3 * torch.sin(2 * np.pi * f0[:, None] * t[None, :]) + 0.1 * torch.sin(2 * np.pi * 3.01 * f0[:, None] * t[None, :] + c)
    return x


def device_mix(a, mix, name, limit):
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C = a.batch, 2
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    H = e.intervalSamples()
    n_in, n_out = mix_lengths(mix, S, H, a.blocks)
    in_stride, out_stride = int(n_in.max()), int(n_out.max())
    e.reserve(in_stride, out_stride)
    # four distinct input chunks, used in turn (the time only depends on the schedule, which every chunk shares)
    x = signal(S, C, 4 * in_stride)
    chunks = [x[:, :, k * in_stride:(k + 1) * in_stride].contiguous() for k in range(4)]
    del x
    out = torch.empty((S, C, out_stride), dtype=torch.float32, device="cuda")
    if mix == "uniform":
        step = lambda k: e.process(chunks[k % 4], out_stride, out=out)  # noqa: E731
    else:
        step = lambda k: e.process(chunks[k % 4], n_out, out=out, inputSamples=n_in)  # noqa: E731
    for k in range(a.warmup):
        step(k)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for k in range(a.warmup, a.warmup + a.steps):
        step(k)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / a.steps
    e.profile_begin()
    step(0)
    prof = e.profile_end()
    print(json.dumps({
        "mix": mix, "batch": S, "channels": C, "max_blocks_per_step": a.blocks,
        "active_streams": int(np.count_nonzero(n_out)), "output_samples": int(n_out.sum()), "input_samples": int(n_in.sum()),
        "ms_per_step": round(ms, 3), "profile_ms": {k: round(v[0], 3) for k, v in prof.items()},
        "profile_launches": {k: v[1] for k, v in prof.items()}, "gpu": name, "power_limit": limit,
    }))
    sys.stdout.flush()
    del e, chunks, out
    torch.cuda.empty_cache()


def pinned(a, name, limit):
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C = a.batch, 2
    rng = np.random.default_rng(77)
    for kind in ("uniform_async", "per_stream_async"):
        e = BatchStretch(S)
        e.presetDefault(C, SR)
        H = e.intervalSamples()
        out_stride = a.blocks * H
        in_stride = int(round(out_stride / RATIO))
        e.reserve(in_stride, out_stride)
        lens = []
        for _ in range(4):  # lengths that change every call
            n_out = (rng.integers(24, a.blocks + 1, S) * H).astype(np.int32)
            lens.append((np.round(n_out / RATIO).astype(np.int32), n_out))
        xin = [signal(S, C, in_stride).cpu().pin_memory() for _ in range(2)]
        xout = [torch.empty((S, C, out_stride), dtype=torch.float32).pin_memory() for _ in range(2)]

        def step(k):
            i, o = xin[k % 2].data_ptr(), xout[k % 2].data_ptr()
            if kind == "uniform_async":
                e.process_host_ptr_async(i, in_stride, o, out_stride)
            else:
                e.process_per_stream_host_ptr(i, in_stride, lens[k % 4][0], o, out_stride, lens[k % 4][1])

        for k in range(a.warmup):
            step(k)
        e.synchronize()
        e.timer_start()
        for k in range(a.warmup, a.warmup + a.steps):
            step(k)
        ms = e.timer_stop() / a.steps
        print(json.dumps({"mix": kind, "batch": S, "channels": C, "in_stride": in_stride, "out_stride": out_stride,
                          "ms_per_step": round(ms, 3), "gpu": name, "power_limit": limit}))
        sys.stdout.flush()
        del e, xin, xout
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--mix", default=",".join(MIXES))
    ap.add_argument("--pinned", action="store_true")
    a = ap.parse_args()
    name, limit = card()
    for mix in a.mix.split(","):
        device_mix(a, mix, name, limit)
    if a.pinned:
        pinned(a, name, limit)


if __name__ == "__main__":
    main()
