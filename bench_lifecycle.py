#!/usr/bin/env python3
"""bench_lifecycle.py -- device-resident time per step of ONE batch whose streams each run their own operation
(b200s_run_per_stream_device): a streaming server whose slots turn over while the others keep processing.

Workload: batch 1024 stereo, 48 kHz presetDefault, 0.8x, 32 blocks per step, input and output in device memory.
The mixes (per step):
  process_per_stream  every stream PROCESS through b200s_process_per_stream_device (the reference point)
  all_process         the same through b200s_run_per_stream_device with every op PROCESS
  turnover_1          1 % of the slots FLUSH (outputLatency samples at 0.8) and as many OUTPUT_SEEK (the slots flushed in
                      the step before, outputSeekLength(0.8) samples), the rest PROCESS
  turnover_10         the same with 10 %
  half_skip           every other slot SKIP, the others PROCESS
Per mix: warm-up steps, then CUDA-event timing of the timed steps, then one profiled step (per-kernel times of
profile_end(phases=True): "phases" is the pre and post phases of the call).  Prints one JSON line per mix; the card's
name and power limit are read in the same run.

    python bench_lifecycle.py [--steps 20] [--warmup 5] [--batch 1024] [--mix all_process,turnover_1,...]
"""
import argparse
import ctypes
import json
import sys

import numpy as np

from bench_mixed import card
from bench_ragged import signal

SR = 48000.0
RATIO = 0.8
MIXES = ("process_per_stream", "all_process", "turnover_1", "turnover_10", "half_skip")
SKIP, PROCESS, SEEK, OUTPUT_SEEK, FLUSH, RESET = range(6)


def mix_ops(mix, S, k):
    """Per-stream ops of step k."""
    ops = np.full(S, PROCESS, np.int32)
    if mix.startswith("turnover_"):
        m = max(1, int(round(S * int(mix.split("_")[1]) / 100)))
        flush = (k * m + np.arange(m)) % S
        ops[(flush - m) % S] = OUTPUT_SEEK  # the slots flushed in the step before start their next track
        ops[flush] = FLUSH
    elif mix == "half_skip":
        ops[1::2] = SKIP
    elif mix not in ("process_per_stream", "all_process"):
        raise ValueError(mix)
    return ops


def device_mix(a, mix, name, limit):
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C = a.batch, 2
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    H = e.intervalSamples()
    n = a.blocks * H
    in_stride, out_stride = int(round(n / RATIO)), n
    seek_len, flush_len = e.outputSeekLength(RATIO), e.outputLatency()
    e.reserve(in_stride, out_stride)
    x = signal(S, C, 4 * in_stride)
    chunks = [x[:, :, k * in_stride:(k + 1) * in_stride].contiguous() for k in range(4)]
    del x
    out = torch.empty((S, C, out_stride), dtype=torch.float32, device="cuda")
    rates = np.full(S, RATIO)
    # every step's arrays are made before the timed loop: the host work is the engine's, not numpy's
    plans = []
    for k in range(a.warmup + a.steps):
        ops = mix_ops(mix, S, k)
        n_in = np.select([ops == PROCESS, ops == OUTPUT_SEEK], [in_stride, seek_len], 0).astype(np.int32)
        n_out = np.select([ops == PROCESS, ops == FLUSH], [out_stride, flush_len], 0).astype(np.int32)
        plans.append((ops, n_in, n_out))
    lib, h = e._lib, e._h
    ip, dp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)
    e._adopt_torch_stream()

    def step(k):
        ops, n_in, n_out = plans[k]
        src = chunks[k % 4].data_ptr()
        if mix == "process_per_stream":
            rc = lib.b200s_process_per_stream_device(h, src, in_stride, n_in.ctypes.data_as(ip), out.data_ptr(), out_stride, n_out.ctypes.data_as(ip))
        else:
            rc = lib.b200s_run_per_stream_device(h, ops.ctypes.data_as(ip), src, in_stride, n_in.ctypes.data_as(ip), out.data_ptr(), out_stride,
                                                 n_out.ctypes.data_as(ip), rates.ctypes.data_as(dp))
        e._ck(rc)

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
    step(a.warmup)
    prof = e.profile_end(phases=True)
    ops = plans[a.warmup][0]
    print(json.dumps({
        "mix": mix, "batch": S, "channels": C, "blocks_per_step": a.blocks,
        "ops": {k: int(np.count_nonzero(ops == v)) for k, v in (("process", PROCESS), ("flush", FLUSH), ("output_seek", OUTPUT_SEEK), ("skip", SKIP))},
        "ms_per_step": round(ms, 3), "profile_ms": {k: round(v[0], 3) for k, v in prof.items()},
        "profile_launches": {k: v[1] for k, v in prof.items()}, "unserved_random_blocks": e.unserved_random_blocks(),
        "gpu": name, "power_limit": limit,
    }))
    sys.stdout.flush()
    del e, chunks, out
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--mix", default=",".join(MIXES))
    a = ap.parse_args()
    name, limit = card()
    for mix in a.mix.split(","):
        device_mix(a, mix, name, limit)


if __name__ == "__main__":
    main()
