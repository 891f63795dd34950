#!/usr/bin/env python3
"""bench_pcm16.py -- what 16-bit PCM host buffers save on the listed calls (b200s_run_streams_pcm16 against
b200s_run_streams_async).

Workload: bench_subset.py's, batch 1024 stereo, 48 kHz presetDefault, 0.8x, 32 blocks per step (bench.py's main
configuration).  A fixed random share of the slots (10 %, 50 %, 100 %) is listed and processes every step.  Each share
runs in two formats on pinned host buffers [n][2][stride], chained step after step:
  f32     b200s_run_streams_async, float32 rows
  pcm16   b200s_run_streams_pcm16 with wait = 0, int16 rows, converted on the device (k_pcm16_in / k_pcm16_out)
and is measured three ways:
  e2e_ms         host clock around the timed steps, which end in a synchronise; the formats alternate (f32, pcm16, f32,
                 pcm16) so that both see the same machine, and every repetition is listed
  pcie_bytes     bytes over PCIe per step, computed from the shapes (input rows in, output rows out)
  convert_ms     device time of k_pcm16_in and k_pcm16_out per step, from a separate torch.profiler run of the 16-bit
                 format (tracing slows the host, so it is kept out of the e2e figures)
Prints one JSON line per share; the card's name and power limit are read in the same run.

    python bench_pcm16.py [--steps 20] [--warmup 5] [--reps 3] [--share 10,50,100] [--profile-steps 10]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

from bench_mixed import card
from bench_ragged import signal

SR = 48000.0
RATIO = 0.8
PROCESS = 1


def run_share(a, pct, name, limit):
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C = a.batch, 2
    n = max(1, int(round(S * pct / 100)))
    lst = np.sort(np.random.default_rng(int(pct)).permutation(S)[:n]).astype(np.int32)
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    H = e.intervalSamples()
    out_stride = a.blocks * H
    in_stride = int(round(out_stride / RATIO))
    e.reserve(in_stride, out_stride)
    x = signal(n, C, 2 * in_stride)
    # two input slabs [n][C][stride] per format: the 16-bit rows, and the float rows they stand for (x16 / 32768)
    x16 = [torch.clamp(torch.round(x[:, :, k * in_stride:(k + 1) * in_stride] * 32768), -32768, 32767).to(torch.int16) for k in range(2)]
    host_in = {"pcm16": [t.cpu().pin_memory() for t in x16], "f32": [(t.float() / 32768).cpu().pin_memory() for t in x16]}
    del x, x16
    host_out = {"pcm16": torch.empty((n, C, out_stride), dtype=torch.int16).pin_memory(),
                "f32": torch.empty((n, C, out_stride), dtype=torch.float32).pin_memory()}
    ops, n_in, n_out = np.full(n, PROCESS, np.int32), np.full(n, in_stride, np.int32), np.full(n, out_stride, np.int32)

    def step(fmt, k):
        src, dst = host_in[fmt][k % 2].data_ptr(), host_out[fmt].data_ptr()
        if fmt == "pcm16":
            e.run_pcm16_host_ptr(ops, src, in_stride, n_in, dst, out_stride, n_out, streams=lst, wait=False)
        else:
            e.run_streams_host_ptr(lst, ops, src, in_stride, n_in, dst, out_stride, n_out, wait=False)

    def timed(fmt):
        for k in range(a.warmup):
            step(fmt, k)
        e.synchronize()
        t0 = time.perf_counter()
        for k in range(a.steps):
            step(fmt, k)
        e.synchronize()
        return (time.perf_counter() - t0) * 1e3 / a.steps

    fmts = ("f32", "pcm16")
    res = {"share_pct": pct, "listed": n, "batch": S, "channels": C, "blocks_per_step": a.blocks, "ratio": RATIO,
           "in_stride": in_stride, "out_stride": out_stride}
    for f in fmts:
        res[f] = {"e2e_ms": [], "pcie_bytes": n * C * (in_stride + out_stride) * (2 if f == "pcm16" else 4)}
    allocs = None
    for r in range(a.reps):
        for f in fmts:
            res[f]["e2e_ms"].append(round(timed(f), 3))
        if r == 0:
            allocs = e.device_allocations()
    res["allocations_after_first_rep"] = e.device_allocations() - allocs
    res["pcie_bytes_ratio"] = round(res["pcm16"]["pcie_bytes"] / res["f32"]["pcie_bytes"], 4)

    # the conversions' device time: a profiled run of its own
    from torch.profiler import ProfilerActivity, profile

    for k in range(a.warmup):
        step("pcm16", k)
    e.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(a.profile_steps):
            step("pcm16", k)
        e.synchronize()
    conv = {"k_pcm16_in": [0.0, 0], "k_pcm16_out": [0.0, 0]}
    with tempfile.TemporaryDirectory() as d:  # (the kernels' records of the trace: name and duration in microseconds)
        prof.export_chrome_trace(os.path.join(d, "trace.json"))
        with open(os.path.join(d, "trace.json")) as f:
            trace = json.load(f)
    for ev in trace.get("traceEvents", []):
        for kname in conv:
            if ev.get("cat") == "kernel" and kname in ev.get("name", ""):
                conv[kname][0] += ev["dur"] / 1e3
                conv[kname][1] += 1
    res["pcm16"]["convert_ms"] = {k: round(v[0] / a.profile_steps, 4) for k, v in conv.items()}
    res["pcm16"]["convert_launches_per_step"] = {k: v[1] / a.profile_steps for k, v in conv.items()}
    res["unserved_random_blocks"] = e.unserved_random_blocks()
    res["gpu"], res["power_limit"] = name, limit
    print(json.dumps(res))
    sys.stdout.flush()
    del e, host_in, host_out
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--share", default="10,50,100")
    ap.add_argument("--profile-steps", type=int, default=10)
    a = ap.parse_args()
    name, limit = card()
    for pct in a.share.split(","):
        run_share(a, float(pct), name, limit)


if __name__ == "__main__":
    main()
