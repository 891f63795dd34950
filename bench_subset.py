#!/usr/bin/env python3
"""bench_subset.py -- what a call over a list of streams (b200s_run_streams*) saves when only part of a batch is active.

Workload: batch 1024 stereo, 48 kHz presetDefault, 0.8x, 32 blocks per step (bench.py's main configuration).  A fixed
random share of the slots (1 %, 10 %, 50 %, 100 %) processes every step; the others are idle.  Each share runs two ways:
  subset  b200s_run_streams* with the active slots listed, buffers [n][2][stride]
  skip    b200s_run_per_stream* with the idle slots SKIP, buffers [1024][2][stride]
and is measured three ways:
  device_ms    device-resident buffers (the *_device calls), CUDA events around the timed steps, and one profiled step
               (profile_end(phases=True): per-kernel device time and launch counts)
  e2e_ms       pinned host buffers (the *_async calls, chained step after step), host clock around the timed steps,
               which end in a synchronise
  pcie_bytes   bytes over PCIe per step, computed from the shapes (input rows in, output rows out)
The two ways alternate (subset, skip, subset, skip) so that both see the same machine; every figure is listed per
repetition.  Prints one JSON line per share; the card's name and power limit are read in the same run.

    python bench_subset.py [--steps 20] [--warmup 5] [--reps 2] [--share 1,10,50,100]
"""
import argparse
import ctypes
import json
import sys
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
    x = signal(S, C, 2 * in_stride)
    dev_in = [x[:, :, k * in_stride:(k + 1) * in_stride].contiguous() for k in range(2)]  # [S][C][stride], slot order
    del x
    dev_in_list = [d[torch.from_numpy(lst).long().cuda()].contiguous() for d in dev_in]   # [n][C][stride], list order
    dev_out = torch.empty((S, C, out_stride), dtype=torch.float32, device="cuda")
    host_in = [d.cpu().pin_memory() for d in dev_in]
    host_in_list = [d.cpu().pin_memory() for d in dev_in_list]
    host_out = torch.empty((S, C, out_stride), dtype=torch.float32).pin_memory()
    lib, h = e._lib, e._h
    ip, dp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)
    # the arrays of both ways, made before any timed loop
    ops_all = np.zeros(S, np.int32)
    ops_all[lst] = PROCESS
    n_in_all, n_out_all = np.where(ops_all == PROCESS, in_stride, 0).astype(np.int32), np.where(ops_all == PROCESS, out_stride, 0).astype(np.int32)
    ops_l, n_in_l, n_out_l = np.full(n, PROCESS, np.int32), np.full(n, in_stride, np.int32), np.full(n, out_stride, np.int32)
    P = lambda v: v.ctypes.data_as(ip)  # noqa: E731
    e._adopt_torch_stream()

    def step(way, device, k):
        if way == "subset":
            src = (dev_in_list if device else host_in_list)[k % 2].data_ptr()
            fn = lib.b200s_run_streams_device if device else lib.b200s_run_streams_async
            rc = fn(h, n, P(lst), P(ops_l), src, in_stride, P(n_in_l), (dev_out if device else host_out).data_ptr(), out_stride, P(n_out_l), None)
        else:
            src = (dev_in if device else host_in)[k % 2].data_ptr()
            fn = lib.b200s_run_per_stream_device if device else lib.b200s_run_per_stream_async
            rc = fn(h, P(ops_all), src, in_stride, P(n_in_all), (dev_out if device else host_out).data_ptr(), out_stride, P(n_out_all), None)
        e._ck(rc)

    def timed(way, device):
        for k in range(a.warmup):
            step(way, device, k)
        e.synchronize()
        torch.cuda.synchronize()
        if device:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for k in range(a.steps):
                step(way, True, k)
            ev1.record()
            torch.cuda.synchronize()
            return ev0.elapsed_time(ev1) / a.steps
        t0 = time.perf_counter()
        for k in range(a.steps):
            step(way, False, k)
        e.synchronize()
        return (time.perf_counter() - t0) * 1e3 / a.steps

    res = {"share_pct": pct, "listed": n, "batch": S, "channels": C, "blocks_per_step": a.blocks, "ratio": RATIO}
    ways = ("subset", "skip")
    for w in ways:
        res[w] = {"device_ms": [], "e2e_ms": []}
    for _ in range(a.reps):
        for w in ways:
            res[w]["device_ms"].append(round(timed(w, True), 3))
        for w in ways:
            res[w]["e2e_ms"].append(round(timed(w, False), 3))
    for w in ways:
        rows = n if w == "subset" else S
        res[w]["pcie_bytes"] = rows * C * (in_stride + out_stride) * 4
        e.profile_begin()
        step(w, True, 0)
        prof = e.profile_end(phases=True)
        res[w]["profile_ms"] = {k: round(v[0], 3) for k, v in prof.items()}
        res[w]["profile_launches"] = {k: v[1] for k, v in prof.items()}
    res["pcie_bytes_ratio"] = round(res["subset"]["pcie_bytes"] / res["skip"]["pcie_bytes"], 4)
    res["unserved_random_blocks"] = e.unserved_random_blocks()
    res["gpu"], res["power_limit"] = name, limit
    print(json.dumps(res))
    sys.stdout.flush()
    del e, dev_in, dev_in_list, dev_out, host_in, host_in_list, host_out
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--share", default="1,10,50,100")
    a = ap.parse_args()
    name, limit = card()
    for pct in a.share.split(","):
        run_share(a, float(pct), name, limit)


if __name__ == "__main__":
    main()
