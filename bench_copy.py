"""Time stream copies, export and import (b200s_copy_streams / _export_streams / _import_streams).

Batch 1024, stereo 48 kHz presetDefault, after warm-up (every case once, so its staging buffers exist), each case
timed over --reps repetitions:
  * copying 1, 102 and 1024 streams within one engine (device events on the engine's stream);
  * copying 102 streams into a second engine on the same device (events around both engines' streams);
  * export and import of 102 streams through pinned host memory (host clock around the synchronous calls).
Bytes moved come from the record size.  A device copy is one pack and one unpack, each reading and writing every record
once, so it moves 4 x record bytes per stream; its share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s) is that
over its time.  Export / import move one record per stream over PCIe each way.  Prints one JSON line, with the card's
name and power limit read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "unavailable (%s)" % e
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_copy.py needs a CUDA device")
    from signalsmith_stretch_b200 import BatchStretch

    S = args.batch
    g, h = BatchStretch(S), BatchStretch(S, seed=1)
    for e in (g, h):
        e.presetDefault(2, 48000.0)
    H = g.intervalSamples()
    x = np.random.default_rng(0).standard_normal((S, 2, 4 * H)).astype(np.float32) * 0.1
    g.process(x, 3 * H)  # (state worth copying; the timings do not depend on the values)
    R = g.state_bytes()
    rng = np.random.default_rng(1)
    n102 = max(1, S // 10)

    def lists(n):
        return rng.permutation(S)[:n], rng.permutation(S)[:n]

    def time_device(dst, n):
        d, s = lists(n)
        dst.copy_streams(d, s, src=g)  # warm-up: staging sized, modules loaded
        g.synchronize()
        dst.synchronize()
        g.timer_start()
        if dst is not g:
            dst.timer_start()
        for _ in range(args.reps):
            dst.copy_streams(d, s, src=g)
        ms = g.timer_stop() if dst is g else max(g.timer_stop(), dst.timer_stop())
        ms /= args.reps
        moved = 4 * n * R
        return {"streams": n, "ms": ms, "bytes_moved": moved, "GB_per_s": moved / ms / 1e6, "hbm_share": moved / (ms * 1e-3) / HBM_BYTES_PER_S}

    cases = {}
    for n in (1, n102, S):
        cases["copy_within_%d" % n] = time_device(g, n)
    cases["copy_between_engines_%d" % n102] = time_device(h, n102)
    streams = rng.permutation(S)[:n102]
    pinned = torch.empty((n102, R), dtype=torch.uint8).pin_memory()
    buf = pinned.numpy()
    lib = g._lib
    ip = ctypes.POINTER(ctypes.c_int)
    sl = np.ascontiguousarray(streams, np.int32)
    for name, fn, e in (("export", lib.b200s_export_streams, g), ("import", lib.b200s_import_streams, h)):
        if name == "import":
            lib.b200s_export_streams(g._h, sl.ctypes.data_as(ip), n102, buf.ctypes.data)
        assert fn(e._h, sl.ctypes.data_as(ip), n102, buf.ctypes.data) == 0  # warm-up
        t0 = time.perf_counter()
        for _ in range(args.reps):
            assert fn(e._h, sl.ctypes.data_as(ip), n102, buf.ctypes.data) == 0
        ms = (time.perf_counter() - t0) / args.reps * 1e3
        cases["%s_%d_pinned" % (name, n102)] = {"streams": n102, "ms": ms, "bytes_moved": n102 * R, "GB_per_s": n102 * R / ms / 1e6}
    name, q = card()
    print(json.dumps({"metric": "stream state copy / export / import", "batch": S, "config": "presetDefault stereo 48 kHz",
                      "record_bytes": R, "reps": args.reps, "gpu": name, "power_limit_and_max_sm_clock": q, "cases": cases}))


if __name__ == "__main__":
    main()
