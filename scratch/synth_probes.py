"""Where k_synth2's time goes: the benchmark's workload (1024 stereo streams, 48 kHz presetDefault, 0.8x, 32 blocks per
call) under the ablation builds of the synthesis kernel, next to the library as built.

    B200S_EXTRA_NVCC=-DB200S_SYNTH_PROBES builds the ablations (wrong results on purpose; never the shipped library):
    B200S_SYNTH_PROBE = 1 no windowProducts divisor (samples emitted undivided), 2 no ring update of the overlap-add at all,
    3 no wait on the staged spectra before the first pass, 4 inverse-FFT passes 2-3 skipped.

    python scratch/synth_probes.py --lib built.so --probe-lib probes.so [--rounds 3] [--out DIR]

Each measurement is a child process (the probe is read once per process); the rounds alternate the variants.  Prints
one JSON line per measurement: per-kernel device ms per step (CUDA events around every kernel) and the device time of a
whole step."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(lib, steps, warmup):
    import torch

    import bench
    from signalsmith_stretch_b200 import BatchStretch

    w = bench.workload(bench.BATCH_PER_GPU)
    eng = BatchStretch(w["batch"], lib_path=lib)
    eng.presetDefault(bench.CHANNELS, float(bench.SR))
    eng.reserve(w["n_in"], w["n_out"])
    x_host = bench.synth_input(w["batch"], 3 * w["n_in"])
    x = [torch.from_numpy(x_host[:, :, k * w["n_in"]:(k + 1) * w["n_in"]].copy()).cuda() for k in range(3)]
    y = torch.empty((w["batch"], bench.CHANNELS, w["n_out"]), dtype=torch.float32, device="cuda")
    for i in range(warmup):
        eng.process(x[i % 3], w["n_out"], out=y)
    eng.synchronize()
    eng.timer_start()
    for i in range(steps):
        eng.process(x[i % 3], w["n_out"], out=y)
    step_ms = eng.timer_stop() / steps
    eng.profile_begin()
    for i in range(steps):
        eng.process(x[i % 3], w["n_out"], out=y)
    prof = eng.profile_end()
    return {"step_ms": step_ms, "kernel_ms": {k: v[0] / max(v[1], 1) for k, v in prof.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", required=True, help="the library as built")
    ap.add_argument("--probe-lib", required=True, help="the same sources built with -DB200S_SYNTH_PROBES")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to DIR/synth_probes.jsonl")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(child(args.lib, args.steps, args.warmup)))
        return
    variants = [("as built", args.lib, None)] + [("probe %d" % p, args.probe_lib, p) for p in range(1, 5)]
    for r in range(args.rounds):
        for name, lib, probe in variants:
            env = dict(os.environ)
            env.pop("B200S_SYNTH_PROBE", None)
            if probe is not None:
                env["B200S_SYNTH_PROBE"] = str(probe)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--lib", lib, "--probe-lib", args.probe_lib,
                                "--steps", str(args.steps), "--warmup", str(args.warmup)], env=env, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit("%s failed:\n%s%s" % (name, p.stdout, p.stderr))
            res = json.loads(p.stdout.strip().splitlines()[-1])
            res.update(round=r, variant=name, log=[l for l in p.stderr.splitlines() if l.startswith("k_synth2")])
            line = json.dumps(res)
            print(line, flush=True)
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                with open(os.path.join(args.out, "synth_probes.jsonl"), "a") as f:
                    f.write(line + "\n")


if __name__ == "__main__":
    main()
