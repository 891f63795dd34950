"""Every kernel path on the GPU held to the exact answer.  `pytest -m gpu` on an H100.

In exact arithmetic (tuning key 3 = 1) the GPU computes what the emulator's float build computes, bit for bit
(tests/test_gpu_stages.py B), and the emulator is bit-exact against the oracle but for the FFT.  The emulator does not
model what can only go wrong on the device: cp.async, the bulk copies and the mbarriers are synchronous copies there,
static shared memory starts zeroed and the threads of a block run in one fixed interleaving.  A missing wait or fence,
a wrong parity, a read of uninitialised shared memory or a warp-synchronous assumption therefore shows up only on the
GPU, and there only as a small output difference that the phase chain's chaos can hide inside a median tolerance.  So:

A. Path matrix: each row runs a few streams through three calls (an odd one of one to two blocks, then 32 and 40
   blocks: state carried across calls, a second group of 32 frames in the last) on the GPU and on the emulator's float
   build in exact arithmetic, and compares the output of every call and the exported state after every call bit for bit.
   The same rows with the host pipeline split into stream groups (no commit fork beside the synthesis) too.
B. Batch scale: the benchmark's shape (1024 stereo streams, presetDefault 0.8x, three 32-block calls), each of 16
   pool inputs at 64 lanes -- the first and last lanes and both sides of every sub-batch boundary among them.  Every
   copy of a pool member is bit-identical to every other in fast and in exact arithmetic, and in exact arithmetic
   every member equals the emulator's run of it, with and without sub-batches.
C. The fast chain arithmetic (the default, SFU approximations, fused multiply-adds) against the exact one over a step
   or three from the same imported state, per bin, for every fast chain kernel the presets reach.

At the default tuning the shipped library and the emulator build (-DB200S_KEEP_OLD_KERNELS) dispatch the same kernels
for every row here: the two builds differ only for the forced scalar FFT at 3072 / 2560 (tuning key 1) and for chain
generations 1, 3 and 5 (tuning key 0), which no row selects (engine.cu analyse_kernel, synth_kernel, chain_kernel_for,
chain_version).
"""
import os
import time

import numpy as np
import pytest

import signals
import stages

pytestmark = pytest.mark.gpu

STATE_KEYS = ("history", "input", "prevInput", "output", "predEnergy", "pending", "pendingWp")
FLT_MIN = float(np.finfo(np.float32).tiny)


@pytest.fixture(scope="module")
def engines(cuda_lib, emu_libs):
    import torch

    assert torch.cuda.is_available(), "these tests need a GPU"
    from signalsmith_stretch_b200 import BatchStretch

    return {"gpu": lambda S, seed=0: BatchStretch(S, seed=seed),
            "emu": lambda S, seed=0: BatchStretch(S, seed=seed, lib_path=emu_libs["float"])}


def _inputs(S, C, n, sr):
    """S streams of the harmonic fixture; the last one at int16 level, and for stereo the one before it loud in channel
    0 and at 1e-20 in the others (energies below FLT_MIN)."""
    x = signals.batch("harmonic", S, C, n, sr)
    x[S - 1] = signals.edge("harmonic_32768", 1, C, n, sr)[0]
    if C == 2:
        x[S - 2] = signals.edge("loud_and_tiny", 1, C, n, sr)[0]
    return x


def _calls(H, ratio, blocks):
    """(input samples, output samples) per call: output lengths in blocks of H (a float adds 37 samples: an odd
    length), inputs keeping the ratio over the whole run."""
    res, o, i = [], 0, 0
    for b in blocks:
        n_out = int(b * H) + (37 if isinstance(b, float) else 0)
        o += n_out
        n_in = int(round(o / ratio)) - i
        i += n_in
        res.append((n_in, n_out))
    return res


A_BLOCKS = (1.0, 32, 40)  # H + 37 samples, 32 blocks, 40 blocks


def _drive(e, x, calls):
    """Host-API calls; the output of every call and the exported state after it."""
    outs, states, pos = [], [], 0
    for n_in, n_out in calls:
        outs.append(np.array(e.process(np.ascontiguousarray(x[:, :, pos:pos + n_in]), n_out)))
        pos += n_in
        states.append({k: np.array(e.get_state(k)) for k in STATE_KEYS})
    return outs, states


def _assert_bits(what, k, got, want):
    """Bit equality of [S][C][...] arrays; on a mismatch the first differing stream, channel and bin / sample."""
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert g.shape == w.shape, (what, k, g.shape, w.shape)
    gu, wu = g.view(np.uint32), w.view(np.uint32)
    if np.array_equal(gu, wu):
        return
    bad = np.argwhere(gu != wu)
    s, c, i = (int(v) for v in bad[0][:3])
    unit, at = ("bin", i // 2) if np.iscomplexobj(g) else ("sample" if what == "output audio" else "index", i)
    raise AssertionError("%s, call %d: first difference at stream %d, channel %d, %s %d: GPU %r, emulator %r (%d of %d words differ)"
                         % (what, k, s, c, unit, at, g[s, c, at], w[s, c, at], len(bad), gu.size))


def _check_audible(outs, x):
    y = np.concatenate(outs, axis=-1)
    assert np.all(np.isfinite(y)), "non-finite output"
    for s in range(y.shape[0]):
        assert np.abs(y[s]).max() > 1e-3 * np.abs(x[s]).max(), "stream %d is silent" % s


# ------------------------------------------------------------------ A. path matrix, exact mode, GPU against the emulator
def _stereo(o, sr=48000.0):
    o.presetDefault(2, sr)


def _row6(idx):
    """Per stream, by its index in the batch, cycling: plain, +3 st with an 8 kHz tonality limit, +3 st formants (base
    200 Hz), plain."""
    def cfg(o):
        o.presetDefault(2, 48000.0)
        k = np.asarray(idx) % 4
        o.setTransposeSemitones(np.where(k == 1, 3, 0).astype(np.float32), np.where(k == 1, 8000 / 48000, 0).astype(np.float32))
        o.setFormantSemitones(np.where(k == 2, 3, 0).astype(np.float32), np.zeros(len(k), bool))
        o.setFormantBase(np.full(len(k), 200 / 48000, np.float32))
    return cfg


def _cfg(*steps):
    def cfg(o):
        for name, args in steps:
            getattr(o, name)(*args)
    return cfg


# (id naming the kernels reached, configure(engine, the streams' indices in the batch), channels, sample rate, out/in ratio, streams, tuning, seed)
ROWS = [
    ("row1_config3_mono_+7st_k_energy_k_passes_k_prep_map_k_products_2groups_k_chain_t_3072",
     lambda o, idx: signals.cfg_config3(o), 1, 48000, 1.0, 6, (), 0),
    ("row2_config4_formant_comp_stereo_k_energy_k_passes_k_products_k_chain_t",
     lambda o, idx: signals.cfg_config4(o), 2, 48000, 1.0, 6, (), 0),
    ("row3_formant_auto_pitch_k_pitch",
     lambda o, idx: (signals.cfg_config4(o), o.setFormantBase(0)), 2, 48000, 1.0, 4, (), 0),
    ("row4_freq_map_folding_stereo_1.25x_3072_k_prep_map_k_products_k_chain_t",
     lambda o, idx: _cfg(("presetDefault", (2, 48000.0)), ("setFreqMapTable", signals.PWL_FOLDING))(o), 2, 48000, 1.25, 4, (), 0),
    ("row4_freq_map_monotone_mono_cheaper_2560_k_prep_map_k_products_k_chain_t",
     lambda o, idx: _cfg(("presetCheaper", (1, 48000.0)), ("setFreqMapTable", signals.PWL_MONOTONE))(o), 1, 48000, 1.0, 4, (), 0),
    ("row5_random_plain_stereo_2.5x_k_prep_random_k_chain",
     lambda o, idx: _stereo(o), 2, 48000, 2.5, 4, (), 20261015),
    ("row5_random_mapped_mono_cheaper_+4st_3x_k_products_k_prep_random_k_chain",
     lambda o, idx: _cfg(("presetCheaper", (1, 48000.0)), ("setTransposeSemitones", (4, 0)))(o), 1, 48000, 3.0, 4, (), 20261016),
    ("row6_mixed_stereo_0.8x_k_analyse2_mixed_k_chain_direct4_k_chain_t",
     lambda o, idx: _row6(idx)(o), 2, 48000, 0.8, 6, (), 0),
    ("row7_cheaper_stereo_split_1.5x_k_chain_direct4_L3_k_synth2_2560",
     lambda o, idx: o.presetCheaper(2, 48000.0), 2, 48000, 1.5, 4, (), 0),
    ("row8_96k_stereo_0.8x_k_analyse0_k_synth0_6144_k_chain_direct2_multiwarp",
     lambda o, idx: _stereo(o, 96000.0), 2, 96000, 0.8, 4, (), 0),
    ("row8_88k_mono_+5st_k_analyse0_k_synth0_6144_k_energy_k_products_k_chain_t",
     lambda o, idx: _cfg(("presetDefault", (1, 88200.0)), ("setTransposeSemitones", (5, 0)))(o), 1, 88200, 1.0, 4, (), 0),
    ("row9_mono_44k_plain_k_chain_direct2_3072",
     lambda o, idx: o.presetDefault(1, 44100.0), 1, 44100, 1.25, 5, ((5, 0),), 0),
    ("row9_mono_44k_plain_pairs_k_chain_direct6_dual_lone_stream",
     lambda o, idx: o.presetDefault(1, 44100.0), 1, 44100, 1.25, 5, ((5, 1),), 0),
]
ROW_IDS = [r[0] for r in ROWS]
# Row 10: rows 1, 2 and 6 with the host-buffer pipeline in three stream groups (tuning key 2; host calls split when every
# group has at least two streams).  Each group then runs its kernels on its own CUDA stream, and k_commit follows the
# synthesis on that stream instead of running forked beside it.  The emulator's side is the same as for the unsplit row.
SUB_ROWS = [r for r in ROWS if r[0].startswith(("row1_", "row2_", "row6_"))]
SUB_GROUPS = 3


def _run_row(make, row, tuning=(), lo=0, hi=None):
    """Row `row` on streams lo..hi of its batch (every stream is independent of the others, and every stream's random
    generator starts from the engine's seed, so a slice of the batch computes what the whole batch does on it)."""
    name, cfg, C, sr, ratio, S, row_tuning, seed = row
    hi = S if hi is None else hi
    e = make(hi - lo, seed)
    cfg(e, np.arange(lo, hi))
    e.set_tuning(3, 1)
    for key, value in tuple(row_tuning) + tuple(tuning):
        e.set_tuning(key, value)
    calls = _calls(e.intervalSamples(), ratio, A_BLOCKS)
    x = _inputs(S, C, sum(c[0] for c in calls), sr)[lo:hi]
    t0 = time.perf_counter()
    res = _drive(e, x, calls)
    return res, x, time.perf_counter() - t0


def _emu_row_stream(lib, row_id, s):
    """(worker process) one stream of a row on the emulator"""
    from signalsmith_stretch_b200 import BatchStretch

    t0 = time.process_time()
    (outs, states), _, _ = _run_row(lambda S, seed: BatchStretch(S, seed=seed, lib_path=lib), ROWS[ROW_IDS.index(row_id)], (), s, s + 1)
    return outs, states, time.process_time() - t0


def _emu_pool_stream(lib, mixed, p):
    """(worker process) pool member p of part B on the emulator"""
    from signalsmith_stretch_b200 import BatchStretch

    t0 = time.process_time()
    emu = BatchStretch(1, lib_path=lib)
    _b_cfg(mixed, np.array([p]))(emu)
    emu.set_tuning(3, 1)
    calls = _calls(emu.intervalSamples(), 0.8, B_CALLS)
    x = _inputs(B_POOL, 2, sum(c[0] for c in calls), 48000)[p:p + 1]
    outs, _ = _drive(emu, x, calls)
    return outs, None, time.process_time() - t0


@pytest.fixture(scope="module")
def emu_runs(request, emu_libs):
    """The emulator's side of the selected cases of parts A and B, one stream per job over the CPUs this process may use
    (the emulator runs a launch on one core), all submitted up front: {row id or ("B", mixed): futures of the streams in
    order}."""
    import concurrent.futures
    import multiprocessing

    wanted = []
    for item in request.session.items:
        params = getattr(getattr(item, "callspec", None), "params", {})
        key = params["row"][0] if "row" in params else ("B", params["mixed"]) if "mixed" in params else None
        if item.module is request.module and key is not None and key not in wanted:
            wanted.append(key)
    lib = emu_libs["float"]
    pool = concurrent.futures.ProcessPoolExecutor(max_workers=_usable_cpus(), mp_context=multiprocessing.get_context("spawn"))
    jobs = {}
    for key in wanted:
        if isinstance(key, tuple):
            jobs[key] = [pool.submit(_emu_pool_stream, lib, key[1], p) for p in range(B_POOL)]
        else:
            jobs[key] = [pool.submit(_emu_row_stream, lib, key, s) for s in range(ROWS[ROW_IDS.index(key)][5])]
    yield jobs
    pool.shutdown(wait=True, cancel_futures=True)


def _usable_cpus():
    """The CPUs this process may use: its affinity mask, capped by a cgroup CPU quota (os.cpu_count() counts every
    logical CPU of the host)."""
    n = len(os.sched_getaffinity(0))
    try:  # cgroup v2
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(per) + 0.5)))
    except (OSError, ValueError):
        pass
    return n


def _gather(futures):
    """Outputs (and states) of the streams' jobs joined into one batch; the emulator's CPU time over them."""
    res = [f.result() for f in futures]
    outs = [np.concatenate([r[0][k] for r in res]) for k in range(len(res[0][0]))]
    states = None if res[0][1] is None else [{key: np.concatenate([r[1][k][key] for r in res]) for key in STATE_KEYS} for k in range(len(res[0][1]))]
    return outs, states, sum(r[2] for r in res)


def _compare_row(engines, emu_runs, row, tuning=()):
    (go, gs), x, tg = _run_row(engines["gpu"], row, tuning)
    mo, ms, tm = _gather(emu_runs[row[0]])
    _check_audible(go, x)
    for k in range(len(go)):
        _assert_bits("output audio", k, go[k], mo[k])
        for key in STATE_KEYS:
            _assert_bits(key, k, gs[k][key], ms[k][key])
    print("%s: GPU %.2f s, emulator %.1f s of CPU time" % (row[0], tg, tm))


@pytest.mark.parametrize("row", ROWS, ids=ROW_IDS)
def test_path_bit_identical_to_emulator(engines, emu_runs, row):
    _compare_row(engines, emu_runs, row)


@pytest.mark.parametrize("row", SUB_ROWS, ids=["row10_stream_groups_" + r[0] for r in SUB_ROWS])
def test_path_in_stream_groups_bit_identical_to_emulator(engines, emu_runs, row):
    _compare_row(engines, emu_runs, row, ((2, SUB_GROUPS),))


# ------------------------------------------------------------------ B. batch scale: every lane of the benchmark's shape
B_STREAMS, B_POOL, B_SUB = 1024, 16, 4
B_CALLS = (32, 32, 32)


def _lanes(S, P):
    """Pool member of every lane: each aligned run of P lanes holds every member once (7 is odd, so 7 * lane runs over
    every residue mod P within a run) in an order that shifts from run to run.  The first and the last P lanes and the P
    lanes either side of every sub-batch boundary (multiples of S / B_SUB, themselves multiples of P) hold them all."""
    lane = np.arange(S)
    return (7 * lane + lane // P) % P


def _b_cfg(mixed, members):
    """presetDefault stereo; mixed: pool member p with the row-6 kind of index p, at every lane that holds it."""
    def cfg(o):
        if mixed:
            _row6(members)(o)
        else:
            o.presetDefault(2, 48000.0)
    return cfg


def _gpu_batch(make, mixed, exact, sub, lanes, pool_x, calls):
    """The batch through the device API (as bench.py runs it); returns the outputs of the pool members' first lanes,
    after checking every other lane against them bit for bit."""
    import torch

    e = make(len(lanes))
    _b_cfg(mixed, lanes)(e)
    e.set_tuning(3, int(exact))
    if sub > 1:
        e.set_sub_batches(sub)
    xp = torch.from_numpy(pool_x).cuda()
    idx = torch.from_numpy(lanes).cuda()
    first = np.array([int(np.flatnonzero(lanes == p)[0]) for p in range(pool_x.shape[0])])
    outs, pos = [], 0
    t0 = time.perf_counter()
    for k, (n_in, n_out) in enumerate(calls):
        y = e.process(xp[idx, :, pos:pos + n_in].contiguous(), n_out)
        pos += n_in
        yi = y.view(torch.int32)
        same = (yi == yi[torch.from_numpy(first[lanes]).cuda()]).flatten(1).all(dim=1).cpu().numpy()
        if not same.all():
            lane = int(np.flatnonzero(~same)[0])
            raise AssertionError("%s %s, sub-batches %d, call %d: lane %d differs from lane %d, its pool member %d's first copy "
                                 "(%d lanes differ)" % ("exact" if exact else "fast", "mixed" if mixed else "plain", sub, k, lane,
                                                        first[lanes[lane]], lanes[lane], int((~same).sum())))
        outs.append(y[torch.from_numpy(first).cuda()].cpu().numpy())
        del y, yi
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    e.close()
    return outs, dt


@pytest.mark.parametrize("mixed", [False, True], ids=["plain_k_analyse2_persistent_k_chain_direct4", "mixed_k_analyse2_mixed_k_products_k_chain_t"])
def test_batch_scale_every_lane(engines, emu_runs, mixed):
    """1024 stereo streams, 48 kHz presetDefault 0.8x, three 32-block calls: about 65,000 k_analyse2 items over 2 CTAs per
    SM, so every persistent CTA runs hundreds of items (mbarrier phases, staging buffers reused).  Plain: the benchmark's
    call; mixed: the pool members carry the row-6 kinds."""
    e = engines["gpu"](1)
    e.presetDefault(2, 48000.0)
    calls = _calls(e.intervalSamples(), 0.8, B_CALLS)
    pool_x = _inputs(B_POOL, 2, sum(c[0] for c in calls), 48000)
    ref, _, tm = _gather(emu_runs[("B", mixed)])
    _check_audible(ref, pool_x)
    lanes = _lanes(B_STREAMS, B_POOL)
    times = {}
    for exact in (True, False):
        for sub in (1, B_SUB):
            outs, times[(exact, sub)] = _gpu_batch(engines["gpu"], mixed, exact, sub, lanes, pool_x, calls)
            if exact:
                for k, (g, m) in enumerate(zip(outs, ref)):
                    _assert_bits("output audio (sub-batches %d)" % sub, k, g, m)
    print("batch scale %s: emulator %.1f s of CPU time; GPU %s" % ("mixed" if mixed else "plain", tm,
                                                      ", ".join("%s/%d sub %.2f s" % ("exact" if ex else "fast", sb, t) for (ex, sb), t in times.items())))


# ------------------------------------------------------------------ C. fast against exact chain arithmetic, a step at a time
# Per stream-channel, relative as in tests/stages.py (_rel), over the "output" spectra and predEnergy after a one-block call
# and a two-block call, both engines starting from the same state.
#   Emulator (rcp / rsqrt / sqrt correctly rounded): <= 1.9e-7 rms, <= 2.5e-7 max over the five cases.
#   H100 (NVIDIA H100 80GB HBM3, 700 W power limit; SFU approximations): <= 2.2e-7 rms, <= 2.8e-7 max, the largest at
#   96 kHz.  The gates are about 4x that: a wrong term order, a dropped fused term or a bad scaling fails them.
FAST_RMS = 1e-6
FAST_MAX = 1.2e-6

# (id naming the fast kernel, configure, channels, sample rate, tuning key 5)
FAST_CASES = [
    ("k_chain_direct4_L4_stereo_default", lambda o: o.presetDefault(2, 48000.0), 2, 48000, 0),
    ("k_chain_direct4_L3_stereo_cheaper", lambda o: o.presetCheaper(2, 48000.0), 2, 48000, 0),
    ("k_chain_direct2_mono_default", lambda o: o.presetDefault(1, 48000.0), 1, 48000, 0),
    ("k_chain_direct6_dual_mono_default_pair_and_lone", lambda o: o.presetDefault(1, 48000.0), 1, 48000, 1),
    ("k_chain_direct2_mono_96k", lambda o: o.presetDefault(1, 96000.0), 1, 96000, 0),
]
FAST_LEVELS = {"harmonic": 1.0, "int16": 32768.0}


def _fast_inputs(C, n, sr, level, tiny_from):
    """Streams 0 and 1 at the level; stream 2 reaches energies below FLT_MIN in most bins.  Stereo: int16 level in channel
    0, 1e-20 in channel 1.  Mono: the harmonic fixture at the level, down to 1e-20 from sample tiny_from on (a stream at 1e-20 all
    along would be silent, and the silence bypass would leave every bin zero)."""
    x = signals.batch("harmonic", 3, C, n, sr) * np.float32(level)
    if C == 2:
        x[2] = signals.edge("loud_and_tiny", 1, C, n, sr)[0]
    else:
        x[2, :, tiny_from:] *= np.float32(1e-20 / level)
    return x.astype(np.float32)


@pytest.mark.parametrize("level", list(FAST_LEVELS), ids=list(FAST_LEVELS))
@pytest.mark.parametrize("name,cfg,C,sr,dual", FAST_CASES, ids=[c[0] for c in FAST_CASES])
def test_fast_chain_per_bin_vs_exact(engines, name, cfg, C, sr, dual, level):
    """An exact engine warmed up over several calls exports its three streams; a fast and an exact engine import them and
    take the same one-block call, then the same two-block call.  Per stream-channel the fast output spectra and predicted
    energies stay within FAST_RMS / FAST_MAX of the exact ones wherever the channel carries signal; every fast bin is
    finite, and a fast bin is zero exactly where the exact bin is zero or its energy is subnormal (sqrt_fast flushes a
    subnormal energy to zero, kernels.cuh)."""
    make = engines["gpu"]
    warm = make(3)
    cfg(warm)
    warm.set_tuning(3, 1)
    warm.set_tuning(5, dual)
    H, B = warm.intervalSamples(), warm.blockSamples()
    warm_calls = _calls(H, 1.0, (1.0, 7, 12))
    calls = _calls(H, 1.0, (1, 2))
    n_warm = sum(c[0] for c in warm_calls)
    # (mono: the windows of the compared blocks lie within the quiet end, which stays shorter than the 2 blocks of quiet
    # input after which a stream counts as silent)
    x = _fast_inputs(C, n_warm + sum(c[0] for c in calls), sr, FAST_LEVELS[level], n_warm - B)
    _drive(warm, x, warm_calls)
    rec = warm.export_streams([0, 1, 2])
    runs = []
    for exact in (1, 0):
        e = make(3)
        cfg(e)
        e.set_tuning(3, exact)
        e.set_tuning(5, dual)
        e.import_streams([0, 1, 2], rec)
        runs.append(_drive(e, np.ascontiguousarray(x[:, :, n_warm:]), calls)[1])
    worst = {"output": [0.0, 0.0], "predEnergy": [0.0, 0.0]}
    flushed = 0  # bins whose exact value is nonzero while their energy is subnormal: the edge of sqrt_fast
    for k, (ex, fa) in enumerate(zip(*runs)):
        assert not np.array_equal(ex["output"], fa["output"]), "call %d: fast and exact identical (fast mode not in use?)" % k
        xo, fo = ex["output"], fa["output"]
        assert np.all(np.isfinite(fo.view(np.float32))), "call %d: non-finite fast bins" % k
        # the energy each bin's output was made with (Prediction::energy of the call's last block); it rounds a little
        # differently in the two modes, so no claim is made within 1 % of FLT_MIN
        en = ex["predEnergy"].astype(np.float64)
        zero = fo == 0
        must_zero = (xo == 0) | (en < FLT_MIN * 0.99)
        must_live = (xo != 0) & (en > FLT_MIN * 1.01)
        flushed += int(((xo != 0) & (en < FLT_MIN * 0.99)).sum())
        assert np.all(zero[must_zero]), "call %d: %d fast bins nonzero where the exact bin is zero or its energy subnormal" % (k, int((~zero & must_zero).sum()))
        assert not np.any(zero[must_live]), "call %d: %d fast bins zero where the exact bin is not and its energy is normal" % (k, int((zero & must_live).sum()))
        # the error gate on the channels that carry signal (the 1e-20 channels sit at the subnormal edge throughout)
        live = np.sqrt(np.mean(en, axis=-1)) > 1e-10
        for key in ("output", "predEnergy"):
            d, r = fa[key] - ex[key], ex[key]
            if key == "output":
                d = np.where(must_live, d, 0)
            er, em = stages._rel(d, r, "rms")[live], stages._rel(d, r, "max")[live]
            worst[key] = [max(worst[key][0], float(er.max())), max(worst[key][1], float(em.max()))]
            assert er.max() <= FAST_RMS and em.max() <= FAST_MAX, (k, key, float(er.max()), float(em.max()))
    assert flushed > 0, "no bin reached a subnormal energy with a nonzero exact value: the flush-to-zero edge went untested"
    print("%s %s: fast vs exact, output rms %.2e max %.2e, predEnergy rms %.2e max %.2e; %d bins at the subnormal edge"
          % (name, level, *worst["output"], *worst["predEnergy"], flushed))
