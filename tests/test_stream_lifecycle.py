"""Per-stream operations (b200s_run_per_stream*): in one call every stream processes, seeks, output-seeks, flushes, resets
or sits the call out, each with its own counts.

Under the CPU emulator (exact arithmetic, the oracle's FFT swapped in) every stream must be bit-identical to its own
one-stream oracle that calls the reference methods its ops name, in the same order, and nothing for its SKIP calls.  On
the H100 (-m gpu) every stream must be bit-identical to the same stream driven through the batch-wide calls, the exact
mode must equal the emulator's float build, the calls must allocate nothing after reserve(), and chained asynchronous
calls must equal synchronous ones.
"""
import ctypes

import numpy as np
import pytest

import signals

SR = 48000.0
PLAIN = (0, 0, 0, False, 0)
SKIP, PROC, SEEK, OSEEK, FLUSH, RESET = range(6)
STATE_NAMES = ("input", "prevInput", "output", "predEnergy", "history", "pending", "pendingWp")


def rms(a):
    return float(np.sqrt(np.mean(np.square(a, dtype=np.float64))))


def _emu(path, batch, seed=321, exact_math=True):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=seed, lib_path=path)
    e.set_tuning(3, 1 if exact_math else 0)
    return e


def _set_batch(e, prm):
    semis, ton, fsemi, comp, base = (np.array(v) for v in zip(*prm))
    e.setTransposeSemitones(semis.astype(np.float32), ton.astype(np.float32))
    e.setFormantSemitones(fsemi.astype(np.float32), comp.astype(bool))
    e.setFormantBase(base.astype(np.float32))


def _set_one(o, p):
    o.setTransposeSemitones(p[0], p[1])
    o.setFormantSemitones(p[2], p[3])
    o.setFormantBase(p[4])


def _oracle():
    from oracle.hdrref import CpuStretch

    return CpuStretch("orc", 321)


def _norm(script):
    """script: per call, per stream (op, n_in, n_out, rate) with n_in / n_out / rate optional."""
    return [[tuple(list(t) + [0] * (4 - len(t))) for t in call] for call in script]


def _calls(x, script, pad=4, fill=0.75):
    """Per call: (ops, [S][C][stride] input slab, n_in, n_out, rates); stream s's inputs are consecutive pieces of x[s]."""
    S, C = x.shape[:2]
    pos = np.zeros(S, int)
    out = []
    for call in script:
        ops = np.array([t[0] for t in call], np.int32)
        n_in = np.array([t[1] for t in call], np.int32)
        n_out = np.array([t[2] for t in call], np.int32)
        rates = np.array([t[3] for t in call], np.float64)
        stride = (int(n_in.max()) + pad + 3) // 4 * 4
        buf = np.full((S, C, stride), fill, np.float32)
        for s in range(S):
            buf[s, :, :n_in[s]] = x[s, :, pos[s]:pos[s] + n_in[s]]
        pos += n_in
        out.append((ops, buf, n_in, n_out, rates))
    assert np.all(pos <= x.shape[-1])
    return out


def _run(g, x, script, out_pad=0):
    """Drive a batch engine with run(); returns, per stream, the list of outputs of its PROCESS / FLUSH calls, and checks
    that every sample an op does not produce is zero."""
    S = x.shape[0]
    ys = [[] for _ in range(S)]
    for ops, buf, n_in, n_out, rates in _calls(x, script):
        C = buf.shape[1]
        out = np.full((S, C, int(n_out.max()) + out_pad), np.nan, np.float32)
        y = np.array(g.run(ops, buf, n_out, inputSamples=n_in, playbackRates=rates, out=out))
        for s in range(S):
            assert not np.any(y[s, :, n_out[s]:]), "stream %d: the output tail is not zero" % s
            if ops[s] in (PROC, FLUSH):
                ys[s].append(y[s, :, :n_out[s]])
    return ys


def _drive_oracle(o, xs, script, s):
    outs, pos = [], 0
    for call in script:
        op, n_in, n_out, rate = call[s]
        seg = xs[:, pos:pos + n_in]
        pos += n_in
        if op == PROC:
            outs.append(o.process(seg, int(n_out)))
        elif op == SEEK:
            o.seek(seg, rate)
        elif op == OSEEK:
            o.outputSeek(seg)
        elif op == FLUSH:
            outs.append(o.flush(int(n_out), float(np.float32(rate))))
        elif op == RESET:
            o.reset()
    return outs


def _check_vs_oracles(ys, cfg, prm, x, script):
    for s in range(len(ys)):
        o = _oracle()
        cfg(o)
        _set_one(o, prm[s])
        ref = _drive_oracle(o, x[s], script, s)
        assert len(ys[s]) == len(ref)
        for k, (a, b) in enumerate(zip(ys[s], ref)):
            assert a.shape == b.shape, (s, k, a.shape, b.shape)
            assert np.array_equal(a, b), "stream %d, output %d: max diff %g" % (s, k, np.abs(a - b).max())


# ------------------------------------------------------------------ CPU emulator, against the oracle
SIX_PRM = [PLAIN, (3, 0.25, 0, False, 0), PLAIN, (0, 0, 3, False, 0), PLAIN, (-5, 0, 0, True, 200 / SR)]
# configure(2, 512, 128): inputLatency 256, outputLatency 256
# one row per call, one column per stream: s0 output-seeks, processes, flushes at rate 1 (n > interval), output-seeks
# again | s1 runs of SKIP | s2 seeks at a slow rate (random path) | s3 (formants) flushes at rate 0, later tail only |
# s4 resets mid-stream | s5 (mapped + formant compensation) turns over
SIX_SCRIPT = _norm([
    [(OSEEK, 600), (PROC, 400, 320), (SEEK, 640, 0, 0.3), (PROC, 401, 320), (PROC, 400, 320), (PROC, 640, 320)],
    [(PROC, 400, 320), (SKIP,), (PROC, 100, 320), (PROC, 398, 333), (PROC, 300, 300), (PROC, 600, 300)],
    [(PROC, 420, 336), (SKIP,), (PROC, 90, 300), (FLUSH, 0, 300, 0.0), (PROC, 260, 320), (FLUSH, 0, 500, 1.0)],
    [(PROC, 350, 280), (PROC, 400, 320), (PROC, 120, 350), (PROC, 402, 290), (RESET,), (OSEEK, 700)],
    [(FLUSH, 0, 450, 1.0), (SKIP,), (PROC, 100, 320), (FLUSH, 0, 100, 0.5), (PROC, 300, 300), (PROC, 500, 250)],
    [(OSEEK, 700), (PROC, 300, 240), (SKIP,), (PROC, 401, 320), (PROC, 300, 300), (PROC, 640, 320)],
    [(PROC, 400, 320), (SKIP,), (PROC, 130, 325), (PROC, 400, 320), (SKIP,), (PROC, 640, 320)],
    [(PROC, 400, 320), (PROC, 420, 336), (PROC, 100, 250), (SKIP,), (PROC, 200, 320), (PROC, 640, 320)],
])


def _six_inputs():
    x = signals.batch("harmonic", 6, 2, 6000, 48000)
    return x


def test_six_streams_with_own_ops_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Output seeks, flushes at rate 1 and 0, a tail-only flush, runs of SKIP, a slow seek that reaches the random path, a
    reset mid-stream, mapped and formant streams turning over: the ops change every call."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    x = _six_inputs()
    g = _emu(emu_libs["exact"], 6)
    cfg(g)
    _set_batch(g, SIX_PRM)
    ys = _run(g, x, SIX_SCRIPT, out_pad=5)
    assert g.unserved_random_blocks() == 0
    _check_vs_oracles(ys, cfg, SIX_PRM, x, SIX_SCRIPT)


def test_stereo_preset_turnover_bit_exact_vs_oracle(emu_libs, oracle_port):
    """presetDefault stereo, 32-block calls (k_analyse2<3072>, the packed chain, k_synth2), a few streams turning over."""
    cfg = lambda o: o.presetDefault(2, 48000.0)  # noqa: E731
    H = 1440
    n = 32 * H
    ni = int(round(n / 0.8))
    prm = [PLAIN, PLAIN, (4, 8000 / SR, 0, False, 0), PLAIN]
    script = _norm([
        [(PROC, ni, n), (FLUSH, 0, 6 * H, 1.25), (OSEEK, 7000), (PROC, ni, n)],
        [(PROC, ni, n), (OSEEK, 6049), (PROC, ni, n), (SKIP,)],
        [(PROC, ni, n), (PROC, ni, n), (PROC, ni, n), (PROC, ni, n)],
    ])
    x = signals.batch("harmonic", 4, 2, 4 * ni, 48000)
    g = _emu(emu_libs["exact"], 4)
    cfg(g)
    _set_batch(g, prm)
    ys = _run(g, x, script, out_pad=3)
    assert g.unserved_random_blocks() == 0
    _check_vs_oracles(ys, cfg, prm, x, script)


def test_cheaper_split_mono_turnover_bit_exact_vs_oracle(emu_libs, oracle_port):
    """presetCheaper mono with split computation: k_flush_tail and k_add_output read the ring at the split offset."""
    cfg = lambda o: o.presetCheaper(1, 48000.0)  # noqa: E731
    H = 1920
    script = _norm([
        [(PROC, 12 * H, 10 * H), (OSEEK, 9000), (PROC, 10 * H, 10 * H)],
        [(FLUSH, 0, 5 * H + 7, 1.0), (PROC, 8 * H, 6 * H), (OSEEK, 7001)],
        [(OSEEK, 8000), (FLUSH, 0, 3 * H, 0.0), (PROC, 9 * H, 8 * H)],
        [(PROC, 7 * H, 7 * H), (PROC, 5 * H, 5 * H), (FLUSH, 0, H - 5, 1.0)],
    ])
    x = signals.batch("harmonic", 3, 1, 40 * H, 48000)
    g = _emu(emu_libs["exact"], 3)
    cfg(g)
    ys = _run(g, x, script)
    assert g.unserved_random_blocks() == 0
    _check_vs_oracles(ys, cfg, [PLAIN] * 3, x, script)


def test_skip_leaves_the_state_byte_identical(emu_libs, oracle_port):
    """A skipped stream is absent: b200s_get_state returns the same bytes for it, for every `what`, and a later block that
    draws random factors (stream 0 stretches beyond 2x) still matches the oracle, so its random engine did not advance."""
    cfg = lambda o: o.configure(1, 512, 128)  # noqa: E731
    x = signals.batch("harmonic", 3, 1, 3000, 48000)
    g = _emu(emu_libs["exact"], 3)
    cfg(g)
    first = _norm([[(PROC, 120, 320), (PROC, 400, 400), (PROC, 300, 300)]])
    skips = _norm([[(SKIP,), (PROC, 400, 400), (SKIP,)], [(SKIP,), (OSEEK, 500), (FLUSH, 0, 300, 1.0)]])
    after = _norm([[(PROC, 130, 330), (PROC, 400, 400), (PROC, 300, 300)]])
    calls = _calls(x, first + skips + after)
    ys = [[] for _ in range(3)]

    def do(k):
        ops, buf, n_in, n_out, rates = calls[k]
        y = g.run(ops, buf, n_out, inputSamples=n_in, playbackRates=rates)
        for s in range(3):
            if ops[s] in (PROC, FLUSH):
                ys[s].append(y[s, :, :n_out[s]])

    do(0)
    before = {n: g.get_state(n) for n in STATE_NAMES}
    do(1)
    mid = {n: g.get_state(n) for n in STATE_NAMES}
    for n in STATE_NAMES:
        for s in (0, 2):
            assert before[n][s].tobytes() == mid[n][s].tobytes(), (n, s)
    do(2)
    for n in STATE_NAMES:
        assert before[n][0].tobytes() == g.get_state(n)[0].tobytes(), n
    do(3)
    assert g.unserved_random_blocks() == 0
    _check_vs_oracles(ys, cfg, [PLAIN] * 3, x, first + skips + after)


def test_output_seek_process_flush_equal_exact(emu_libs, oracle_port):
    """exact() per stream is OUTPUT_SEEK, PROCESS, FLUSH over three calls, each stream with its own lengths."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    S = 3
    n_in = [3000, 2600, 2000]
    n_out = [2400, 3900, 2000]
    x = signals.batch("harmonic", S, 2, max(n_in), 48000)
    g = _emu(emu_libs["exact"], S)
    cfg(g)
    seek, idx, rate = [], [], []
    for s in range(S):
        r = np.float32(n_in[s]) / np.float32(n_out[s])
        L = g.outputSeekLength(float(r))
        seek.append(L)
        idx.append(int(np.float32(n_out[s]) - np.float32(L) / r))
        rate.append(float(r))
    script = _norm([
        [(OSEEK, seek[s]) for s in range(S)],
        [(PROC, n_in[s] - seek[s], idx[s]) for s in range(S)],
        [(FLUSH, 0, n_out[s] - idx[s], rate[s]) for s in range(S)],
    ])
    ys = _run(g, x, script)
    for s in range(S):
        o = _oracle()
        cfg(o)
        ok, ref = o.exact(x[s][:, :n_in[s]], n_out[s])
        assert ok
        got = np.concatenate(ys[s], axis=-1)
        assert np.array_equal(got, ref), (s, np.abs(got - ref).max())


def test_all_process_equals_the_uniform_call(emu_libs):
    """Float emulator: run() with every op PROCESS and every stream at the call's lengths gives the uniform b200s_process
    call's output bit for bit, with the same kernel launches (five per call: plan, analyse, chain, synth, commit)."""
    S, C = 3, 2
    x = signals.batch("harmonic", S, C, 3000, 48000)
    outs, launches = [], []
    chunks = list(signals.chunks(x.shape[-1], 0.8, 500))
    for use_run in (False, True):
        g = _emu(emu_libs["float"], S, exact_math=False)
        g.configure(C, 512, 128)
        n0 = g.kernel_launches()
        ys = []
        for i, ci, co in chunks:
            a = np.ascontiguousarray(x[:, :, i:i + ci])
            ys.append(np.array(g.run(PROC, a, co) if use_run else g.process(a, co)))
        outs.append(np.concatenate(ys, axis=-1))
        launches.append(g.kernel_launches() - n0)
    assert np.array_equal(outs[0], outs[1])
    assert launches[0] == launches[1] == 5 * len(chunks)


def test_run_arguments_are_validated(emu_libs):
    """Every refused argument returns B200S_EINVAL before anything is enqueued, names the stream, and leaves every stream's
    state unchanged; Python refuses wrong shapes with ValueError."""
    from signalsmith_stretch_b200 import StretchError

    S, C = 3, 2
    g = _emu(emu_libs["float"], S)
    g.configure(C, 512, 128)
    g.process(signals.batch("harmonic", S, C, 600, 48000), 500)
    lib, h = g._lib, g._h
    ip, dp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)
    buf = np.zeros((S, C, 256), np.float32)
    out = np.zeros((S, C, 256), np.float32)
    rates = np.ones(S)

    def arr(v):
        return np.array(v, np.int32)

    state0 = {n: g.get_state(n) for n in STATE_NAMES}
    n0 = g.kernel_launches()
    ok_ops, ok_in, ok_out = arr([PROC, SEEK, FLUSH]), arr([100, 200, 0]), arr([100, 0, 200])
    for fn in ("b200s_run_per_stream", "b200s_run_per_stream_async", "b200s_run_per_stream_device"):
        f = getattr(lib, fn)
        A = lambda ops=ok_ops, ni=ok_in, no=ok_out, si=256, so=256, r=rates: f(  # noqa: E731
            h, None if ops is None else ops.ctypes.data_as(ip), buf.ctypes.data, si, None if ni is None else ni.ctypes.data_as(ip),
            out.ctypes.data, so, None if no is None else no.ctypes.data_as(ip), None if r is None else r.ctypes.data_as(dp))
        assert A(ops=None) == -1 and A(ni=None) == -1 and A(no=None) == -1
        assert A(si=-1) == -1 and A(so=-4) == -1
    cases = [  # (ops, n_in, n_out, rates, stream)
        ([PROC, 6, PROC], [1, 1, 1], [1, 1, 1], rates, 1),
        ([PROC, PROC, -1], [1, 1, 1], [1, 1, 1], rates, 2),
        ([PROC, SEEK, PROC], [1, 100, 1], [1, 0, 1], None, 1),
        ([FLUSH, PROC, PROC], [5, 1, 1], [300 - 44, 1, 1], rates, 0),
        ([PROC, RESET, PROC], [1, 3, 1], [1, 0, 1], rates, 1),
        ([PROC, PROC, SKIP], [1, 1, 2], [1, 1, 0], rates, 2),
        ([SEEK, PROC, PROC], [100, 1, 1], [9, 1, 1], rates, 0),
        ([PROC, OSEEK, PROC], [1, 100, 1], [1, 1, 1], rates, 1),
        ([PROC, RESET, PROC], [1, 0, 1], [1, 2, 1], rates, 1),
        ([PROC, PROC, SKIP], [1, 1, 0], [1, 1, 3], rates, 2),
        ([PROC, PROC, PROC], [1, 257, 1], [1, 1, 1], rates, 1),
        ([PROC, PROC, PROC], [1, 1, 1], [1, 1, -2], rates, 2),
        ([FLUSH, PROC, PROC], [0, 1, 1], [300, 1, 1], rates, 0),
    ]
    for ops, ni, no, r, stream in cases:
        o, a, b = arr(ops), arr(ni), arr(no)
        rc = lib.b200s_run_per_stream(h, o.ctypes.data_as(ip), buf.ctypes.data, 256, a.ctypes.data_as(ip), out.ctypes.data, 256,
                                      b.ctypes.data_as(ip), None if r is None else r.ctypes.data_as(dp))
        assert rc == -1, (ops, ni, no)
        assert ("stream %d" % stream) in lib.b200s_last_error(h).decode(), (ops, lib.b200s_last_error(h))
    assert g.kernel_launches() == n0  # nothing was enqueued
    for n in STATE_NAMES:
        assert state0[n].tobytes() == g.get_state(n).tobytes(), n
    with pytest.raises(StretchError, match="stream 1"):
        g.run_per_stream_host_ptr([PROC, RESET, PROC], buf.ctypes.data, 256, [0, 3, 0], out.ctypes.data, 256, [0, 0, 0], wait=True)
    for call in (lambda: g.run([PROC, PROC], buf, 10), lambda: g.run(7, buf, 10), lambda: g.run(PROC, buf, 10, playbackRates=[1, 2]),
                 lambda: g.run(PROC, buf, [10, 10, 10], inputSamples=[1, 2, 300])):
        with pytest.raises(ValueError):
            call()
    assert g.kernel_launches() == n0


def test_profile_keeps_six_kinds_unless_phases_are_asked_for(emu_libs):
    """profile_end() reports the six kernels; phases=True adds the pre and post phases of run()."""
    S, C = 2, 1
    g = _emu(emu_libs["float"], S)
    g.configure(C, 512, 128)
    x = signals.batch("harmonic", S, C, 600, 48000)
    for phases in (False, True):
        g.profile_begin()
        g.run([PROC, OSEEK], x, [500, 0])
        g.run([FLUSH, PROC], x, [300, 500], inputSamples=[0, 600])
        p = g.profile_end(phases=phases)
        assert set(p) == set(g.KERNELS) | ({"phases"} if phases else set())
        assert p["plan"][1] > 0
        if phases:
            assert p["phases"][1] > 0


# ------------------------------------------------------------------ H100
def _gpu_script(S, H, calls=3, seed=7, turnover=0.25):
    """presetDefault stereo: per call, a share of the slots turn over (FLUSH, then OUTPUT_SEEK next call), a few SKIP."""
    rng = np.random.default_rng(seed)
    n = 16 * H
    ni = int(round(n / 0.8))
    script, pending = [], set()
    for k in range(calls):
        call = []
        for s in range(S):
            if s in pending:
                call.append((OSEEK, 5000 + 13 * s))
                pending.discard(s)
            elif k > 0 and rng.random() < turnover:
                call.append((FLUSH, 0, 3 * H + s, 1.25))
                pending.add(s)
            elif rng.random() < 0.08:
                call.append((SKIP,))
            elif rng.random() < 0.08:  # a seek, every other one slow enough for random time factors (b200s_seek_rates)
                call.append((SEEK, 5760, 0, 0.3 if s % 2 else 1.25))
            elif rng.random() < 0.05:
                call.append((RESET,))
            else:
                call.append((PROC, ni - 4 * (s % 3), n - (s % 2)))
        script.append(call)
    return _norm(script)


def _batchwide(C, xs, script, s, exact_math=False):
    """Stream s alone, through the batch-wide calls (b200s_process / _flush / _output_seek / _seek_rates / _reset)."""
    from signalsmith_stretch_b200 import BatchStretch

    u = BatchStretch(1, seed=0)
    u.presetDefault(C, SR)
    if exact_math:
        u.set_tuning(3, 1)
    outs, pos = [], 0
    for call in script:
        op, n_in, n_out, rate = call[s]
        seg = xs[None, :, pos:pos + n_in]
        pos += n_in
        if op == PROC:
            outs.append(np.array(u.process(seg, int(n_out)))[0])
        elif op == SEEK:
            u.seek(seg, np.array([rate]))
        elif op == OSEEK:
            u.outputSeek(seg)
        elif op == FLUSH:
            outs.append(u.flush(int(n_out), float(rate))[0])
        elif op == RESET:
            u.reset()
    return outs


@pytest.mark.gpu
def test_turnover_batch_equals_batchwide_calls_on_the_gpu(cuda_lib, oracle_port):
    """24 stereo presetDefault streams, fast arithmetic, three calls with turnovers, skips and resets: each stream is
    bit-identical to the same stream driven through the batch-wide calls, and within the short-horizon tolerance of its
    oracle."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C, H = 24, 2, 1440
    script = _gpu_script(S, H)
    x = signals.batch("harmonic", S, C, 3 * 30000, 48000)
    g = BatchStretch(S)
    g.presetDefault(C, SR)
    ys = _run(g, x, script)
    assert g.unserved_random_blocks() == 0
    ops = {t[0] for call in script for t in call}
    assert {PROC, FLUSH, OSEEK, SKIP, SEEK} <= ops
    for s in range(S):
        ref = _batchwide(C, x[s], script, s)
        assert len(ref) == len(ys[s])
        for a, b in zip(ys[s], ref):
            assert np.array_equal(a, b), "stream %d: max diff %g" % (s, np.abs(a - b).max())
    # short horizon: the first output after the stream's start, an output seek or a reset (fast arithmetic drifts from the
    # oracle's over a long stream, as on the uniform path)
    per = []
    for s in range(S):
        o = oracle_port()
        o.presetDefault(C, SR)
        ref = _drive_oracle(o, x[s], script, s)
        fresh, k = True, 0
        for call in script:
            op = call[s][0]
            if op in (PROC, FLUSH):
                if fresh and op == PROC:
                    m = min(ys[s][k].shape[-1], g.outputLatency() + 6 * H)
                    per.append(rms(ys[s][k][:, :m] - ref[k][:, :m]))
                fresh, k = False, k + 1
            elif op in (OSEEK, RESET):
                fresh = True
    assert len(per) >= S // 2
    per = np.array(per)
    assert np.median(per) <= 1e-4, per
    assert per.max() <= 1e-3, per


@pytest.mark.gpu
def test_exact_mode_turnover_bit_identical_to_emulator(cuda_lib, emu_libs):
    """Exact arithmetic: a small turnover batch gives the emulator's float build bit for bit."""
    from signalsmith_stretch_b200 import BatchStretch

    H = 1440
    script = _norm([
        [(PROC, 14400, 12 * H), (OSEEK, 6000), (PROC, 9001, 7 * H + 1), (SKIP,)],
        [(FLUSH, 0, 4 * H, 1.0), (PROC, 8640, 8 * H), (SEEK, 5760, 0, 0.4), (PROC, 11520, 9 * H)],
        [(OSEEK, 7000), (PROC, 12000, 10 * H), (PROC, 4000, 9 * H), (FLUSH, 0, 2 * H, 0.0)],
    ])
    x = signals.batch("harmonic", 4, 2, 40000, 48000)
    outs = []
    for e in (BatchStretch(4), BatchStretch(4, lib_path=emu_libs["float"])):
        e.presetDefault(2, SR)
        e.set_tuning(3, 1)
        outs.append(_run(e, x, script, out_pad=2))
    for s in range(4):
        for a, b in zip(outs[0][s], outs[1][s]):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (s, np.abs(a - b).max())


@pytest.mark.gpu
def test_run_allocates_nothing_after_reserve(cuda_lib):
    """After reserve() with the strides, turnover calls whose flushes read at most in_stride zeros allocate nothing.  A
    flush at rate 0 stretches beyond 2x: like any call beyond 2x, its first one allocates the random path's rows, and
    later ones allocate nothing."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C = 16, 2
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    H = e.intervalSamples()
    in_stride, out_stride = 12 * H, 9 * H
    e.reserve(in_stride, out_stride)
    x = signals.batch("harmonic", S, C, in_stride, 48000)
    before = e.device_allocations()
    script = _gpu_script(S, H, calls=5, seed=3, turnover=0.3)
    for call in script:
        ops = np.array([t[0] for t in call])
        n_in = np.minimum([t[1] for t in call], in_stride)
        n_out = np.minimum([t[2] for t in call], out_stride)
        e.run(ops, x, n_out, inputSamples=n_in, playbackRates=1.0)
    e.synchronize()
    assert e.device_allocations() == before
    flush0 = np.where(np.arange(S) % 4 == 0, FLUSH, PROC)
    n_out0 = np.where(flush0 == FLUSH, 3 * H, 8 * H)
    n_in0 = np.where(flush0 == FLUSH, 0, 10 * H)
    e.run(flush0, x, n_out0, inputSamples=n_in0)  # rate 0 (NULL rates): the random path's rows, once
    e.synchronize()
    after_first = e.device_allocations()
    for k in range(3):
        e.run(np.roll(flush0, k + 1), x, np.roll(n_out0, k + 1), inputSamples=np.roll(n_in0, k + 1))
    e.synchronize()
    assert e.device_allocations() == after_first


@pytest.mark.gpu
def test_chained_async_run_calls_equal_synchronous_calls(cuda_lib):
    """Chained b200s_run_per_stream_async calls on pinned buffers, alternating turnover calls (which join) with
    PROCESS / SKIP calls (which chain), equal the synchronous calls bit for bit."""
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C, calls = 48, 2, 6
    rng = np.random.default_rng(11)
    e0 = BatchStretch(1)
    e0.presetDefault(C, SR)
    H = e0.intervalSamples()
    in_stride, out_stride = 10 * H, 8 * H
    plan = []
    for k in range(calls):
        if k % 2:
            ops = rng.choice([PROC, FLUSH, OSEEK, SKIP], S, p=[0.7, 0.1, 0.1, 0.1]).astype(np.int32)
        else:
            ops = rng.choice([PROC, SKIP], S, p=[0.8, 0.2]).astype(np.int32)
        n_in = np.where((ops == PROC) | (ops == OSEEK), rng.integers(0, in_stride + 1, S), 0).astype(np.int32)
        n_out = np.where((ops == PROC) | (ops == FLUSH), rng.integers(0, out_stride + 1, S), 0).astype(np.int32)
        plan.append((ops, n_in, n_out))
    x = signals.batch("harmonic", S, C, calls * in_stride, 48000)
    slabs = [np.ascontiguousarray(x[:, :, k * in_stride:(k + 1) * in_stride]) for k in range(calls)]
    sync = BatchStretch(S)
    sync.presetDefault(C, SR)
    ref = [sync.run(plan[k][0], slabs[k], plan[k][2], inputSamples=plan[k][1], playbackRates=1.0,
                    out=np.empty((S, C, out_stride), np.float32)) for k in range(calls)]
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    e.reserve(in_stride, out_stride)
    pin_in = [torch.from_numpy(slabs[k]).pin_memory() for k in range(calls)]
    pin_out = [torch.empty((S, C, out_stride), dtype=torch.float32).pin_memory() for _ in range(calls)]
    for k in range(calls):
        pin_out[k].fill_(float("nan"))
    for k in range(calls):
        e.run_per_stream_host_ptr(plan[k][0], pin_in[k].data_ptr(), in_stride, plan[k][1], pin_out[k].data_ptr(), out_stride, plan[k][2],
                                  playback_rates=1.0)
    e.synchronize()
    for k in range(calls):
        got = pin_out[k].numpy()
        assert np.array_equal(got, ref[k]), (k, np.nanmax(np.abs(got - ref[k])))
