"""Per-stream transpose / formant parameters (b200s_set_*_per_stream): one batch whose streams take different paths.

Under the CPU emulator (exact arithmetic, the oracle's FFT swapped in) every stream of a mixed batch must be bit-identical
to its own one-stream oracle configured with that stream's parameters.  On the H100 (-m gpu) every stream of a mixed batch
must be bit-identical to the same stream in a uniform batch with its parameters, and allocate nothing in process().
"""
import ctypes

import numpy as np
import pytest

import signals

SR = 48000.0


def rms(a):
    return float(np.sqrt(np.mean(np.square(a, dtype=np.float64))))


def _emu(path, batch, seed=0, exact_math=True, pairs=False, step_major=True):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=seed, lib_path=path)
    e.set_tuning(3, 1 if exact_math else 0)
    if pairs:
        e.set_tuning(5, 1)
    if not step_major:
        e.set_tuning(4, 0)
    return e


# per stream: (transpose semitones, tonality limit, formant semitones, formant compensation, formant base / sample rate)
PLAIN = (0, 0, 0, False, 0)
SIX = [
    PLAIN,
    (3, 0.25, 0, False, 0),
    (-5, 0, 0, False, 0),
    (12, 0, 0, True, 200 / SR),
    (5, 0, 0, True, 0),   # formant compensation, automatic pitch estimate
    (0, 0, 3, False, 0),  # formants +3 st without transposition (automatic pitch)
]


def _set_batch(e, prm):
    semis, ton, fsemi, comp, base = (np.array(v) for v in zip(*prm))
    e.setTransposeSemitones(semis.astype(np.float32), ton.astype(np.float32))
    e.setFormantSemitones(fsemi.astype(np.float32), comp.astype(bool))
    e.setFormantBase(base.astype(np.float32))


def _set_one(o, p):
    o.setTransposeSemitones(p[0], p[1])
    o.setFormantSemitones(p[2], p[3])
    o.setFormantBase(p[4])


def _oracles(make, cfg, prm, x, ratio, chunk):
    outs = []
    for s, p in enumerate(prm):
        o = make()
        cfg(o)
        _set_one(o, p)
        outs.append(signals.run_single(o, x[s], ratio, chunk))
    return np.stack(outs)


def _check(y, ref):
    for s in range(ref.shape[0]):
        assert np.array_equal(y[s], ref[s]), "stream %d: max diff %g" % (s, np.abs(y[s] - ref[s]).max())


# ------------------------------------------------------------------ CPU emulator, against the oracle
@pytest.mark.parametrize("ratio", [1.0, 0.8])
def test_six_paths_in_one_small_stereo_batch_bit_exact_vs_oracle(emu_libs, oracle_port, ratio):
    """Plain, mapped with and without a tonality limit, formant compensation at a fixed base and with the automatic pitch
    estimate, formants alone: six streams of one configure(2, 512, 128) batch."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    x = signals.batch("harmonic", len(SIX), 2, 4000, 48000)
    g = _emu(emu_libs["exact"], len(SIX))
    cfg(g)
    _set_batch(g, SIX)
    y = signals.run_batch(g, x, ratio, 640)
    _check(y, _oracles(oracle_port, cfg, SIX, x, ratio, 640))


def test_stereo_preset_plain_and_mapped_streams_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Paired FFT with interleaved rows for the plain streams and planar rows for the mapped ones (k_analyse2's per-item
    store), k_chain_direct4 next to k_chain_t, k_synth2: 32 blocks per call, streams alternating plain / mapped."""
    cfg = lambda o: o.presetDefault(2, 48000.0)  # noqa: E731
    prm = [PLAIN, (7, 8000 / SR, 0, False, 0), PLAIN, (12, 0, 0, True, 200 / SR)]
    x = signals.batch("harmonic", len(prm), 2, 2 * 57600, 48000)
    g = _emu(emu_libs["exact"], len(prm))
    cfg(g)
    _set_batch(g, prm)
    y = signals.run_batch(g, x, 0.8, 46080)
    _check(y, _oracles(oracle_port, cfg, prm, x, 0.8, 46080))


def test_mono_stream_pairs_with_mapped_partners_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Mono presetDefault on the paired wavefront (tuning key 5): pairs (plain, mapped) and (mapped, plain) run their plain
    stream alone; the odd stream of the batch is plain."""
    cfg = lambda o: o.presetDefault(1, 48000.0)  # noqa: E731
    prm = [PLAIN, (7, 8000 / SR, 0, False, 0), (-3, 0, 0, False, 0), PLAIN, PLAIN]
    x = signals.batch("harmonic", len(prm), 1, 57600 + 14400, 48000)
    g = _emu(emu_libs["exact"], len(prm), pairs=True)
    cfg(g)
    _set_batch(g, prm)
    y = signals.run_batch(g, x, 0.8, 46080)
    _check(y, _oracles(oracle_port, cfg, prm, x, 0.8, 46080))


def test_per_stream_parameter_changes_between_calls_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Stream 0 goes plain -> mapped -> formants with automatic pitch -> plain while stream 1 goes the reverse way: the
    interleaved and planar spectrum state is carried across layout switches, and only the automatic-pitch stream's
    pitch smoother advances."""
    mapped, formant = (3, 0.2, 0, False, 0), (3, 0.2, 3.0, True, 0)
    phases = [(PLAIN, PLAIN), (mapped, formant), (formant, mapped), (PLAIN, PLAIN), (PLAIN, formant)]
    x = signals.batch("harmonic", 2, 2, 2 * len(phases) * 5760, 48000)

    def run(objs, setp, proc):
        outs, pos = [], 0
        for ph in phases:
            setp(ph)
            for n_in in (5760, 7200):
                outs.append(proc(x[:, :, pos:pos + n_in], 5760))
                pos += n_in
        return np.concatenate(outs, axis=-1)

    g = _emu(emu_libs["exact"], 2)
    g.presetDefault(2, 48000.0)
    y = run(g, lambda ph: _set_batch(g, list(ph)), lambda a, n: np.array(g.process(a, n)))
    refs = []
    for s in range(2):
        o = oracle_port()
        o.presetDefault(2, 48000.0)
        refs.append(run(o, lambda ph, o=o, s=s: _set_one(o, ph[s]), lambda a, n, o=o, s=s: o.process(a[s], n)[None])[0])
    _check(y, np.stack(refs))


@pytest.mark.parametrize("step_major", [True, False], ids=["step_major", "round1"])
def test_random_time_factors_in_a_mixed_batch_bit_exact_vs_oracle(emu_libs, step_major):
    """2.5x stretch: every block draws random time factors; plain and mapped streams of one batch all go through the one
    random-only k_prep + k_chain launch (or, on the round-1 kernels, through k_prep + k_chain with the mapped streams)."""
    from oracle.hdrref import CpuStretch

    seed = 321
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    prm = [PLAIN, (3, 0.25, 0, False, 0), (12, 0, 0, True, 200 / SR), PLAIN]
    x = signals.batch("harmonic", len(prm), 2, 2000, 48000)
    g = _emu(emu_libs["exact"], len(prm), seed=seed, step_major=step_major)
    cfg(g)
    _set_batch(g, prm)
    y = signals.run_batch(g, x, 2.5, 1280)
    _check(y, _oracles(lambda: CpuStretch("orc", seed), cfg, prm, x, 2.5, 1280))


def test_equal_per_stream_values_equal_the_broadcast_setters(emu_libs):
    """Per-stream setters with the same value everywhere: the same outputs and the same launch sequence as the broadcast
    setters; a broadcast setter after per-stream values resets every stream; bad arguments are refused."""
    from signalsmith_stretch_b200 import StretchError  # noqa: F401

    S, C = 3, 2
    x = signals.batch("harmonic", S, C, 3000, 48000)
    outs, launches = [], []
    for per in (False, True):
        g = _emu(emu_libs["float"], S)
        g.configure(C, 512, 128)
        if per:
            g.setTransposeSemitones(np.full(S, 4, np.float32), np.full(S, 0.2, np.float32))
            g.setFormantFactor(np.full(S, 1.1, np.float32), np.ones(S, bool))
            g.setFormantBase(np.full(S, 150 / SR, np.float32))
        else:
            g.setTransposeSemitones(4, 0.2)
            g.setFormantFactor(1.1, True)
            g.setFormantBase(150 / SR)
        n0 = g.kernel_launches()
        outs.append(signals.run_batch(g, x, 0.8, 640))
        launches.append(g.kernel_launches() - n0)
    assert np.array_equal(outs[0], outs[1])
    assert launches[0] == launches[1]

    # a broadcast setter overrides earlier per-stream values on every stream
    ys = []
    for mixed_first in (False, True):
        g = _emu(emu_libs["float"], S)
        g.configure(C, 512, 128)
        if mixed_first:
            _set_batch(g, [PLAIN, (5, 0, 2, True, 0), (-7, 0.1, 0, False, 0)])
        g.setTransposeSemitones(0, 0)
        g.setFormantSemitones(0, False)
        g.setFormantBase(0)
        n0 = g.kernel_launches()
        ys.append(signals.run_batch(g, x, 0.8, 640))
        launches.append(g.kernel_launches() - n0)
    assert np.array_equal(ys[0], ys[1]) and launches[2] == launches[3]

    # NULL arrays: refused; NULL tonality limits / compensation flags mean 0 for every stream
    lib, h = g._lib, g._h
    fp = ctypes.POINTER(ctypes.c_float)
    ones = np.ones(S, np.float32)
    for fn in ("b200s_set_transpose_factor_per_stream", "b200s_set_transpose_semitones_per_stream",
               "b200s_set_formant_factor_per_stream", "b200s_set_formant_semitones_per_stream"):
        assert getattr(lib, fn)(h, None, None) == -1, fn
        assert getattr(lib, fn)(h, ones.ctypes.data_as(fp), None) == 0, fn
    assert lib.b200s_set_formant_base_per_stream(h, None) == -1
    assert lib.b200s_set_transpose_semitones_per_stream(None, ones.ctypes.data_as(fp), None) == -1
    for call in (lambda: g.setTransposeSemitones(np.zeros(S + 1), 0), lambda: g.setTransposeFactor(1.0, np.zeros(S - 1)),
                 lambda: g.setFormantFactor(np.ones(2), True), lambda: g.setFormantSemitones(0, np.zeros(S + 2, bool)),
                 lambda: g.setFormantBase(np.zeros((S, 1)))):
        with pytest.raises(ValueError):
            call()


class _OneStreamWithParams:
    """A one-stream oracle object behind the calls LiveBatch makes, including the per-stream parameter setters."""

    def __init__(self, o):
        self.o, self.batch = o, 1

    def channels(self):
        return self.o.channels

    def inputLatency(self):
        return self.o.inputLatency()

    def outputLatency(self):
        return self.o.outputLatency()

    def seek(self, win, rates):
        self.o.seek(win[0], float(rates[0]))

    def process(self, x, n_out):
        return self.o.process(x[0], n_out)[None]

    def setTransposeSemitones(self, semis, ton):
        self.o.setTransposeSemitones(float(np.float32(semis[0])), float(np.float32(ton[0])))

    def setFormantSemitones(self, semis, comp):
        self.o.setFormantSemitones(float(np.float32(semis[0])), bool(comp[0]))

    def setFormantBase(self, base):
        self.o.setFormantBase(float(np.float32(base[0])))


@pytest.mark.parametrize("bank", [None, "numpy"], ids=["host_windows", "device_bank"])
def test_live_batch_per_segment_parameters_bit_exact_vs_oracle(emu_libs, oracle_port, bank):
    """The worklet's per-segment semitones / tonalityHz / formant fields (web-wrapper.js:23-27, set every quantum at
    :233-235): three streams whose time maps change their parameters at different times, against three oracle objects
    whose parameters are set every quantum like the worklet's."""
    from signalsmith_stretch_b200.live import LiveBatch

    sr, S, C, quantum = SR, 3, 2, 128
    audio = signals.batch("harmonic", S, C, 12000, 48000)
    g = _emu(emu_libs["exact"], S)
    g.configure(C, 512, 128)
    live = LiveBatch(g, sr, bank=bank)
    refs = []
    for s in range(S):
        o = oracle_port()
        o.configure(C, 512, 128)
        refs.append(LiveBatch(_OneStreamWithParams(o), sr))
    # (the one-stream adapters are driven every quantum: force their setters on in every quantum)

    def both(fn):
        fn(live, lambda s: s)
        for s, r in enumerate(refs):
            fn(r, lambda _s, s=s: 0 if _s == s else None)

    def setup(lv, idx):
        for s in range(S):
            if idx(s) is not None:
                lv.add_buffers(idx(s), audio[s])
        for s, kw in enumerate([dict(rate=0.8, offset=0.01), dict(rate=1.0, offset=0.0, semitones=4), dict(rate=1.2, offset=0.02)]):
            if idx(s) is not None:
                lv.start(idx(s), when=0.004 * s, **kw)
        if idx(2) is not None:
            lv.schedule(idx(2), dict(outputTime=0.03, semitones=-5, tonalityHz=6000, formantSemitones=2, formantBaseHz=180))

    both(setup)
    outs, ref_outs = [], [[] for _ in range(S)]
    for qn in range(36):
        if qn == 20:  # stream 0: formant compensation with automatic pitch from now; stream 1 slows down (inherits +4 st)
            both(lambda lv, idx: [lv.schedule(idx(0), dict(semitones=7, formantCompensation=True)) if idx(0) is not None else None,
                                  lv.schedule(idx(1), dict(rate=0.7)) if idx(1) is not None else None])
        outs.append(live.process(quantum))
        for s, r in enumerate(refs):
            r._prm_sent = None  # the worklet sets its parameters in every quantum
            ref_outs[s].append(r.process(quantum)[0])
    y = np.concatenate(outs, axis=-1)
    for s in range(S):
        r = np.concatenate(ref_outs[s], axis=-1)
        assert np.array_equal(y[s], r), "stream %d: max diff %g" % (s, np.abs(y[s] - r).max())
    assert np.abs(y).max() > 0.05


def test_live_batch_parameter_fields_are_inherited_and_optional():
    """schedule() inherits the parameter fields like the others; without any parameter field no setter is ever called."""
    from signalsmith_stretch_b200.live import LiveBatch

    class Eng:
        batch = 2

        def __init__(self):
            self.calls = []

        def channels(self):
            return 1

        def inputLatency(self):
            return 64

        def outputLatency(self):
            return 64

        def seek(self, win, rates):
            pass

        def process(self, x, n):
            return np.zeros((2, 1, n), np.float32)

        def setTransposeSemitones(self, *a):
            self.calls.append(("t",) + tuple(np.array(v).tolist() for v in a))

        def setFormantSemitones(self, *a):
            self.calls.append(("f",) + tuple(np.array(v).tolist() for v in a))

        def setFormantBase(self, *a):
            self.calls.append(("b",) + tuple(np.array(v).tolist() for v in a))

    e = Eng()
    lv = LiveBatch(e, SR)
    lv.start(0, when=0.0)
    lv.schedule(1, dict(outputTime=0.0, active=True, rate=1.5))
    for _ in range(4):
        lv.process(64)
    assert e.calls == []  # no parameter field anywhere: the engine's own parameters stay
    lv.start(1, when=lv.current_time, semitones=3)
    seg = lv.schedule(1, dict(outputTime=lv.current_time + 0.01, rate=0.5))
    assert seg["semitones"] == 3 and seg["rate"] == 0.5
    lv.process(64)
    assert len(e.calls) == 3 and e.calls[0][1] == [0.0, 3.0]
    assert e.calls[0][2] == pytest.approx([8000 / SR] * 2)
    lv.process(64)
    assert len(e.calls) == 3  # unchanged values are not sent again


def test_live_batch_parameter_change_takes_effect_at_the_worklets_quantum():
    """Which segment's parameters a quantum uses, against a hand-written table of the worklet (web-wrapper.js).  The
    quantum starting at sample q*n looks the segment up at outputTime = (q*n + outputLatency) / sampleRate (:226-231) and
    sets semitones, tonalityHz / sampleRate, formant semitones and compensation, formantBaseHz / sampleRate from it
    (:233-235).  `schedule` itself shifts the map up to the new point (:97-101), so a point scheduled before quantum q --
    even with a later output time -- is the segment of quantum q; fields it does not give are inherited (:75-80)."""
    from signalsmith_stretch_b200.live import LiveBatch

    n, out_lat = 128, 96

    class Eng:  # records the parameters the engine holds after each quantum
        batch = 2

        def __init__(self):
            self.p = dict(semis=[0.0, 0.0], ton=[0.0, 0.0], fsemi=[0.0, 0.0], comp=[False, False], base=[0.0, 0.0])

        def channels(self):
            return 1

        def inputLatency(self):
            return 64

        def outputLatency(self):
            return out_lat

        def seek(self, win, rates):
            pass

        def process(self, x, k):
            return np.zeros((2, 1, k), np.float32)

        def setTransposeSemitones(self, semis, ton):
            self.p["semis"], self.p["ton"] = list(np.float64(semis)), list(np.float64(ton) * SR)

        def setFormantSemitones(self, semis, comp):
            self.p["fsemi"], self.p["comp"] = list(np.float64(semis)), [bool(c) for c in comp]

        def setFormantBase(self, base):
            self.p["base"] = list(np.float64(base) * SR)

    e = Eng()
    lv = LiveBatch(e, SR)
    at = lambda samples: samples / SR  # noqa: E731
    lv.start(0, when=0.0, semitones=2)
    events = {  # before quantum q
        3: lambda: lv.schedule(1, dict(outputTime=at(6 * n + out_lat), formantSemitones=4, formantCompensation=True, formantBaseHz=150)),
        6: lambda: lv.schedule(0, dict(outputTime=at(5 * n), semitones=-3, tonalityHz=4000)),
        8: lambda: lv.stop(1),  # stream 1 stops: its parameters are inherited
    }
    expect = []
    for q in range(10):
        expect.append(dict(semis=[2.0 if q < 6 else -3.0, 0.0], ton=[8000.0 if q < 6 else 4000.0, 8000.0],
                           fsemi=[0.0, 0.0 if q < 3 else 4.0], comp=[False, q >= 3], base=[0.0, 0.0 if q < 3 else 150.0]))
    for q in range(10):
        if q in events:
            events[q]()
        lv.process(n)
        got = e.p
        for k, v in expect[q].items():
            assert got[k] == pytest.approx(v, rel=1e-6), (q, k, got[k], v)


# ------------------------------------------------------------------ H100
def _random_mix(S, seed=1234):
    """The benchmark's last mix (bench_mixed.py): semitones from [-12, 12], 10 % plain, 10 % formant compensation at 200 Hz."""
    rng = np.random.default_rng(seed)
    semis = rng.uniform(-12, 12, S).astype(np.float32)
    order = rng.permutation(S)
    comp = np.zeros(S, bool)
    base = np.zeros(S, np.float32)
    n10 = S // 10
    semis[order[:n10]] = 0
    comp[order[n10:2 * n10]] = True
    base[order[n10:2 * n10]] = 200 / SR
    return [(float(semis[s]), 8000 / SR, 0.0, bool(comp[s]), float(base[s])) for s in range(S)]


@pytest.mark.gpu
def test_mixed_batch_equals_uniform_batches_on_the_gpu(cuda_lib, oracle_port):
    """64 stereo streams, presetDefault 0.8x, 32 blocks per call, per-stream parameters, fast arithmetic: each stream is
    bit-identical to the same stream in a batch whose streams all share its parameters (the plain streams run the same
    kernels either way, and so do the mapped ones), and within the usual tolerances of its oracle."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C = 64, 2
    prm = _random_mix(S)
    n_out, calls = 46080, 2
    n_in = int(round(n_out / 0.8))
    x = signals.batch("harmonic", S, C, calls * n_in, 48000)
    g = BatchStretch(S)
    g.presetDefault(C, SR)
    _set_batch(g, prm)
    y = signals.run_batch(g, x, 0.8, n_out)
    groups = {}
    for s, p in enumerate(prm):
        groups.setdefault(p, []).append(s)
    assert len(groups) > 2
    for p, idx in groups.items():
        u = BatchStretch(len(idx))
        u.presetDefault(C, SR)
        _set_one(u, p)
        yu = signals.run_batch(u, x[idx], 0.8, n_out)
        for j, s in enumerate(idx):
            assert np.array_equal(y[s], yu[j]), "stream %d %s: max diff %g" % (s, p, np.abs(y[s] - yu[j]).max())
    ref = _oracles(oracle_port, lambda o: o.presetDefault(C, SR), prm, x, 0.8, n_out)
    H = g.intervalSamples()
    lat = g.outputLatency() + int(g.inputLatency() * 0.8)
    per = np.array([rms((y[s] - ref[s])[:, : lat + 8 * H]) for s in range(S)])
    assert np.median(per) <= 1e-4, per
    assert per.max() <= 1e-3, per


@pytest.mark.gpu
def test_mixed_parameters_allocate_nothing_in_process(cuda_lib):
    """After reserve() with mixed per-stream parameters, process() allocates nothing -- also when the per-stream values
    change between calls."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C = 16, 2
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    _set_batch(e, _random_mix(S, seed=7))
    H = e.intervalSamples()
    n_out = 8 * H
    n_in = int(round(n_out / 0.8))
    e.reserve(n_in, n_out)
    x = signals.batch("harmonic", S, C, 4 * n_in, 48000)
    before = e.device_allocations()
    for k in range(4):
        if k:
            _set_batch(e, _random_mix(S, seed=7 + k))
        e.process(x[:, :, k * n_in:(k + 1) * n_in], n_out)
    e.synchronize()
    assert e.device_allocations() == before
