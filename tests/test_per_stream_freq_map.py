"""Every stream of a batch with its own frequency-map table (b200s_set_freq_map_table_per_stream).

Under the CPU emulator (exact arithmetic, the oracle's FFT swapped in) every stream of a batch whose streams carry
different tables -- monotone, folding, one point (a shift), two points, 2049 points, none, the engine's table, a table
with formant compensation -- is bit-identical to its own one-stream oracle given that table, over calls between which a
table changes; on the random path too.  The setters interplay as the reference's would, stream copies carry the
tables, and bad arguments change nothing.  On the H100 (-m gpu) the GPU equals the emulator bit for bit in exact
arithmetic, at the preset sizes and at batch scale.
"""
import ctypes

import numpy as np
import pytest

import signals

SR = 48000.0
PLAIN = (0, 0, 0, False, 0)
STATE_KEYS = ("history", "input", "prevInput", "output", "predEnergy", "pending", "pendingWp")


def _tab(fn, n):
    fin = np.linspace(0.0, 0.5, n).astype(np.float32)
    return fin, np.array([fn(float(f)) for f in fin], np.float32)


ENGINE = _tab(lambda f: 0.9 * f + 0.1 * f * f, 9)
ONE = (np.array([0.05], np.float32), np.array([0.065], np.float32))  # mapN == 1: a shift by 0.015
TWO = (np.array([0.0, 0.5], np.float32), np.array([0.0, 0.6], np.float32))
DENSE = _tab(lambda f: f * (1.15 + 0.2 * np.sin(40 * f)), 2049)
# per stream: (table or "engine" or None, (semitones, tonality, formant semitones, compensation, formant base))
MIX = [
    (signals.PWL_MONOTONE, PLAIN),
    (signals.PWL_FOLDING, PLAIN),
    (ONE, PLAIN),
    (TWO, PLAIN),
    (DENSE, PLAIN),
    (None, (3, 0, 0, False, 0)),
    ("engine", PLAIN),
    (signals.PWL_MONOTONE, (0, 0, 2, True, 200 / SR)),
]


def _emu(path, batch, seed=0, exact_math=True, step_major=True):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=seed, lib_path=path)
    e.set_tuning(3, 1 if exact_math else 0)
    if not step_major:
        e.set_tuning(4, 0)
    return e


def _set_mix(e, mix):
    """Transpose and formant values first (a transpose setter clears every map), then the engine table on every stream,
    then the streams' own tables (None: no map)."""
    semis, ton, fsemi, comp, base = (np.array(v) for v in zip(*[p for _, p in mix]))
    e.setTransposeSemitones(semis.astype(np.float32), ton.astype(np.float32))
    e.setFormantSemitones(fsemi.astype(np.float32), comp.astype(bool))
    e.setFormantBase(base.astype(np.float32))
    e.setFreqMapTable(*ENGINE)
    own = [s for s, (t, _) in enumerate(mix) if not (isinstance(t, str) and t == "engine")]
    e.setFreqMapTable([mix[s][0] for s in own], streams=own)


def _oracle(cfg, entry, seed=0):
    from oracle.hdrref import CpuStretch

    t, p = entry
    o = CpuStretch("orc", seed)
    cfg(o)
    o.setTransposeSemitones(p[0], p[1])
    o.setFormantSemitones(p[2], p[3])
    o.setFormantBase(p[4])
    if t is not None:
        o.setFreqMapTable(*(ENGINE if isinstance(t, str) else t))
    return o


def _same(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s: max diff %g" % (what, np.abs(a - b).max())


def _states(e):
    return {k: np.array(e.get_state(k)) for k in STATE_KEYS}


def _calls(H, ratio, blocks):
    res, o, i = [], 0, 0
    for b in blocks:
        o += int(b * H)
        n_in = int(round(o / ratio)) - i
        i += n_in
        res.append((n_in, int(b * H)))
    return res


# ------------------------------------------------------------------ CPU emulator, against the oracle
CFGS = {
    "stereo_2_512_128": (2, lambda o: o.configure(2, 512, 128)),
    "mono_1_512_128": (1, lambda o: o.configure(1, 512, 128)),
    "stereo_presetDefault": (2, lambda o: o.presetDefault(2, SR)),
    "mono_presetDefault": (1, lambda o: o.presetDefault(1, SR)),
}


@pytest.mark.parametrize("step_major", [True, False], ids=["step_major", "round1"])
@pytest.mark.parametrize("cfg_id", list(CFGS))
def test_mixed_tables_bit_exact_vs_oracle(emu_libs, oracle_port, cfg_id, step_major):
    """The eight kinds of stream in one batch over three calls; before the third, stream 0 takes the folding table and
    stream 5 the dense one (its transposition stays), the others keep theirs."""
    C, cfg = CFGS[cfg_id]
    g = _emu(emu_libs["exact"], len(MIX), step_major=step_major)
    cfg(g)
    _set_mix(g, MIX)
    H = g.intervalSamples()
    blocks = (2.0, 3.0, 3.0) if g.blockSamples() < 1000 else (1.0, 4.0, 3.0)
    calls = _calls(H, 0.8, blocks)
    n = sum(c[0] for c in calls)
    x = signals.batch("harmonic", len(MIX), C, n, 48000)
    later = {0: signals.PWL_FOLDING, 5: DENSE}
    ys, pos = [], 0
    for k, (n_in, n_out) in enumerate(calls):
        if k == 2:
            g.setFreqMapTable([later[s] for s in later], streams=list(later))
        ys.append(np.array(g.process(np.ascontiguousarray(x[:, :, pos:pos + n_in]), n_out)))
        pos += n_in
    for s, entry in enumerate(MIX):
        o = _oracle(cfg, entry)
        pos = 0
        for k, (n_in, n_out) in enumerate(calls):
            if k == 2 and s in later:
                o.setFreqMapTable(*later[s])
            _same(ys[k][s], o.process(x[s][:, pos:pos + n_in], n_out), "stream %d, call %d" % (s, k))
            pos += n_in


@pytest.mark.parametrize("step_major", [True, False], ids=["step_major", "round1"])
def test_random_path_with_mapped_and_plain_streams(emu_libs, step_major):
    """2.5x stretch (every block draws random time factors): own tables, the engine table and plain streams in one batch."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    mix = [(signals.PWL_FOLDING, PLAIN), (None, PLAIN), ("engine", PLAIN), (ONE, PLAIN), (None, (4, 0, 0, False, 0))]
    g = _emu(emu_libs["exact"], len(mix), seed=321, step_major=step_major)
    cfg(g)
    _set_mix(g, mix)
    x = signals.batch("harmonic", len(mix), 2, 2000, 48000)
    y = signals.run_batch(g, x, 2.5, 1280)
    assert g.unserved_random_blocks() == 0
    for s, entry in enumerate(mix):
        o = _oracle(cfg, entry, seed=321)
        _same(y[s], signals.run_single(o, x[s], 2.5, 1280), "stream %d" % s)


def test_same_table_per_stream_equals_the_engine_table(emu_libs):
    """The engine's table set on every stream through the per-stream call: the same outputs, state and launches."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    x = signals.batch("harmonic", 3, 2, 4000, 48000)
    runs = []
    for per_stream in (False, True):
        g = _emu(emu_libs["float"], 3)
        cfg(g)
        if per_stream:
            g.setFreqMapTable(*signals.PWL_FOLDING, streams=[2, 0, 1])
        else:
            g.setFreqMapTable(*signals.PWL_FOLDING)
        y = signals.run_batch(g, x, 0.8, 640)
        runs.append((y, _states(g), g.kernel_launches(), g.export_streams([0, 1, 2])[:, 128:]))
    _same(runs[0][0], runs[1][0], "outputs")
    for k in STATE_KEYS:
        _same(runs[0][1][k], runs[1][1][k], k)
    assert runs[0][2] == runs[1][2]
    assert np.array_equal(runs[0][3], runs[1][3])  # the records' state, after their headers


def _header(rec):
    """(table flags, mapN, customMap) of a record's header (engine.cu StreamRecordHeader): flags 4 = the engine's table,
    8 = the stream's own."""
    w = np.frombuffer(rec[:128].tobytes(), np.int32)
    return int(w[9]) & 12, int(w[10]), int(w[20])


def test_setter_interplay(emu_libs):
    """Per-stream tables replace only the listed streams'; the engine-wide setter replaces every stream's; a transpose
    setter, broadcast or per stream, clears every stream's map."""
    g = _emu(emu_libs["float"], 4)
    g.configure(1, 512, 128)
    g.setFreqMapTable(*ENGINE)
    g.setFreqMapTable([signals.PWL_FOLDING, None], streams=[1, 3])
    kinds = [_header(r)[0] for r in g.export_streams([0, 1, 2, 3])]
    assert kinds == [4, 8, 4, 0]  # engine table, own, engine table, none
    g.setFreqMapTable([ONE], streams=[0])
    assert [_header(r)[0] for r in g.export_streams([0, 1, 2, 3])] == [8, 8, 4, 0]
    assert _header(g.export_streams([0])[0])[1] == 1
    g.setFreqMapTable(*signals.PWL_MONOTONE)
    assert [_header(r)[:2] for r in g.export_streams([0, 1, 2, 3])] == [(4, 5)] * 4
    g.setFreqMapTable([TWO], streams=[2])
    g.setTransposeSemitones(np.zeros(4, np.float32))
    assert [_header(r)[0] for r in g.export_streams([0, 1, 2, 3])] == [0] * 4
    g.setFreqMapTable([TWO], streams=[2])
    g.setTransposeFactor(1.0)
    assert [_header(r)[0] for r in g.export_streams([0, 1, 2, 3])] == [0] * 4
    # a stream with its own table runs as a one-stream engine given that table, after all of the above
    g.setFreqMapTable([DENSE], streams=[3])
    x = signals.batch("harmonic", 4, 1, 3000, 48000)
    y = signals.run_batch(g, x, 1.0, 640)
    h = _emu(emu_libs["float"], 1)
    h.configure(1, 512, 128)
    h.setFreqMapTable(*DENSE)
    _same(y[3], signals.run_batch(h, x[3:], 1.0, 640)[0], "stream 3")


def test_bad_arguments_change_nothing(emu_libs):
    from signalsmith_stretch_b200 import StretchError

    g = _emu(emu_libs["float"], 3)
    g.configure(1, 512, 128)
    g.setFreqMapTable([signals.PWL_FOLDING], streams=[1])
    x = signals.batch("harmonic", 3, 1, 1500, 48000)
    g.process(x, 1200)
    rec = g.export_streams([0, 1, 2])
    before = (g.kernel_launches(), g.device_allocations())
    lib, h = g._lib, g._h
    ip, fp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float)
    fin, fout = (np.ascontiguousarray(a, np.float32) for a in signals.PWL_MONOTONE)
    cases = [
        ([0, 3], [5, 5], "streams[1] = 3 is outside [0, 3)"),
        ([-1], [5], "streams[0] = -1 is outside"),
        ([2, 2], [5, 0], "streams[1]: stream 2 is listed twice"),
        ([0, 1], [5, -1], "n_points[1] = -1 is negative"),
    ]
    for streams, pts, msg in cases:
        s, p = np.array(streams, np.int32), np.array(pts, np.int32)
        with pytest.raises(StretchError, match=msg.replace("[", r"\[").replace("]", r"\]").replace("(", r"\(").replace(")", r"\)")):
            g._ck(lib.b200s_set_freq_map_table_per_stream(h, s.ctypes.data_as(ip), len(s), p.ctypes.data_as(ip),
                                                         np.concatenate([fin, fin]).ctypes.data_as(fp), np.concatenate([fout, fout]).ctypes.data_as(fp)))
    one = np.array([0], np.int32)
    five = np.array([5], np.int32)
    for args, msg in [((None, 1, five.ctypes.data_as(ip), fin.ctypes.data_as(fp), fout.ctypes.data_as(fp)), "streams must not be NULL"),
                      ((one.ctypes.data_as(ip), 1, None, fin.ctypes.data_as(fp), fout.ctypes.data_as(fp)), "n_points must not be NULL"),
                      ((one.ctypes.data_as(ip), -1, five.ctypes.data_as(ip), fin.ctypes.data_as(fp), fout.ctypes.data_as(fp)), "negative stream count"),
                      ((one.ctypes.data_as(ip), 1, five.ctypes.data_as(ip), None, fout.ctypes.data_as(fp)), "freq_in and freq_out must not be NULL")]:
        with pytest.raises(StretchError, match=msg):
            g._ck(lib.b200s_set_freq_map_table_per_stream(h, *args))
    assert (g.kernel_launches(), g.device_allocations()) == before
    assert np.array_equal(g.export_streams([0, 1, 2]), rec)
    # nothing changed: the next call equals that of an engine that never saw the bad calls
    y = np.array(g.process(x, 1200))
    r = _emu(emu_libs["float"], 3)
    r.configure(1, 512, 128)
    r.setFreqMapTable([signals.PWL_FOLDING], streams=[1])
    r.process(x, 1200)
    _same(y, np.array(r.process(x, 1200)), "after the refused calls")


def test_second_set_within_capacity_allocates_nothing(emu_libs):
    """The pool grows on the first set; a later set that fits, with other tables, allocates nothing, and 16 streams that
    share 2 tables hold 2."""
    g = _emu(emu_libs["float"], 16)
    g.configure(1, 512, 128)
    g.setFreqMapTable([DENSE if s % 2 else signals.PWL_FOLDING for s in range(16)])
    a = g.device_allocations()
    g.setFreqMapTable([ONE if s % 2 else TWO for s in range(16)])
    g.setFreqMapTable([signals.PWL_MONOTONE], streams=[5])
    g.setFreqMapTable(*DENSE)
    assert g.device_allocations() == a


# ------------------------------------------------------------------ stream copies, export, import, clone
def _run_pair(a, b, x, calls):
    """The same calls on two engines; every output equal bit for bit."""
    pos = 0
    for n_in, n_out in calls:
        seg = np.ascontiguousarray(x[:, :, pos:pos + n_in])
        _same(np.array(a.process(seg, n_out)), np.array(b.process(seg, n_out)), "outputs")
        pos += n_in


def test_copies_within_one_engine_fork_and_swap_without_allocation(emu_libs, oracle_port):
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    mix = [(signals.PWL_FOLDING, PLAIN), (ONE, PLAIN), (None, (2, 0, 0, False, 0)), (None, PLAIN)]
    g = _emu(emu_libs["exact"], 4)
    cfg(g)
    _set_mix(g, mix)
    x = signals.batch("harmonic", 4, 2, 6000, 48000)
    g.process(x[:, :, :1500], 1200)
    g.copy_streams([0, 1, 2], [0, 1, 2])  # (warms the staging: copies onto themselves)
    a = g.device_allocations()
    g.copy_streams([1, 0, 3], [0, 1, 0])  # swap 0 and 1, fork 0 into 3
    assert g.device_allocations() == a
    y1 = np.array(g.process(np.ascontiguousarray(x[:, :, 1500:3000][[1, 0, 2, 0]]), 1200))
    for slot, src in ((0, 1), (1, 0), (3, 0)):
        o = _oracle(cfg, mix[src])
        o.process(x[src][:, :1500], 1200)
        _same(y1[slot], o.process(x[src][:, 1500:3000], 1200), "slot %d (stream %d)" % (slot, src))


def test_copy_across_engines_carries_the_table(emu_libs):
    """Own tables travel to an engine that has other tables (and none of the source's); an engine-table stream still
    needs the same engine table."""
    from signalsmith_stretch_b200 import StretchError

    src = _emu(emu_libs["float"], 3)
    src.configure(2, 512, 128)
    src.setFreqMapTable(*ENGINE)
    src.setFreqMapTable([signals.PWL_FOLDING, DENSE], streams=[0, 1])
    dst = _emu(emu_libs["float"], 5, seed=7)
    dst.configure(2, 512, 128)
    dst.setFreqMapTable([TWO, TWO], streams=[0, 4])
    x = signals.batch("harmonic", 3, 2, 5000, 48000)
    src.process(x[:, :, :1500], 1200)
    dst.copy_streams([3, 1], [0, 1], src=src)
    with pytest.raises(StretchError, match="frequency-map table"):
        dst.copy_streams([2], [2], src=src)
    ref = src.clone()
    xd = np.zeros((5, 2, 1500), np.float32)
    xd[3], xd[1] = x[0, :, 1500:3000], x[1, :, 1500:3000]
    yd = np.array(dst.process(xd, 1200))
    ys = np.array(ref.process(np.ascontiguousarray(x[:, :, 1500:3000]), 1200))
    _same(yd[3], ys[0], "stream 0 in slot 3")
    _same(yd[1], ys[1], "stream 1 in slot 1")
    # the carried table is the stream's own: its record says so
    assert _header(dst.export_streams([3])[0])[:2] == (8, 5)


def test_export_import_needs_the_table_in_the_slot(emu_libs):
    from signalsmith_stretch_b200 import StretchError

    g = _emu(emu_libs["float"], 3)
    g.configure(1, 512, 128)
    g.setFreqMapTable([signals.PWL_FOLDING, None], streams=[0, 1])
    x = signals.batch("harmonic", 3, 1, 4000, 48000)
    g.process(x[:, :, :1500], 1200)
    rec = g.export_streams([0])
    assert _header(rec[0])[:2] == (8, 5)
    h = _emu(emu_libs["float"], 3)
    h.configure(1, 512, 128)
    with pytest.raises(StretchError, match="record 0: .*table"):
        h.import_streams([2], rec)
    h.setFreqMapTable([signals.PWL_MONOTONE], streams=[2])
    with pytest.raises(StretchError, match="record 0: .*table"):
        h.import_streams([2], rec)
    bad = rec.copy()
    bad[0, 36] |= 0x40  # an unknown flag bit
    h.setFreqMapTable([signals.PWL_FOLDING], streams=[2])
    with pytest.raises(StretchError, match="record 0: unknown flags"):
        h.import_streams([2], bad)
    h.import_streams([2], rec)  # the slot holds the same table now
    h.setFreqMapTable(*signals.PWL_FOLDING)  # ... or the engine table, on stream 1
    h.import_streams([1], rec)
    seg = np.ascontiguousarray(x[:, :, 1500:3000])
    y = np.array(h.process(np.ascontiguousarray(seg[[1, 0, 0]]), 1200))
    ref = np.array(g.process(seg, 1200))[0]
    _same(y[2], ref, "imported into an own-table slot")
    _same(y[1], ref, "imported into an engine-table slot")


def test_clone_carries_the_tables(emu_libs):
    g = _emu(emu_libs["float"], 4)
    g.configure(2, 512, 128)
    g.setFreqMapTable(*ENGINE)
    g.setFreqMapTable([signals.PWL_FOLDING, ONE, None], streams=[0, 1, 3])
    x = signals.batch("harmonic", 4, 2, 5000, 48000)
    g.process(x[:, :, :1500], 1200)
    c = g.clone()
    _run_pair(g, c, x[:, :, 1500:], _calls(128, 0.8, (3.0, 4.0)))
    u = _emu(emu_libs["float"], 2)  # unconfigured: the tables still go along
    u.setFreqMapTable([DENSE], streams=[1])
    v = u.clone()
    for e in (u, v):
        e.configure(2, 512, 128)
    _run_pair(u, v, x[:2, :, :3000], _calls(128, 0.8, (3.0, 4.0)))


def test_records_without_own_tables_are_unchanged(emu_libs):
    """Streams without a table and streams on the engine table export the same bytes whether or not other streams of
    the engine have their own tables."""
    recs = []
    for own in (False, True):
        g = _emu(emu_libs["float"], 3)
        g.configure(1, 512, 128)
        g.setFreqMapTable(*signals.PWL_MONOTONE)
        g.setFreqMapTable([None] + ([DENSE] if own else []), streams=[0] + ([2] if own else []))
        g.process(signals.batch("harmonic", 3, 1, 1500, 48000), 1200)
        recs.append(g.export_streams([0, 1]))
    assert np.array_equal(recs[0], recs[1])
    assert _header(recs[0][0]) == (0, 0, 0) and _header(recs[0][1]) == (4, 5, 1)


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def engines(cuda_lib, emu_libs):
    import torch

    assert torch.cuda.is_available(), "these tests need a GPU"
    from signalsmith_stretch_b200 import BatchStretch

    return {"gpu": lambda S, seed=0: BatchStretch(S, seed=seed),
            "emu": lambda S, seed=0: BatchStretch(S, seed=seed, lib_path=emu_libs["float"])}


def _drive(e, x, calls):
    outs, states, pos = [], [], 0
    for n_in, n_out in calls:
        outs.append(np.array(e.process(np.ascontiguousarray(x[:, :, pos:pos + n_in]), n_out)))
        pos += n_in
        states.append(_states(e))
    return outs, states


@pytest.mark.gpu
@pytest.mark.parametrize("preset", ["default_stereo_3072", "cheaper_mono_2560"])
def test_gpu_equals_the_emulator_in_exact_mode(engines, preset):
    C = 2 if preset.startswith("default") else 1
    mix = [MIX[0], MIX[1], MIX[6], MIX[7], MIX[5]] if C == 2 else [MIX[2], MIX[4], MIX[5], MIX[3]]
    res = []
    for kind in ("gpu", "emu"):
        e = engines[kind](len(mix))
        e.set_tuning(3, 1)
        (e.presetDefault if C == 2 else e.presetCheaper)(C, SR)
        _set_mix(e, mix)
        calls = _calls(e.intervalSamples(), 0.8, (1.0, 32, 40))
        x = signals.batch("harmonic", len(mix), C, sum(c[0] for c in calls), 48000)
        res.append(_drive(e, x, calls))
    for k in range(3):
        _same(res[0][0][k], res[1][0][k], "outputs, call %d" % k)
        for name in STATE_KEYS:
            _same(res[0][1][k][name], res[1][1][k][name], "%s after call %d" % (name, k))


@pytest.mark.gpu
def test_gpu_batch_scale_sixteen_tables(engines):
    """1024 stereo streams, presetDefault 0.8x, 16 distinct 2049-point tables (stream s: table and input s % 16).  In
    exact mode every copy of a (table, input) pair is bit-identical and the sampled pairs equal the emulator; in fast mode
    the sampled streams agree with the oracle within 1e-4 RMS over the first 8 blocks."""
    from oracle.hdrref import CpuStretch

    S, P = 1024, 16
    tabs = [_tab(lambda f, k=k: f * (0.8 + 0.025 * k) + 0.01 * np.sin(30 * f), 2049) for k in range(P)]
    probe = engines["gpu"](1)
    probe.presetDefault(2, SR)
    calls = _calls(probe.intervalSamples(), 0.8, (32, 32))
    n = sum(c[0] for c in calls)
    pool = signals.batch("harmonic", P, 2, n, 48000)
    x = np.ascontiguousarray(pool[np.arange(S) % P])
    sampled = [3, 14]
    for exact in (1, 0):
        e = engines["gpu"](S)
        e.set_tuning(3, exact)
        e.presetDefault(2, SR)
        e.setFreqMapTable([tabs[s % P] for s in range(S)])
        outs, _ = _drive(e, x, calls)
        y = np.concatenate(outs, axis=-1)
        assert np.all(np.isfinite(y))
        if exact:
            for s in range(P, S):
                _same(y[s], y[s % P], "stream %d against stream %d" % (s, s % P))
            m = engines["emu"](len(sampled))
            m.set_tuning(3, 1)
            m.presetDefault(2, SR)
            m.setFreqMapTable([tabs[k] for k in sampled])
            ye = np.concatenate(_drive(m, np.ascontiguousarray(pool[sampled]), calls[:1])[0], axis=-1)
            for i, k in enumerate(sampled):
                _same(y[k, :, :ye.shape[-1]], ye[i], "stream %d against the emulator" % k)
        else:
            m8 = 8 * probe.intervalSamples()
            for k in sampled:
                o = CpuStretch("orc")
                o.presetDefault(2, SR)
                o.setFreqMapTable(*tabs[k])
                ref = o.process(pool[k][:, :calls[0][0]], calls[0][1])
                err = float(np.sqrt(np.mean((y[k, :, :m8].astype(np.float64) - ref[:, :m8]) ** 2)))
                assert err <= 1e-4, (k, err)


@pytest.mark.gpu
def test_gpu_cross_device_copy_carries_the_table(cuda_lib):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from signalsmith_stretch_b200 import BatchStretch

    a, b = BatchStretch(2, device=0), BatchStretch(3, device=1)
    for e in (a, b):
        e.set_tuning(3, 1)
        e.presetDefault(2, SR)
    a.setFreqMapTable([signals.PWL_FOLDING, DENSE], streams=[0, 1])
    x = signals.batch("harmonic", 2, 2, 3 * 14400, 48000)
    a.process(np.ascontiguousarray(x[:, :, :14400]), 11520)
    b.copy_streams([2, 0], [0, 1], src=a)
    ya = np.array(a.process(np.ascontiguousarray(x[:, :, 14400:28800]), 11520))
    xb = np.zeros((3, 2, 14400), np.float32)
    xb[2], xb[0] = x[0, :, 14400:28800], x[1, :, 14400:28800]
    yb = np.array(b.process(xb, 11520))
    _same(yb[2], ya[0], "stream 0 on the second GPU")
    _same(yb[0], ya[1], "stream 1 on the second GPU")
