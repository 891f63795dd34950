"""Copying, exporting and importing single streams (b200s_copy_streams / _export_streams / _import_streams / _clone).

Under the CPU emulator (exact arithmetic, the oracle's FFT swapped in) a copied stream and its source, fed the same calls,
give the same bits, and both equal a one-stream oracle driven through the stream's whole history -- within one engine
(swaps and forks included), across engines with another batch, seed and tuning, and through exported records.  On the
H100 (-m gpu) copies continue bit-identically in fast arithmetic, equal the emulator in exact arithmetic, wait for
chained asynchronous calls, and allocate nothing the second time.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import signals

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 48000.0
SKIP, PROC, SEEK, OSEEK, FLUSH, RESET = range(6)
STATE_NAMES = ("input", "prevInput", "output", "predEnergy", "history", "pending", "pendingWp")
PLAIN = (0, 0, 0, False, 0)
# the five kinds of stream: plain, transposed with a tonality limit, formants with compensation, formants with the
# automatic pitch estimate, and one that uses the engine's frequency-map table ("table")
KINDS = [PLAIN, (3, 8000 / SR, 0, False, 0), (-2, 0, 3, True, 200 / SR), (0, 0, -4, False, 0), "table"]


def _engine(path, batch, seed=321, exact_math=True):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=seed, lib_path=path)
    e.set_tuning(3, 1 if exact_math else 0)
    return e


def _set_params(e, prm):
    """prm: one entry per stream, a (semitones, tonality, formant semitones, compensate, base) tuple or "table".  The
    table streams are made by importing a record taken while the table was on for every stream: the transpose setters
    turn it off for the whole batch."""
    table = [s for s, p in enumerate(prm) if p == "table"]
    if table:
        e.setFreqMapTable(*signals.PWL_MONOTONE)
        rec = e.export_streams(table)
    semis, ton, fsemi, comp, base = (np.array(v) for v in zip(*[PLAIN if p == "table" else p for p in prm]))
    e.setTransposeSemitones(semis.astype(np.float32), ton.astype(np.float32))
    e.setFormantSemitones(fsemi.astype(np.float32), comp.astype(bool))
    e.setFormantBase(base.astype(np.float32))
    if table:
        e.import_streams(table, rec)


def _oracle(cfg, p):
    from oracle.hdrref import CpuStretch

    o = CpuStretch("orc", 321)
    cfg(o)
    if p == "table":
        o.setFreqMapTable(*signals.PWL_MONOTONE)
    else:
        o.setTransposeSemitones(p[0], p[1])
        o.setFormantSemitones(p[2], p[3])
        o.setFormantBase(p[4])
    return o


def _step(g, call, xs, pos):
    """One run() call: call[s] = (op, n_in, n_out, rate); stream s reads the next n_in samples of xs[s].  Returns the
    outputs of its PROCESS / FLUSH streams as {s: [C][n_out]}."""
    S, C = len(call), xs[0].shape[0]
    ops = np.array([t[0] for t in call], np.int32)
    n_in = np.array([t[1] for t in call], np.int32)
    n_out = np.array([t[2] for t in call], np.int32)
    rates = np.array([t[3] for t in call], np.float64)
    stride = (int(n_in.max()) + 7) // 4 * 4
    buf = np.full((S, C, stride), 0.5, np.float32)
    for s in range(S):
        buf[s, :, :n_in[s]] = xs[s][:, pos[s]:pos[s] + n_in[s]]
        pos[s] += n_in[s]
    y = np.array(g.run(ops, buf, n_out, inputSamples=n_in, playbackRates=rates))
    return {s: y[s, :, :n_out[s]] for s in range(S) if ops[s] in (PROC, FLUSH)}


def _drive_oracle(o, x, calls):
    outs, pos = [], 0
    for op, n_in, n_out, rate in calls:
        seg = x[:, pos:pos + n_in]
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


def _states(g):
    return {n: g.get_state(n) for n in STATE_NAMES}


def _same(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "%s: max diff %g" % (what, np.abs(a - b).max())


def _lineage_scripts(H, lat):
    """Per kind: the calls before the copy and the calls after it (op, n_in, n_out, rate)."""
    P = lambda a, b: (PROC, int(a * H), int(b * H), 0.0)  # noqa: E731
    before = [[P(3.1, 2.5), P(3.0, 2.5)], [P(2.5, 2.5), P(3.2, 2.0)], [P(3.0, 2.5), (SKIP, 0, 0, 0.0)],
              [P(1.0, 2.7), P(3.1, 2.5)], [P(3.0, 2.5), P(3.0, 2.4)]]
    after = [[P(3.0, 2.5), (FLUSH, 0, int(2.3 * H), 1.0), (OSEEK, lat + H // 2, 0, 0.0), P(3.1, 2.5)],
             [(SKIP, 0, 0, 0.0), P(3.0, 2.5), (FLUSH, 0, int(1.5 * H), 0.5), (OSEEK, lat + 5, 0, 0.0)],
             [P(3.1, 2.5), (OSEEK, lat + H, 0, 0.0), P(2.9, 2.5), P(3.0, 2.5)],
             [P(0.9, 2.6), P(3.0, 2.5), (SKIP, 0, 0, 0.0), (FLUSH, 0, int(2.0 * H), 1.0)],
             [P(3.0, 2.5), P(3.0, 2.5), (OSEEK, lat + 3, 0, 0.0), P(2.2, 3.0)]]
    return before, after


# slots 0..4 start as the five kinds, 5..9 as plain or transposed streams that the copy overwrites; then a swap of 0 and
# 1, a fork of kind 0 to slots 1 and 5 (through the swap) and of kind 4 to slots 8 and 9
COPY_DST = [1, 0, 5, 6, 7, 8, 9]
COPY_SRC = [0, 1, 0, 2, 3, 4, 4]


@pytest.mark.parametrize("preset", [False, True], ids=["configure_2_512_128", "preset_default_stereo"])
def test_mixed_batch_copies_swap_and_fork_match_the_oracle(emu_libs, oracle_port, preset):
    cfg = (lambda o: o.presetDefault(2, SR)) if preset else (lambda o: o.configure(2, 512, 128))
    S = 10
    g = _engine(emu_libs["exact"], S)
    cfg(g)
    H, lat = g.intervalSamples(), g.inputLatency()
    others = [PLAIN, (5, 0, 0, False, 0), PLAIN, (0, 0, 2, True, 0), PLAIN]
    _set_params(g, KINDS + others)
    before, after = _lineage_scripts(H, lat)
    n = 20 * H
    x = signals.batch("harmonic", S, 2, n, 48000)
    xa = signals.batch("sweep", 5, 2, n, 48000)  # the input after the copy, per kind
    pos = [0] * S
    outs_before = [[] for _ in range(S)]
    for k in range(2):
        call = [before[s][k] for s in range(5)] + [(PROC, int(2.4 * H), int(2 * H), 0.0)] * 5
        for s, y in _step(g, call, x, pos).items():
            outs_before[s].append(y)
    s0 = _states(g)
    g.copy_streams(COPY_DST, COPY_SRC)
    s1 = _states(g)
    kind = list(range(5)) + [None] * 5  # which kind each slot holds now
    for d, s in zip(COPY_DST, COPY_SRC):
        kind[d] = s
    for slot in range(S):
        for nm in STATE_NAMES:
            assert s1[nm][slot].tobytes() == s0[nm][kind[slot]].tobytes(), (slot, nm)
    xs = [xa[kind[s]] for s in range(S)]
    pos = [0] * S
    outs = [[] for _ in range(S)]
    for k in range(4):
        for s, y in _step(g, [after[kind[s]][k] for s in range(S)], xs, pos).items():
            outs[s].append(y)
    assert g.unserved_random_blocks() == 0
    for slot in range(S):
        twin = kind[slot]  # the slot of the same kind that was not overwritten (or the kind's own copy)
        for a, b in zip(outs[slot], outs[COPY_DST[COPY_SRC.index(twin)]] if twin in (0, 1) else outs[twin]):
            _same(a, b, "slot %d vs its twin" % slot)
    for k in range(5):
        o = _oracle(cfg, KINDS[k])
        ref = _drive_oracle(o, x[k], before[k]) + _drive_oracle(o, xa[k], after[k])
        slot = kind.index(k)
        got = outs_before[k] + outs[slot]
        assert len(got) == len(ref)
        for i, (a, b) in enumerate(zip(got, ref)):
            _same(a, b, "kind %d, output %d" % (k, i))


@pytest.mark.parametrize("dst_exact", [0, 1])
def test_copy_across_engines_with_other_batch_seed_and_tuning(emu_libs, oracle_port, dst_exact):
    """Mono, batch 3 -> batch 7 with another seed, the paired mono chain (tuning key 5) on and exact math off at the copy;
    the destination then runs in exact math and matches the oracle, as the source does."""
    cfg = lambda o: o.configure(1, 512, 128)  # noqa: E731
    prm = [PLAIN, (4, 0, 0, False, 0), (0, 0, 3, True, 150 / SR)]
    src = _engine(emu_libs["exact"], 3)
    cfg(src)
    _set_params(src, prm)
    dst = _engine(emu_libs["exact"], 7, seed=99, exact_math=bool(dst_exact))
    dst.set_tuning(5, 1)
    cfg(dst)
    x = signals.batch("harmonic", 3, 1, 8000, 48000)
    pos = [0, 0, 0]
    first = [(PROC, 400, 320, 0.0), (PROC, 100, 330, 0.0), (PROC, 420, 336, 0.0)]
    b = _step(src, first, x, pos)
    dst_slots = [6, 2, 4]
    dst.copy_streams(dst_slots, [0, 1, 2], src=src)
    dst.set_tuning(3, 1)
    nxt = [[(PROC, 401, 320, 0.0), (PROC, 400, 320, 0.0), (FLUSH, 0, 300, 1.0)],
           [(OSEEK, 600, 0, 0.0), (PROC, 390, 320, 0.0), (PROC, 300, 250, 0.0)]]
    xd = [np.zeros((1, 8000), np.float32)] * 7
    pd = [0] * 7
    for i, s in enumerate(dst_slots):
        xd[s] = x[i]
        pd[s] = pos[i]
    outs_src, outs_dst = [[] for _ in range(3)], [[] for _ in range(3)]
    for call in nxt:
        for s, y in _step(src, call, x, pos).items():
            outs_src[s].append(y)
        dcall = [(SKIP, 0, 0, 0.0)] * 7
        for i, s in enumerate(dst_slots):
            dcall[s] = call[i]
        got = _step(dst, dcall, xd, pd)
        for i, s in enumerate(dst_slots):
            if s in got:
                outs_dst[i].append(got[s])
    assert src.unserved_random_blocks() == 0 and dst.unserved_random_blocks() == 0
    for i in range(3):
        o = _oracle(cfg, prm[i])
        ref = _drive_oracle(o, x[i], [first[i]] + [c[i] for c in nxt])
        assert np.array_equal(b[i], ref[0])
        for k, (a, c, r) in enumerate(zip(outs_src[i], outs_dst[i], ref[1:])):
            _same(a, r, "source %d, output %d" % (i, k))
            _same(c, r, "copy of %d, output %d" % (i, k))


def test_copy_after_a_slow_seek_draws_random_factors(emu_libs, oracle_port):
    """A stream copied right after a seek at rate 0.3 into an engine that never seeked: its next blocks stretch beyond 2x
    and draw random factors there, as in the oracle, and no block goes unserved."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    src = _engine(emu_libs["exact"], 2)
    cfg(src)
    dst = _engine(emu_libs["exact"], 2, seed=5)
    cfg(dst)
    x = signals.batch("harmonic", 2, 2, 6000, 48000)
    pos = [0, 0]
    _step(src, [(PROC, 400, 320, 0.0), (PROC, 400, 320, 0.0)], x, pos)
    _step(src, [(SEEK, 640, 0, 0.3), (PROC, 400, 320, 0.0)], x, pos)
    _step(dst, [(PROC, 400, 320, 0.0), (PROC, 400, 320, 0.0)], x, [0, 0])
    dst.copy_streams([1], [0], src=src)
    xd = [x[1], x[0]]
    pd = [pos[1], pos[0]]
    call = [(PROC, 400, 320, 0.0), (PROC, 400, 320, 0.0)]
    a = _step(src, call, x, pos)[0]
    b = _step(dst, call, xd, pd)[1]
    assert src.unserved_random_blocks() == 0 and dst.unserved_random_blocks() == 0
    o = _oracle(cfg, PLAIN)
    ref = _drive_oracle(o, x[0], [(PROC, 400, 320, 0.0), (SEEK, 640, 0, 0.3), (PROC, 400, 320, 0.0)])
    _same(a, ref[1], "source")
    _same(b, ref[1], "copy")


def test_export_import_round_trip_continues_bit_identically(emu_libs):
    """Records exported from one engine and imported into a fresh one (another batch and seed, the same table): the
    imported streams continue as the originals do, with their parameters."""
    S = 3
    g = _engine(emu_libs["exact"], S)
    g.configure(2, 512, 128)
    _set_params(g, [(2, 0, 0, False, 0), "table", (0, 0, -3, False, 0)])
    x = signals.batch("harmonic", S, 2, 6000, 48000)
    pos = [0] * S
    _step(g, [(PROC, 400, 320, 0.0), (SEEK, 600, 0, 0.4), (PROC, 420, 336, 0.0)], x, pos)
    rec = g.export_streams([0, 1, 2])
    assert rec.shape == (S, g.state_bytes()) and rec.dtype == np.uint8
    h = _engine(emu_libs["exact"], 4, seed=77)
    h.configure(2, 512, 128)
    h.setFreqMapTable(*signals.PWL_MONOTONE)
    h.setTransposeSemitones(0)  # (the table stays, no stream uses it until the import)
    slots = [3, 0, 1]
    h.import_streams(slots, rec)
    assert np.array_equal(h.export_streams(slots)[:, 128:], rec[:, 128:])
    xh = [np.zeros((2, 6000), np.float32)] * 4
    ph = [0] * 4
    for i, s in enumerate(slots):
        xh[s], ph[s] = x[i], pos[i]
    for call in ([(PROC, 400, 320, 0.0), (PROC, 300, 330, 0.0), (FLUSH, 0, 200, 1.0)],
                 [(PROC, 401, 320, 0.0), (PROC, 400, 320, 0.0), (OSEEK, 500, 0, 0.0)]):
        a = _step(g, call, x, pos)
        hc = [(SKIP, 0, 0, 0.0)] * 4
        for i, s in enumerate(slots):
            hc[s] = call[i]
        b = _step(h, hc, xh, ph)
        for i, s in enumerate(slots):
            if i in a:
                _same(a[i], b[s], "stream %d" % i)
    assert g.unserved_random_blocks() == 0 and h.unserved_random_blocks() == 0


def test_clone_continues_like_the_original(emu_libs):
    """clone(): same configuration, tuning, parameters and state; both continue identically.  A clone of an unconfigured
    engine is unconfigured."""
    g = _engine(emu_libs["float"], 3, exact_math=False)
    assert g.clone().channels() == 0
    g.configure(2, 512, 128)
    _set_params(g, [PLAIN, "table", (0, 0, 2, True, 0)])
    x = signals.batch("harmonic", 3, 2, 3000, 48000)
    g.process(x[:, :, :700], 560)
    c = g.clone()
    assert c.channels() == 2 and c.batch == 3
    for nm in STATE_NAMES:
        assert c.get_state(nm).tobytes() == g.get_state(nm).tobytes(), nm
    _same(np.array(g.process(x[:, :, 700:1500], 640)), np.array(c.process(x[:, :, 700:1500], 640)), "clone")


def test_rejected_calls_enqueue_nothing(emu_libs):
    """Every refused call returns B200S_EINVAL, names the offending entry, and leaves launches and state unchanged."""
    S = 3
    g = _engine(emu_libs["float"], S)
    g.configure(2, 512, 128)
    g.setFreqMapTable(*signals.PWL_MONOTONE)
    g.process(signals.batch("harmonic", S, 2, 600, 48000), 500)
    other = _engine(emu_libs["float"], 4)
    other.configure(2, 512, 128)
    mono = _engine(emu_libs["float"], 4)
    mono.configure(1, 512, 128)
    bare = _engine(emu_libs["float"], 4)
    lib, h = g._lib, g._h
    ip = ctypes.POINTER(ctypes.c_int)

    def arr(v):
        return np.array(v, np.int32)

    def copy(dst, d, src, s, n=None):
        d, s = arr(d), arr(s)
        return lib.b200s_copy_streams(dst._h, None if d is None else d.ctypes.data_as(ip), src._h,
                                      None if s is None else s.ctypes.data_as(ip), len(d) if n is None else n)

    def err(e):
        return lib.b200s_last_error(e._h).decode()

    rec = g.export_streams([0, 1])
    state0 = {e: _states(e) for e in (g, other)}
    n0 = {e: e.kernel_launches() for e in (g, other, mono)}
    assert lib.b200s_copy_streams(g._h, None, g._h, arr([0]).ctypes.data_as(ip), 1) == -1 and "dst_streams" in err(g)
    assert lib.b200s_copy_streams(g._h, arr([0]).ctypes.data_as(ip), g._h, None, 1) == -1 and "src_streams" in err(g)
    assert copy(g, [0], g, [1], n=-1) == -1 and "negative" in err(g)
    assert copy(g, [0, 3], g, [1, 2]) == -1 and "dst_streams[1] = 3" in err(g)
    assert copy(g, [0, 1], g, [2, -1]) == -1 and "src_streams[1] = -1" in err(g)
    assert copy(g, [0, 2, 0], g, [1, 1, 2]) == -1 and "dst_streams[2]: stream 0 is listed twice" in err(g)
    assert copy(other, [0], bare, [0]) == -1 and "source engine not configured" in err(other)
    assert copy(bare, [0], g, [0]) == -1 and "destination engine not configured" in err(g)
    assert copy(mono, [0], g, [0]) == -1 and "configurations differ" in err(mono)
    assert copy(other, [0, 1], g, [2, 1]) == -1 and "src_streams[0]: stream 2" in err(other) and "table" in err(other)
    # export / import
    assert lib.b200s_export_streams(h, arr([0, 5]).ctypes.data_as(ip), 2, rec.ctypes.data) == -1 and "streams[1] = 5" in err(g)
    assert lib.b200s_export_streams(h, None, 1, rec.ctypes.data) == -1
    assert lib.b200s_export_streams(h, arr([0]).ctypes.data_as(ip), 1, None) == -1
    assert lib.b200s_export_streams(mono._h, arr([0]).ctypes.data_as(ip), -1, rec.ctypes.data) == -1
    assert bare._lib.b200s_stream_state_bytes(bare._h) == -1
    bad = rec.copy()
    bad[1, 0] ^= 1
    assert lib.b200s_import_streams(h, arr([0, 1]).ctypes.data_as(ip), 2, bad.ctypes.data) == -1 and "record 1: not a stream record" in err(g)
    bad = rec.copy()
    bad[0, 8] += 1
    assert lib.b200s_import_streams(h, arr([0, 1]).ctypes.data_as(ip), 2, bad.ctypes.data) == -1 and "record 0: record format" in err(g)
    assert lib.b200s_import_streams(h, arr([1, 1]).ctypes.data_as(ip), 2, rec.ctypes.data) == -1 and "listed twice" in err(g)
    assert lib.b200s_import_streams(other._h, arr([0, 1]).ctypes.data_as(ip), 2, rec.ctypes.data) == -1 and "record 0" in err(other) and "table" in err(other)
    recm = np.zeros((1, g.state_bytes()), np.uint8)
    recm[0, :128] = rec[0, :128]
    recm[0, 20] = 1  # channels 1 (C is the first field after magic, version and size)
    assert lib.b200s_import_streams(h, arr([0]).ctypes.data_as(ip), 1, recm.ctypes.data) == -1 and "record 0: recorded with another configuration" in err(g)
    with pytest.raises(ValueError):
        g.copy_streams([0, 1], [2])
    with pytest.raises(ValueError):
        g.import_streams([0], rec)
    assert {e: e.kernel_launches() for e in (g, other, mono)} == n0
    for e in (g, other):
        for nm in STATE_NAMES:
            assert state0[e][nm].tobytes() == e.get_state(nm).tobytes(), nm
    launches = g.kernel_launches()
    g.copy_streams([], [])
    assert g.kernel_launches() == launches


FACADE = r"""
#include <cmath>
#include <cstdio>
#include <type_traits>
#include <utility>
#include <vector>
#include "signalsmith-stretch/signalsmith-stretch.h"
using Stretch = signalsmith::stretch::SignalsmithStretch<float>;
static_assert(std::is_copy_constructible<Stretch>::value, "copy-constructible");
static_assert(std::is_copy_assignable<Stretch>::value, "copy-assignable");
static_assert(std::is_move_constructible<Stretch>::value, "move-constructible");
static_assert(std::is_move_assignable<Stretch>::value, "move-assignable");

static std::vector<float> in0(700), in1(700), in2(700);
static int run(Stretch &s, int k, std::vector<float> &o0, std::vector<float> &o1) { // one stereo block of input, returns 0 on success
	float *ins[2] = {in0.data() + 0, (k ? in2 : in1).data()};
	o0.assign(560, 0.f); o1.assign(560, 0.f);
	float *outs[2] = {o0.data(), o1.data()};
	s.process(ins, 700, outs, 560);
	return 0;
}
static bool same(Stretch &a, Stretch &b, int k) {
	std::vector<float> a0, a1, b0, b1;
	run(a, k, a0, a1);
	run(b, k, b0, b1);
	return a0 == b0 && a1 == b1;
}
int main() {
	for (int i = 0; i < 700; ++i) {
		in0[i] = 0.3f * std::sin(0.05f * i);
		in1[i] = 0.2f * std::sin(0.031f * i + 1.f);
		in2[i] = 0.1f * std::sin(0.07f * i);
	}
	Stretch a(7);
	a.configure(2, 512, 128);
	a.setTransposeSemitones(3);
	std::vector<float> o0, o1;
	run(a, 0, o0, o1);
	auto b = a;                              // copy construction
	if (!same(a, b, 1)) { std::puts("copy differs"); return 1; }
	Stretch c;
	c.configure(1, 1024, 256);               // another configuration, replaced by the assignment
	c = a;
	if (!same(a, c, 0)) { std::puts("assignment differs"); return 2; }
	Stretch d = std::move(c);                // move construction
	if (!same(a, d, 1)) { std::puts("move differs"); return 3; }
	Stretch m;
	m = std::move(d);                        // move assignment
	if (!same(a, m, 0)) { std::puts("move assignment differs"); return 4; }
	std::vector<Stretch> v;
	for (int i = 0; i < 3; ++i) v.push_back(a); // reallocation copies or moves the elements
	std::vector<float> r0, r1, e0, e1;
	run(a, 1, r0, r1);
	for (auto &s : v) {
		run(s, 1, e0, e1);
		if (e0 != r0 || e1 != r1) { std::puts("vector element differs"); return 5; }
	}
	std::puts("ok");
	return 0;
}
"""


def test_facade_is_copyable_and_movable(emu_libs, tmp_path):
    """The C++ facade has the reference class's copy and move members: a copy, an assignment over another configuration,
    moves and std::vector::push_back all continue exactly where the original was."""
    src = tmp_path / "facade_copy.cpp"
    src.write_text(FACADE)
    exe = str(tmp_path / "facade_copy")
    d = os.path.dirname(emu_libs["float"])
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src), emu_libs["float"],
                    "-Wl,-rpath," + d], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr


# ------------------------------------------------------------------ H100
def _copy_and_continue(lib, exact, across):
    """presetDefault stereo, the five kinds and plain streams; one call, a copy with a fork (within the engine, or into a
    second engine with another batch and seed), then two calls in which every copy gets its source's ops and input.
    Returns {(call, engine, slot): output} and the (destination slot, source slot) pairs."""
    from signalsmith_stretch_b200 import BatchStretch

    S = 8
    g = BatchStretch(S, lib_path=lib)
    g.presetDefault(2, SR)
    g.set_tuning(3, exact)
    _set_params(g, KINDS + [PLAIN] * 3)
    dst = g
    if across:
        dst = BatchStretch(S + 3, seed=9, lib_path=lib)
        dst.presetDefault(2, SR)
        dst.set_tuning(3, exact)
        dst.setFreqMapTable(*signals.PWL_MONOTONE)  # (the table stream needs the same table there)
        dst.setTransposeSemitones(0)
    H = g.intervalSamples()
    x = signals.batch("harmonic", S, 2, 16 * H, 48000)
    rng = np.random.default_rng(1)
    pos = [0] * S
    _step(g, [(PROC, int(rng.integers(3 * H, 4 * H)), 3 * H + s % 3, 0.0) for s in range(S)], x, pos)
    pairs = list(zip([10, 0, 3, 5, 7, 9], range(5))) + [(1, 4)] if across else [(5, 0), (6, 2), (7, 4), (1, 4)]
    dst.copy_streams([d for d, _ in pairs], [s for _, s in pairs], src=g)
    xd, pd = list(x) + [x[0]] * (dst.batch - S), pos + [0] * (dst.batch - S)
    for d, s in pairs:
        xd[d], pd[d] = x[s], pos[s]
    outs = {}
    for k in (1, 2):
        call = [(PROC, int(rng.integers(3 * H, 4 * H)), 3 * H + int(rng.integers(0, 3)), 0.0) for _ in range(S)]
        if across:
            for s, y in _step(g, call, x, pos).items():
                outs[k, 0, s] = y
            dcall = [(SKIP, 0, 0, 0.0)] * dst.batch
        else:
            dcall = list(call)
        for d, s in pairs:
            dcall[d] = call[s]
        for s, y in _step(dst, dcall, xd, pd).items():
            outs[k, 1, s] = y
    assert g.unserved_random_blocks() == 0 and dst.unserved_random_blocks() == 0
    if not across:  # the sources ran inside the same engine
        outs.update({(k, 0, s): y for (k, e, s), y in list(outs.items())})
    return outs, pairs


@pytest.mark.gpu
@pytest.mark.parametrize("across", [False, True], ids=["one_engine", "two_engines"])
def test_gpu_copies_continue_bit_identically(cuda_lib, emu_libs, across):
    """Copies within one engine or into a second engine on device 0 continue bit-identically to their sources in fast
    arithmetic; in exact arithmetic they also equal the emulator's float build."""
    for exact in (0, 1):
        outs, pairs = _copy_and_continue(None, exact, across)
        for k in (1, 2):
            for d, s in pairs:
                _same(outs[k, 1, d], outs[k, 0, s], "exact %d, call %d, slot %d from %d" % (exact, k, d, s))
        if exact:
            emu, _ = _copy_and_continue(emu_libs["float"], exact, across)
            assert emu.keys() == outs.keys()
            for key in outs:
                _same(outs[key], emu[key], "GPU vs emulator %s" % (key,))


@pytest.mark.gpu
def test_gpu_copy_after_chained_async_calls_equals_copy_after_sync_calls(cuda_lib):
    """A copy enqueued right after chained process_per_stream_async calls on pinned buffers takes the state those calls
    leave, the same as after synchronous calls."""
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C, calls = 48, 2, 3
    e0 = BatchStretch(1)
    e0.presetDefault(C, SR)
    H = e0.intervalSamples()
    in_stride, out_stride = 10 * H, 8 * H
    rng = np.random.default_rng(5)
    lens = [(rng.integers(6 * H, in_stride + 1, S).astype(np.int32), rng.integers(5 * H, out_stride + 1, S).astype(np.int32)) for _ in range(calls)]
    x = signals.batch("harmonic", S, C, (calls + 1) * in_stride, 48000)
    slabs = [np.ascontiguousarray(x[:, :, k * in_stride:(k + 1) * in_stride]) for k in range(calls + 1)]
    recs = []
    for chained in (False, True):
        e = BatchStretch(S)
        e.presetDefault(C, SR)
        e.reserve(in_stride, out_stride)
        dst = BatchStretch(S)
        dst.presetDefault(C, SR)
        pin_in = [torch.from_numpy(slabs[k]).pin_memory() for k in range(calls)]
        pin_out = [torch.empty((S, C, out_stride), dtype=torch.float32).pin_memory() for _ in range(calls)]
        for k in range(calls):
            e.process_per_stream_host_ptr(pin_in[k].data_ptr(), in_stride, lens[k][0], pin_out[k].data_ptr(), out_stride, lens[k][1], wait=not chained)
        dst.copy_streams(np.arange(S)[::-1], np.arange(S), src=e)
        y = dst.process(slabs[calls][::-1].copy(), out_stride)
        e.synchronize()
        recs.append((dst.export_streams(np.arange(S)), np.array(y)))
    assert np.array_equal(recs[0][0][:, 128:], recs[1][0][:, 128:])
    assert np.array_equal(recs[0][1], recs[1][1])


@pytest.mark.gpu
def test_gpu_second_copy_and_import_allocate_nothing(cuda_lib):
    """Copies and imports stage through buffers that grow on first use: calls with at most as many streams allocate
    nothing."""
    from signalsmith_stretch_b200 import BatchStretch

    S = 16
    g, h = BatchStretch(S), BatchStretch(S)
    for e in (g, h):
        e.presetDefault(2, SR)
    g.process(signals.batch("harmonic", S, 2, 12 * 1440, 48000), 9 * 1440)
    h.copy_streams(np.arange(8), np.arange(8, 16), src=g)
    g.copy_streams([0, 1], [2, 3])
    rec = g.export_streams(np.arange(8))
    h.import_streams(np.arange(8, 16), rec)
    h.synchronize()
    g.synchronize()
    before = (g.device_allocations(), h.device_allocations())
    h.copy_streams(np.arange(5), np.arange(3, 8), src=g)
    g.copy_streams([4, 5], [6, 7])
    h.import_streams(np.arange(3), rec[:3])
    g.export_streams(np.arange(8))
    h.synchronize()
    g.synchronize()
    assert (g.device_allocations(), h.device_allocations()) == before


@pytest.mark.gpu
def test_gpu_copy_between_two_devices(cuda_lib):
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    S = 8
    g = BatchStretch(S, device=0)
    g.presetDefault(2, SR)
    h = BatchStretch(S, device=1)
    h.presetDefault(2, SR)
    x = signals.batch("harmonic", S, 2, 30 * 1440, 48000)
    g.process(x[:, :, :10 * 1440], 8 * 1440)
    h.copy_streams(np.arange(S)[::-1], np.arange(S), src=g)
    a = np.array(g.process(x[:, :, 10 * 1440:], 16 * 1440))
    b = np.array(h.process(np.ascontiguousarray(x[::-1, :, 10 * 1440:]), 16 * 1440))
    assert np.array_equal(a[::-1], b)
