"""The windowProducts divisor of the paired synthesis kernel (k_synth2, the preset sizes 3072 and 2560).

k_synth2 carries no windowProducts ring: each emitted sample computes its divisor from the block schedule -- a table
entry per phase where the call's blocks cover it as a full run H apart, the carried value plus the call's own terms at
the start of a call and in the ring's tail.  Under the CPU emulator (exact arithmetic, the oracle's FFT swapped in):

* after every call, the carried windowProducts state (pendingWp) equals, bit for bit, a plain replay of the reference's
  ring accumulation (:397-399, :408-414): every block adds window^2 * N to the ring, oldest first, and every emitted slot
  is cleared to ALMOST_ZERO; and the outputs equal those of the generic synthesis kernel (k_synth), which still carries
  the ring;
* under per-stream operations (reset, seek, flush, output seek, SKIP, per-stream lengths with idle streams) the state
  and the outputs equal the generic kernel's after every call, and the outputs equal the one-stream oracle's.
"""
import math

import numpy as np
import pytest

import signals

SR = 48000.0
ALMOST_ZERO = np.float32(1e-30)
SKIP, PROC, SEEK, OSEEK, FLUSH, RESET = range(6)


def _emu(path, batch, generic=False):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=321, lib_path=path)
    e.set_tuning(3, 1)
    if generic:
        e.set_tuning(1, 1)  # the first-generation kernels: k_synth with its windowProducts ring in shared memory
    return e


def _win_prod(B, H, N):
    """window[i]^2 * N in float: the Kaiser window with forced perfect reconstruction of DynamicSTFT::configure."""

    def bessel0(x):
        s, term, q = 1.0, 1.0, x * x * 0.25
        for k in range(1, 200):
            term *= q / (float(k) * k)
            s += term
            if term < s * 1e-17:
                break
        return s

    bw = B / H
    bw += 8 / ((bw + 3) * (bw + 3)) + 0.25 * max(3 - bw, 0.0)
    bw = max(bw, 2.0)
    beta = math.pi * math.sqrt(bw * bw * 0.25 - 1)
    w = [bessel0(beta * math.sqrt(max(0.0, 1 - ((2.0 * i + 1) / B - 1) ** 2))) / bessel0(beta) for i in range(B)]
    for i in range(min(H, B)):
        s2 = 0.0
        for k in range(i, B, H):
            s2 += w[k] * w[k]
        f = 1 / math.sqrt(s2)
        for k in range(i, B, H):
            w[k] *= f
    win = np.array(w, np.float32)
    return (win * win) * np.float32(N)


class RingReplay:
    """The reference's windowProducts ring of one channel over process() calls, linearised: slot 0 is the next output."""

    def __init__(self, e, start):
        self.B, self.H = e.blockSamples(), e.intervalSamples()
        self.add_off = self.H if e.splitComputation() else 0
        self.win_prod = _win_prod(self.B, self.H, e.fftSamples())
        self.ring = np.array(start, np.float32)
        self.since_last = None  # samplesSinceLast: "never" after configure / reset

    def _emit(self, n):
        P = len(self.ring)
        if n >= P:
            self.ring[:] = ALMOST_ZERO
        elif n > 0:
            self.ring = np.concatenate([self.ring[n:], np.full(n, ALMOST_ZERO, np.float32)])

    def process(self, n_out):
        H = self.H
        t = 0 if self.since_last is None or self.since_last >= H else H - self.since_last
        emitted, last = 0, None
        while t < n_out:  # :281-286
            self._emit(t - emitted)
            emitted = last = t
            seg = slice(self.add_off, self.add_off + self.B)
            self.ring[seg] = self.ring[seg] + self.win_prod
            t += H
        self._emit(n_out - emitted)
        if last is not None:
            self.since_last = n_out - last
        elif self.since_last is not None:
            self.since_last += n_out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


PRESETS = [
    ("default_stereo", lambda o: o.presetDefault(2, SR), 2, 1440),
    ("cheaper_split_mono", lambda o: o.presetCheaper(1, SR), 1, 1920),
]


@pytest.mark.parametrize("name,cfg,C,H", PRESETS, ids=[p[0] for p in PRESETS])
def test_pending_wp_equals_ring_replay_over_call_lengths(emu_libs, name, cfg, C, H):
    """Calls of 32 blocks, of a few samples, shorter than the ring, not multiples of four, and empty: the first samples of a
    call (carried values), the steady run (the table) and the tail all meet the replay after every call."""
    lengths = [32 * H, 3 * H + 5, 17, H - 1, 0, 2 * H + 2, 5 * H, 9 * H + 3]
    n_in = [int(round(n / 0.8)) for n in lengths]
    x = signals.batch("harmonic", 2, C, sum(n_in), 48000)
    e, gen = _emu(emu_libs["exact"], 2), _emu(emu_libs["exact"], 2, generic=True)
    for g in (e, gen):
        cfg(g)
    start = e.get_state("pendingWp")
    replay = RingReplay(e, start[0, 0])
    pos = 0
    for k, (n, ni) in enumerate(zip(lengths, n_in)):
        seg = np.ascontiguousarray(x[:, :, pos:pos + ni])
        pos += ni
        y, yg = e.process(seg, n), gen.process(seg, n)
        replay.process(n)
        wp = e.get_state("pendingWp")
        for s in range(2):
            for c in range(C):
                assert np.array_equal(_bits(wp[s, c]), _bits(replay.ring)), (k, s, c, np.flatnonzero(wp[s, c] != replay.ring)[:8])
        assert np.array_equal(_bits(wp), _bits(gen.get_state("pendingWp"))), k
        assert np.array_equal(_bits(y), _bits(yg)), (k, np.abs(y - yg).max())


def _script_run(g, x, script):
    """script: per call, per stream (op, n_in, n_out, rate); stream s's inputs are consecutive pieces of x[s]."""
    S, C = x.shape[:2]
    pos = np.zeros(S, int)
    for call in script:
        ops = np.array([t[0] for t in call], np.int32)
        n_in = np.array([t[1] for t in call], np.int32)
        n_out = np.array([t[2] for t in call], np.int32)
        rates = np.array([t[3] for t in call], np.float64)
        buf = np.zeros((S, C, (int(n_in.max()) + 7) // 4 * 4), np.float32)
        for s in range(S):
            buf[s, :, :n_in[s]] = x[s, :, pos[s]:pos[s] + n_in[s]]
        pos += n_in
        yield ops, n_out, np.array(g.run(ops, buf, n_out, inputSamples=n_in, playbackRates=rates))


def _norm(script):
    return [[tuple(list(t) + [0] * (4 - len(t))) for t in call] for call in script]


def _oracle_outputs(cfg, xs, script, s):
    from oracle.hdrref import CpuStretch

    o = CpuStretch("orc", 321)
    cfg(o)
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


H_D, H_C = 1440, 1920
N_D = int(round(7 * H_D / 0.8))
# one row per call, one column per stream
OPS = [
    # presetDefault stereo: s0 resets and seeks, s1 output-seeks and flushes at rate 1 and 0, s2 runs short calls and sits two
    # out, s3 runs lengths that are not multiples of four, a call of 14 blocks and an output seek
    ("default_stereo", lambda o: o.presetDefault(2, SR), 2, _norm([
        [(PROC, N_D, 7 * H_D), (OSEEK, 7000), (PROC, 1000, 800), (PROC, N_D + 3, 7 * H_D + 3)],
        [(RESET,), (PROC, N_D, 7 * H_D), (SKIP,), (PROC, 401, 321)],
        [(SEEK, 6000, 0, 1.0), (FLUSH, 0, 3 * H_D + 1, 1.0), (SKIP,), (PROC, 2 * N_D, 14 * H_D + 6)],
        [(PROC, 3 * H_D, 2 * H_D + 5), (PROC, N_D, 7 * H_D), (PROC, 40, 32), (OSEEK, 6500)],
        [(PROC, N_D, 7 * H_D), (FLUSH, 0, H_D - 3, 0.0), (PROC, N_D, 7 * H_D), (PROC, 900, 5 * H_D)],
    ])),
    # presetCheaper mono, split computation (the blocks land H into the ring)
    ("cheaper_split_mono", lambda o: o.presetCheaper(1, SR), 1, _norm([
        [(PROC, 12 * H_C, 10 * H_C), (OSEEK, 9000), (PROC, 10 * H_C + 1, 10 * H_C - 3)],
        [(FLUSH, 0, 5 * H_C + 7, 1.0), (PROC, 8 * H_C, 6 * H_C), (RESET,)],
        [(SEEK, 8000, 0, 1.0), (SKIP,), (PROC, 9 * H_C, 8 * H_C)],
        [(PROC, 7 * H_C, 7 * H_C), (PROC, 50, 40), (FLUSH, 0, H_C - 5, 1.0)],
    ])),
]


@pytest.mark.parametrize("name,cfg,C,script", OPS, ids=[p[0] for p in OPS])
def test_pending_wp_and_outputs_under_per_stream_ops(emu_libs, oracle_port, name, cfg, C, script):
    S = len(script[0])
    total = [sum(call[s][1] for call in script) for s in range(S)]
    x = signals.batch("harmonic", S, C, max(total), 48000)
    e, gen = _emu(emu_libs["exact"], S), _emu(emu_libs["exact"], S, generic=True)
    for g in (e, gen):
        cfg(g)
    ys = [[] for _ in range(S)]
    for k, ((ops, n_out, y), (_, _, yg)) in enumerate(zip(_script_run(e, x, script), _script_run(gen, x, script))):
        assert np.array_equal(_bits(e.get_state("pendingWp")), _bits(gen.get_state("pendingWp"))), k
        assert np.array_equal(_bits(e.get_state("pending")), _bits(gen.get_state("pending"))), k
        assert np.array_equal(_bits(y), _bits(yg)), (k, np.abs(y - yg).max())
        for s in range(S):
            if ops[s] in (PROC, FLUSH):
                ys[s].append(y[s, :, :n_out[s]])
    for s in range(S):
        ref = _oracle_outputs(cfg, x[s], script, s)
        assert len(ys[s]) == len(ref)
        for k, (a, b) in enumerate(zip(ys[s], ref)):
            assert np.array_equal(_bits(a), _bits(b)), (s, k, np.abs(a - b).max())
