"""16-bit PCM forms of the per-stream and listed calls (b200s_run_per_stream_pcm16, b200s_run_streams_pcm16).

Every case drives two engines built the same way: one with the 16-bit call, its twin with the float call (the same list,
ops and counts) fed x16 / 32768, its output converted here the way b200s_process_pcm16's tests convert it: * 32768, round
to nearest with halves away from zero, clamp to int16.  The outputs must be equal sample for sample, the 16-bit output
buffers start filled with 0x7fff so that every sample an op does not produce must have been written as 0, and every
slot's exported record must be equal byte for byte between the twins after every call.
"""
import ctypes

import numpy as np
import pytest

import signals

SR = 48000.0
SKIP, PROC, SEEK, OSEEK, FLUSH, RESET = range(6)
PLAIN = (0, 0, 0, False, 0)
FLAGS = slice(36, 40)  # StreamRecordHeader::flags
FILL = 0x7fff
# configure(2, 512, 128) with plain, transposed (with a tonality limit), formant, and formant-compensated streams (fixed
# base and the automatic pitch estimate)
SIX_PRM = [PLAIN, (3, 0.25, 0, False, 0), PLAIN, (0, 0, 3, False, 0), (5, 0, 0, True, 0), (-5, 0, 0, True, 200 / SR)]


def to_float(x16):
    return x16.astype(np.float32) * np.float32(1 / 32768)


def to_pcm16(v):
    v = v * np.float32(32768)
    return np.clip(np.sign(v) * np.floor(np.abs(v) + np.float32(0.5)), -32768, 32767).astype(np.int16)


def _emu(path, batch, groups=0):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=321, lib_path=path)
    e.set_tuning(3, 1)
    if groups:
        e.set_tuning(2, groups)
    e.configure(2, 512, 128)
    semis, ton, fsemi, comp, base = (np.array(v) for v in zip(*SIX_PRM[:batch] + [PLAIN] * max(0, batch - len(SIX_PRM))))
    e.setTransposeSemitones(semis.astype(np.float32), ton.astype(np.float32))
    e.setFormantSemitones(fsemi.astype(np.float32), comp.astype(bool))
    e.setFormantBase(base.astype(np.float32))
    return e


def _without_flags(rec):
    r = rec.copy()
    r[:, FLAGS] = 0
    return r


class Twins:
    """An engine driven by the 16-bit calls and its twin driven by the float calls; x16[s] ([C][n] int16) is slot s's
    audio, consumed call by call."""

    def __init__(self, make, x16):
        self.pcm, self.flt = make(), make()
        self.x16 = x16
        self.S, self.C = len(x16), self.pcm.channels()
        self.pos = np.zeros(self.S, int)
        self.clamped = [False, False]

    def call(self, streams, ops, n_in=0, n_out=0, rates=None, out_pad=3, in_pad=4):
        """streams None: the whole batch (b200s_run_per_stream_pcm16), else a list (b200s_run_streams_pcm16)."""
        S, C = self.S, self.C
        slots = np.arange(S) if streams is None else np.asarray(streams, np.int32)
        n = slots.size
        ops = np.broadcast_to(np.asarray(ops, np.int32), (n,)).copy()
        n_in = np.broadcast_to(np.asarray(n_in, np.int32), (n,)).copy()
        n_out = np.broadcast_to(np.asarray(n_out, np.int32), (n,)).copy()
        rates = None if rates is None else np.broadcast_to(np.asarray(rates, np.float64), (n,)).copy()
        in_stride = int(n_in.max(initial=0)) + in_pad
        out_stride = int(n_out.max(initial=0)) + out_pad
        buf = np.full((n, C, in_stride), -12345, np.int16)  # (past each stream's count: never read)
        for i, s in enumerate(slots):
            buf[i, :, :n_in[i]] = self.x16[s][:, self.pos[s]:self.pos[s] + n_in[i]]
            self.pos[s] += n_in[i]
        before = self.pcm.export_streams(range(S))
        lst = None if streams is None else slots
        y = self.pcm.run_pcm16(ops, buf, n_out, inputSamples=n_in, playbackRates=rates, streams=lst,
                               out=np.full((n, C, out_stride), FILL, np.int16))
        yf = self.flt.run(ops, to_float(buf), n_out, inputSamples=n_in, playbackRates=rates, streams=lst,
                          out=np.full((n, C, out_stride), np.nan, np.float32))
        assert y.shape == (n, C, out_stride) and y.dtype == np.int16
        assert not np.isnan(yf).any()
        v = yf * np.float32(32768)
        self.clamped[0] |= bool((v < -32768.5).any())
        self.clamped[1] |= bool((v > 32767.5).any())
        want = to_pcm16(yf)
        for i, s in enumerate(slots):
            assert np.array_equal(y[i], want[i]), "entry %d (slot %d, op %d): %d samples differ" % (i, s, ops[i], (y[i] != want[i]).sum())
            assert not y[i, :, n_out[i]:].any(), "entry %d: the tail past output_samples is not zero" % i
        after, twin = self.pcm.export_streams(range(S)), self.flt.export_streams(range(S))
        for s in range(S):
            assert after[s].tobytes() == twin[s].tobytes(), "slot %d: state differs from the float twin's" % s
        unlisted = np.setdiff1d(np.arange(S), slots)
        if unlisted.size:
            assert _without_flags(after[unlisted]).tobytes() == _without_flags(before[unlisted]).tobytes()
        return y


def _twins(emu_libs, S=6, gain=1.0, n=20000, **kw):
    x = signals.batch("harmonic", S, 2, n, 48000) * gain
    x16 = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    return Twins(lambda: _emu(emu_libs["exact"], S, **kw), x16)


def test_ragged_whole_batch_calls_equal_the_float_call(emu_libs):
    """b200s_run_per_stream_pcm16 with PROCESS everywhere (per-stream process()), ragged lengths with (0, 0), (0, n) and
    (n, 0), and an odd input stride; SKIP beside PROCESS."""
    t = _twins(emu_libs)
    t.call(None, PROC, 400, 320)
    t.call(None, PROC, [0, 0, 400, 401, 120, 398], [0, 320, 0, 333, 320, 321], in_pad=3)
    t.call(None, PROC, [300, 500, 640, 100, 256, 400], [400, 400, 320, 330, 320, 500], out_pad=0)
    t.call(None, [PROC, SKIP, PROC, SKIP, PROC, PROC], [400, 0, 380, 0, 400, 420], [320, 0, 300, 0, 320, 336])
    assert t.pcm.unserved_random_blocks() == 0


def test_every_op_in_one_call_and_list_order(emu_libs):
    """PROCESS, SEEK (slow: the random path), OUTPUT_SEEK, FLUSH (rate 1), RESET and SKIP in one whole-batch call and in one
    shuffled list call; a FLUSH at rate 0 (the random path); then the turned-over slots process on."""
    t = _twins(emu_libs)
    t.call(None, PROC, 400, 320)
    t.call(None, [PROC, SEEK, OSEEK, FLUSH, RESET, SKIP], [400, 640, 700, 0, 0, 0], [320, 0, 0, 300, 0, 0],
           rates=[1.0, 0.3, 1.0, 1.0, 1.0, 1.0])
    t.call([5, 1, 3, 0, 4, 2], [PROC, SEEK, OSEEK, FLUSH, RESET, SKIP], [400, 640, 700, 0, 0, 0], [320, 0, 0, 300, 0, 0],
           rates=[1.0, 0.3, 1.0, 1.0, 1.0, 1.0])
    t.call([1, 3, 0, 4], [PROC, PROC, FLUSH, PROC], [300, 400, 0, 400], [320, 320, 500, 320], rates=[1.0, 1.0, 0.0, 1.0])
    t.call([2, 0, 1], PROC, 420, 336)
    t.call(None, PROC, 400, 320)
    assert t.pcm.unserved_random_blocks() == 0


@pytest.mark.parametrize("wide", [False, True], ids=["rows_below_output_latency", "rows_above_output_latency"])
def test_output_seek_pre_roll_and_flush_tails_stay_out_of_the_output(emu_libs, wide):
    """An output seek writes outputLatency samples of pre-roll into its row and the post phase takes it back out; a flush
    writes its tail only in the post phase.  Both must be final before the 16-bit conversion, with rows narrower than
    outputLatency (through the scratch rows) and wider."""
    t = _twins(emu_libs)
    lat = t.pcm.outputLatency()
    n_out = 320 if wide else 40
    assert (n_out > lat) == wide
    t.call(None, PROC, 400, 320)
    t.call([4, 1, 2, 0], [OSEEK, PROC, OSEEK, FLUSH], [600, n_out + 60, 650, 0], [0, n_out, 0, n_out], rates=1.0, out_pad=0)
    t.call(None, [OSEEK, FLUSH, PROC, PROC, PROC, OSEEK], [600, 0, 400, 400, 400, 700], [0, n_out, n_out, n_out, n_out, 0],
           rates=[1.0, 0.0, 1.0, 1.0, 1.0, 1.0], out_pad=0)
    t.call([1, 4, 2, 0], PROC, 300, 320)


def test_loud_input_hits_both_clamps(emu_libs):
    """A signal at about 3x full scale, clipped on the way in: the output passes both ends of the 16-bit range."""
    t = _twins(emu_libs, gain=3.0)
    for k in range(3):
        t.call(None, PROC, 400, 320)
        t.call([3, 0, 5], PROC, [400, 300, 500], 320)
    assert t.clamped == [True, True]


def _ptr(a):
    return None if a is None else a.ctypes.data


def test_async_sequences_equal_synchronous_calls(emu_libs):
    """wait = 0: the same list three times (chained stream groups), another list, a float call on the first list in
    between, the first list again, a whole-batch call and a turnover call, then one synchronise: the outputs and state of
    the same calls with wait = 1."""
    S, C = 6, 2
    n_in, n_out = 400, 320
    x = signals.batch("harmonic", S, C, 8000, 48000)
    x16 = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    A, B = [4, 1, 5, 0], [0, 2, 4, 5, 3]
    # (list or None for the whole batch, ops, format)
    seq = [(A, PROC, 16), (A, PROC, 16), (A, PROC, 16), (B, PROC, 16), (A, PROC, 32), (A, PROC, 16), (None, PROC, 16),
           (A, [FLUSH, PROC, OSEEK, PROC], 16), (A, PROC, 16)]
    runs = []
    for wait in (True, False):
        e = _emu(emu_libs["exact"], S, groups=2)  # two stream groups (at least two entries each): the chained pipeline
        outs = []
        for k, (lst, ops, fmt) in enumerate(seq):
            slots = np.arange(S) if lst is None else np.array(lst)
            o = np.broadcast_to(np.asarray(ops, np.int32), (slots.size,)).copy()
            ni = np.where(o == PROC, n_in, np.where(o == OSEEK, 700, 0)).astype(np.int32)
            no = np.where((o == PROC) | (o == FLUSH), n_out, 0).astype(np.int32)
            src = np.ascontiguousarray(x16[slots][:, :, k * 700:k * 700 + 700])
            if fmt == 16:
                out = np.full((slots.size, C, n_out), FILL, np.int16)
                e.run_pcm16_host_ptr(o, _ptr(src), 700, ni, _ptr(out), n_out, no, playback_rates=1.0, streams=lst, wait=wait)
            else:
                src = to_float(src)
                out = np.full((slots.size, C, n_out), np.nan, np.float32)
                e.run_streams_host_ptr(lst, o, _ptr(src), 700, ni, _ptr(out), n_out, no, playback_rates=1.0, wait=wait)
            outs.append((src, out))  # (the buffers stay alive until the synchronise)
        e.synchronize()
        runs.append((e, [o for _, o in outs]))
    for k in range(len(seq)):
        assert np.array_equal(runs[0][1][k], runs[1][1][k], equal_nan=True), k
        assert np.any(runs[0][1][k] != 0), k
    assert runs[0][0].export_streams(range(S)).tobytes() == runs[1][0].export_streams(range(S)).tobytes()


def test_arguments_are_refused_as_by_the_float_calls(emu_libs):
    """Every rule of the float counterpart returns B200S_EINVAL with the same message, before anything is enqueued or
    allocated; the state is unchanged."""
    S, C = 4, 2
    g = _emu(emu_libs["float"], S)
    g.process(signals.batch("harmonic", S, C, 600, 48000), 500)
    lib, h = g._lib, g._h
    ip, dp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)
    buf16, out16 = np.zeros((S, C, 256), np.int16), np.zeros((S, C, 256), np.int16)
    buf, out = np.zeros((S, C, 256), np.float32), np.zeros((S, C, 256), np.float32)
    rates = np.ones(S)

    def arr(v):
        return np.array(v, np.int32)

    def p(a, t=ip):
        return None if a is None else a.ctypes.data_as(t)

    def err(fn):
        m = lib.b200s_last_error(h).decode()
        assert m.startswith(fn + ": "), m
        return m[len(fn) + 2:]

    # each case: the float call, then the 16-bit call with wait = 0 and 1, as (function name, call)
    def listed(n=2, lst=arr([1, 3]), ops=arr([PROC, PROC]), ni=arr([10, 10]), no=arr([10, 10]), r=rates, si=256, so=256):
        a = (n, p(lst), p(ops))
        return [("b200s_run_streams", lambda: lib.b200s_run_streams(h, *a, buf.ctypes.data, si, p(ni), out.ctypes.data, so, p(no), p(r, dp)))] + \
            [("b200s_run_streams_pcm16", lambda w=w: lib.b200s_run_streams_pcm16(h, *a, buf16.ctypes.data, si, p(ni), out16.ctypes.data, so, p(no),
                                                                                  p(r, dp), w)) for w in (0, 1)]

    def whole(ops=arr([PROC] * S), ni=arr([10] * S), no=arr([10] * S), r=rates, si=256, so=256):
        return [("b200s_run_per_stream", lambda: lib.b200s_run_per_stream(h, p(ops), buf.ctypes.data, si, p(ni), out.ctypes.data, so, p(no), p(r, dp)))] + \
            [("b200s_run_per_stream_pcm16", lambda w=w: lib.b200s_run_per_stream_pcm16(h, p(ops), buf16.ctypes.data, si, p(ni), out16.ctypes.data, so,
                                                                                        p(no), p(r, dp), w)) for w in (0, 1)]

    rec0 = g.export_streams(range(S))
    n0, a0 = g.kernel_launches(), g.device_allocations()
    cases = [
        listed(n=-1), listed(n=S + 1, lst=arr(range(S + 1)), ops=arr([PROC] * (S + 1)), ni=arr([1] * (S + 1)), no=arr([1] * (S + 1))),
        listed(lst=None), listed(ops=None), listed(ni=None), listed(no=None), listed(lst=arr([1, S])), listed(lst=arr([-1, 0])),
        listed(lst=arr([2, 2])), listed(ops=arr([PROC, 6])), listed(ops=arr([SEEK, PROC]), r=None), listed(ops=arr([FLUSH, PROC]), ni=arr([5, 10])),
        listed(ops=arr([PROC, RESET]), ni=arr([10, 0])), listed(ops=arr([OSEEK, PROC]), no=arr([5, 10])), listed(ni=arr([10, 257])),
        listed(no=arr([-2, 10])), listed(si=-1), listed(so=-1),
        whole(ops=None), whole(ni=None), whole(no=None), whole(ops=arr([PROC, PROC, -1, PROC])), whole(ops=arr([SEEK] + [PROC] * 3), r=None),
        whole(ops=arr([SKIP] * S), ni=arr([0, 0, 0, 3])), whole(ops=arr([SEEK] * S), no=arr([0, 1, 0, 0])), whole(ni=arr([10, 10, 10, 300])),
        whole(no=arr([10, -1, 10, 10])), whole(si=-1), whole(so=-1),
    ]
    for case in cases:
        msgs = []
        for fn, call in case:
            assert call() == -1, fn
            msgs.append(err(fn))
        assert msgs[0] and msgs[1] == msgs[0] and msgs[2] == msgs[0], msgs
    assert lib.b200s_run_streams_pcm16(h, 0, None, None, None, 0, None, None, 0, None, None, 1) == 0  # n == 0: nothing to do
    assert g.kernel_launches() == n0 and g.device_allocations() == a0
    assert g.export_streams(range(S)).tobytes() == rec0.tobytes()
    with pytest.raises(ValueError):
        g.run_pcm16(PROC, buf16[:2], [10, 10, 10], streams=[0, 1])
    with pytest.raises(ValueError):
        g.run_pcm16(PROC, buf16, 10, streams=[0, 1])  # four rows for two entries
    with pytest.raises(ValueError):
        g.run_pcm16(PROC, buf, 10)  # float samples

    class CudaTensor:  # what run_pcm16 sees of a torch CUDA tensor
        is_cuda = True
        shape = buf16.shape

        def data_ptr(self):
            return 0

    with pytest.raises(TypeError):
        g.run_pcm16(PROC, CudaTensor(), 10)


def test_sixteen_bit_slabs_allocate_once_at_the_largest_strides(emu_libs):
    """The first 16-bit call at the largest strides and positions allocates the two 16-bit slabs; later calls at no larger
    strides or positions, turnovers and lists included, allocate nothing beyond what the float twin allocates."""
    t = _twins(emu_libs, n=40000)
    for e in (t.pcm, t.flt):
        e.reserve(700, 400)
    a_pcm, a_flt = t.pcm.device_allocations(), t.flt.device_allocations()
    t.call(None, PROC, 697, 397)  # strides 701 / 400: past what reserve sized for the float rows
    extra = (t.pcm.device_allocations() - a_pcm) - (t.flt.device_allocations() - a_flt)
    assert extra == 2
    t.call([5, 1, 3], PROC, 500, 320)
    t.call([2, 0, 4], [OSEEK, PROC, FLUSH], [600, 190, 0], [0, 150, 200], rates=[1.0, 1.0, 0.0], out_pad=0)
    t.call(None, [PROC] * 6, 400, [300, 300, 0, 300, 300, 300])
    t.call([3, 2, 1, 0, 5, 4], PROC, 125, 100)
    assert (t.pcm.device_allocations() - a_pcm) - (t.flt.device_allocations() - a_flt) == 2
