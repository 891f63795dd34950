"""Calls over a list of streams (b200s_run_streams*): only the listed slots run, with packed buffers [n][channels][stride].

Every case drives two engines built the same way: one with the list call, its twin with b200s_run_per_stream, the same ops
at the listed slots and SKIP everywhere else, the rows scattered to their slots.  The listed outputs must be equal bit for
bit, every slot's exported record must be equal byte for byte between the twins afterwards, and a slot that is not listed
must keep its record.  (The header's random-path flags are engine-wide hints of which kernels a call launches, and any
call may set them; they are compared between the twins but not against the record before the call.)
"""
import ctypes

import numpy as np
import pytest

import signals

SR = 48000.0
SKIP, PROC, SEEK, OSEEK, FLUSH, RESET = range(6)
PLAIN = (0, 0, 0, False, 0)
FLAGS = slice(36, 40)  # StreamRecordHeader::flags


def _emu(path, batch, seed=321, pairs=False, gen=0):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, seed=seed, lib_path=path)
    e.set_tuning(3, 1)
    if gen:
        e.set_tuning(0, gen)
    if pairs:
        e.set_tuning(5, 1)
    return e


def _set_batch(e, prm):
    semis, ton, fsemi, comp, base = (np.array(v) for v in zip(*prm))
    e.setTransposeSemitones(semis.astype(np.float32), ton.astype(np.float32))
    e.setFormantSemitones(fsemi.astype(np.float32), comp.astype(bool))
    e.setFormantBase(base.astype(np.float32))


def _without_flags(rec):
    r = rec.copy()
    r[:, FLAGS] = 0
    return r


class Twins:
    """An engine driven by list calls and its twin driven by the equivalent whole-batch calls; x[s] ([C][n]) is slot s's
    audio, consumed call by call."""

    def __init__(self, make, x, S=None):
        self.sub, self.full = make(), make()
        self.x = x
        self.S = len(x) if S is None else S
        self.C = self.sub.channels()
        self.pos = np.zeros(self.S, int)

    def call(self, streams, ops, n_in=0, n_out=0, rates=None, out_pad=3, fill=0.75, check=True):
        S, C = self.S, self.C
        lst = np.asarray(streams, np.int32)
        n = lst.size
        ops = np.broadcast_to(np.asarray(ops, np.int32), (n,)).copy()
        n_in = np.broadcast_to(np.asarray(n_in, np.int32), (n,)).copy()
        n_out = np.broadcast_to(np.asarray(n_out, np.int32), (n,)).copy()
        rates = None if rates is None else np.broadcast_to(np.asarray(rates, np.float64), (n,)).copy()
        in_stride = (int(n_in.max(initial=0)) + 4 + 3) // 4 * 4
        out_stride = int(n_out.max(initial=0)) + out_pad
        buf = np.full((n, C, in_stride), fill, np.float32)
        for i, s in enumerate(lst):
            assert self.pos[s] + n_in[i] <= self.x[s].shape[-1]
            buf[i, :, :n_in[i]] = self.x[s][:, self.pos[s]:self.pos[s] + n_in[i]]
            self.pos[s] += n_in[i]
        # the twin: the same ops at the listed slots, SKIP elsewhere
        f_ops, f_in, f_out = np.full(S, SKIP, np.int32), np.zeros(S, np.int32), np.zeros(S, np.int32)
        f_rates = None if rates is None else np.ones(S)
        f_buf = np.zeros((S, C, in_stride), np.float32)
        f_ops[lst], f_in[lst], f_out[lst], f_buf[lst] = ops, n_in, n_out, buf
        if rates is not None:
            f_rates[lst] = rates
        before = self.sub.export_streams(range(S)) if check else None
        y = self.sub.run(ops, buf, n_out, inputSamples=n_in, playbackRates=rates, streams=lst,
                         out=np.full((n, C, out_stride), np.nan, np.float32))
        yf = self.full.run(f_ops, f_buf, f_out, inputSamples=f_in, playbackRates=f_rates,
                           out=np.full((S, C, out_stride), np.nan, np.float32))
        assert y.shape == (n, C, out_stride)
        for i, s in enumerate(lst):
            assert np.array_equal(y[i].view(np.uint32), yf[s].view(np.uint32)), \
                "entry %d (slot %d, op %d): max diff %g" % (i, s, ops[i], np.nanmax(np.abs(y[i] - yf[s])))
        if check:
            self.check_records(before, lst)
        return y

    def check_records(self, before, lst):
        after, twin = self.sub.export_streams(range(self.S)), self.full.export_streams(range(self.S))
        for s in range(self.S):
            assert after[s].tobytes() == twin[s].tobytes(), "slot %d: state differs from the twin's" % s
        unlisted = np.setdiff1d(np.arange(self.S), lst)
        if unlisted.size:
            assert _without_flags(after[unlisted]).tobytes() == _without_flags(before[unlisted]).tobytes()


# configure(2, 512, 128) with plain, mapped, formant (fixed base and the automatic pitch estimate) streams
SIX_PRM = [PLAIN, (3, 0.25, 0, False, 0), PLAIN, (0, 0, 3, False, 0), (5, 0, 0, True, 0), (-5, 0, 0, True, 200 / SR)]


def _six(emu_libs, **kw):
    def make():
        e = _emu(emu_libs["exact"], 6, **kw)
        e.configure(2, 512, 128)
        _set_batch(e, SIX_PRM)
        return e

    return Twins(make, signals.batch("harmonic", 6, 2, 12000, 48000))


def test_lists_of_every_shape_equal_the_per_stream_call(emu_libs):
    """Empty, one slot, every slot in order, every slot permuted, a random strict subset, with 0.8x, 1.25x and (slot 2)
    beyond-2x calls that take the random path; every stream's parameters are its own."""
    t = _six(emu_libs)
    rng = np.random.default_rng(5)
    n0 = t.sub.kernel_launches()
    y = t.sub.run(np.zeros(0, np.int32), None, np.zeros(0, np.int32), streams=[])
    assert y.shape == (0, 2, 0) and t.sub.kernel_launches() == n0  # n == 0 enqueues nothing
    t.call([], [])
    t.call([3], PROC, 400, 320)
    t.call(range(6), PROC, [400, 401, 120, 398, 400, 402], [320, 320, 320, 333, 320, 321])
    t.call([4, 0, 5, 2, 1, 3], PROC, [300, 500, 640, 100, 256, 400], [400, 400, 320, 330, 320, 500])
    for _ in range(3):
        lst = rng.permutation(6)[:rng.integers(2, 6)]
        n_out = rng.integers(250, 400, lst.size)
        n_in = np.where(lst == 2, n_out // 3, (n_out * rng.uniform(0.8, 1.25, lst.size)).astype(int))
        t.call(lst, PROC, n_in, n_out)
    assert t.sub.unserved_random_blocks() == 0


def test_every_op_kind_in_one_list_call(emu_libs):
    """PROCESS, SEEK (slow: the random path), OUTPUT_SEEK, FLUSH (rate 1, rate 0), RESET and SKIP in one call, listed out
    of slot order, then the turned-over slots process on, listed with others."""
    t = _six(emu_libs)
    t.call(range(6), PROC, 400, 320)
    t.call([5, 1, 3, 0, 4, 2], [PROC, SEEK, OSEEK, FLUSH, RESET, SKIP], [400, 640, 700, 0, 0, 0], [320, 0, 0, 300, 0, 0],
           rates=[1.0, 0.3, 1.0, 1.0, 1.0, 1.0])
    t.call([1, 3, 0, 4], [PROC, PROC, FLUSH, PROC], [300, 400, 0, 400], [320, 320, 500, 320], rates=[1.0, 1.0, 0.0, 1.0])
    t.call([2, 0, 1], PROC, 420, 336)
    assert t.sub.unserved_random_blocks() == 0


def test_narrow_rows_take_the_output_seeks_through_the_packed_scratch(emu_libs):
    """Output rows narrower than outputLatency: the output seeks' pre-roll goes through the [n][C][outputLatency] scratch,
    indexed by list position."""
    t = _six(emu_libs)
    t.call(range(6), PROC, 400, 320)
    t.call([4, 1, 2], [OSEEK, PROC, OSEEK], [600, 200, 650], [0, 40, 0], out_pad=0)
    t.call([1, 4, 2, 0], PROC, 300, 320)


@pytest.mark.parametrize("gen", [4, 6])
def test_stereo_chain_generations(emu_libs, gen):
    """presetDefault stereo (k_analyse2, k_chain_direct4 / 6, k_synth2): lists in and out of slot order."""
    H = 1440

    def make():
        e = _emu(emu_libs["exact"], 4, gen=gen)
        e.presetDefault(2, SR)
        return e

    t = Twins(make, signals.batch("harmonic", 4, 2, 40000, 48000))
    t.call([2, 0, 3], PROC, 7200, 6 * H)
    t.call([3, 1, 0], PROC, [6000, 9000, 7000], [5 * H, 7 * H, 6 * H - 3])
    t.call([1, 2], [FLUSH, PROC], [0, 7000], [3 * H, 5 * H], rates=1.0)


def test_mono_pairs_follow_the_list(emu_libs):
    """Mono streams two per warp (tuning key 5): the pairs are list neighbours, here slots far apart, and a pair whose
    schedules differ runs one stream at a time."""
    def make():
        e = _emu(emu_libs["exact"], 7, pairs=True)
        e.configure(1, 512, 128)
        return e

    t = Twins(make, signals.batch("harmonic", 7, 1, 9000, 48000))
    t.call(range(7), PROC, 400, 320)
    t.call([6, 0, 3, 5, 1], PROC, 400, 320)
    t.call([2, 4, 6, 1, 0], PROC, [400, 400, 300, 400, 500], [320, 320, 320, 300, 320])
    t.call([5, 2, 3], PROC, 400, 320)


def test_async_list_calls_chain_and_equal_synchronous_calls(emu_libs):
    """Consecutive b200s_run_streams_async calls with one list, then another list, then the first again: the same outputs
    and state as b200s_run_streams."""
    S, C = 6, 2
    x = signals.batch("harmonic", S, C, 8000, 48000)
    lists = [[4, 1, 5, 0], [4, 1, 5, 0], [4, 1, 5, 0], [0, 2, 4, 5, 3], [4, 1, 5, 0]]
    n_in, n_out = 400, 320
    slabs = [np.ascontiguousarray(x[np.array(l)][:, :, k * n_in:(k + 1) * n_in]) for k, l in enumerate(lists)]
    engines = []
    for use_async in (False, True):
        e = _emu(emu_libs["exact"], S)
        e.configure(C, 512, 128)
        _set_batch(e, SIX_PRM)
        e.set_tuning(2, 2)  # two stream groups (at least two entries each): the chained pipeline at these small lists
        outs = [np.full((len(l), C, n_out), np.nan, np.float32) for l in lists]
        for k, l in enumerate(lists):
            if use_async:
                e.run_streams_host_ptr(l, PROC, slabs[k].ctypes.data, n_in, n_in, outs[k].ctypes.data, n_out, n_out)
            else:
                e.run(PROC, slabs[k], n_out, streams=l, out=outs[k])
        e.synchronize()
        engines.append((e, outs))
    for k in range(len(lists)):
        assert np.array_equal(engines[0][1][k], engines[1][1][k]), k
    assert engines[0][0].export_streams(range(S)).tobytes() == engines[1][0].export_streams(range(S)).tobytes()


def test_process_with_streams_equals_run(emu_libs):
    """process(..., streams=) is run(OP_PROCESS, ..., streams=)."""
    t = _six(emu_libs)
    x = signals.batch("harmonic", 3, 2, 500, 48000)
    e = t.sub
    y = e.process(x, 300, streams=[5, 0, 2])
    y2 = t.full.run(PROC, x, 300, streams=[5, 0, 2])
    assert y.shape == (3, 2, 300) and np.array_equal(y, y2)


def test_list_arguments_are_validated(emu_libs):
    """Every refused call returns B200S_EINVAL before anything is enqueued and names the entry; the state is unchanged."""
    S, C = 4, 2
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

    def err():
        return lib.b200s_last_error(h).decode()

    rec0 = g.export_streams(range(S))
    n0 = g.kernel_launches()
    for fn in ("b200s_run_streams", "b200s_run_streams_async", "b200s_run_streams_device"):
        f = getattr(lib, fn)

        def A(n=2, lst=arr([1, 3]), ops=arr([PROC, PROC]), ni=arr([10, 10]), no=arr([10, 10]), r=rates, si=256, so=256):
            p = lambda a, t=ip: None if a is None else a.ctypes.data_as(t)  # noqa: E731
            return f(h, n, p(lst), p(ops), buf.ctypes.data, si, p(ni), out.ctypes.data, so, p(no), p(r, dp))

        assert A(n=-1) == -1 and "n = -1" in err()
        assert A(n=S + 1, lst=arr(range(S + 1)), ops=arr([PROC] * (S + 1)), ni=arr([1] * (S + 1)), no=arr([1] * (S + 1))) == -1
        assert A(lst=None) == -1 and "streams must not be NULL" in err()
        assert A(ops=None) == -1 and A(ni=None) == -1 and A(no=None) == -1
        assert A(lst=arr([1, S])) == -1 and "streams[1] = %d" % S in err()
        assert A(lst=arr([-1, 0])) == -1 and "streams[0] = -1" in err()
        assert A(lst=arr([2, 2])) == -1 and "listed twice" in err()
        assert A(ops=arr([PROC, 6])) == -1 and "entry 1 (stream 3)" in err()
        assert A(ops=arr([SEEK, PROC]), r=None) == -1 and "entry 0 (stream 1)" in err()
        assert A(ops=arr([FLUSH, PROC]), ni=arr([5, 10])) == -1 and "entry 0" in err()
        assert A(ops=arr([PROC, RESET]), ni=arr([10, 0])) == -1 and "entry 1" in err()
        assert A(ni=arr([10, 257])) == -1 and "entry 1" in err()
        assert A(no=arr([-2, 10])) == -1 and "entry 0" in err()
        assert A(si=-1) == -1 and A(so=-1) == -1
        assert A(n=0, lst=None, ops=None, ni=None, no=None, r=None) == 0  # n == 0: nothing to check, nothing enqueued
    assert g.kernel_launches() == n0
    assert g.export_streams(range(S)).tobytes() == rec0.tobytes()
    with pytest.raises(ValueError):
        g.run(PROC, buf[:2], [10, 10, 10], streams=[0, 1])
    with pytest.raises(ValueError):
        g.run(PROC, buf, 10, streams=[0, 1])  # four rows for two entries


def test_list_calls_allocate_nothing_after_reserve(emu_libs):
    """reserve(in_stride, out_stride) sizes list calls as it sizes b200s_run_per_stream: turnovers with rows narrower than
    outputLatency included."""
    S, C = 6, 2
    e = _emu(emu_libs["float"], S)
    e.configure(C, 512, 128)
    in_stride, out_stride = 700, 200
    e.reserve(in_stride, out_stride)
    x = signals.batch("harmonic", S, C, in_stride, 48000)
    e.run(PROC, x, 150, inputSamples=150)
    before = e.device_allocations()
    e.run(PROC, x[:3], 160, inputSamples=180, streams=[5, 1, 3])
    e.run([OSEEK, PROC, FLUSH], x[:3], [0, 150, 200], inputSamples=[600, 190, 0], playbackRates=1.0, streams=[2, 0, 4])
    e.run([PROC] * 6, x, 100, inputSamples=125, streams=[3, 2, 1, 0, 5, 4])
    assert e.device_allocations() == before


def test_listed_stream_equals_the_oracle(emu_libs, oracle_port):
    """A stream that is listed in three calls (among others, at different positions) is the one-stream oracle bit for bit."""
    from oracle.hdrref import CpuStretch

    t = _six(emu_libs)
    calls = [([3, 1, 0], [400, 300, 420], [320, 240, 336]), ([0, 5, 4, 2], [401, 300, 300, 300], [320, 300, 300, 300]),
             ([2, 4, 0], [200, 300, 398], [320, 320, 333])]
    ys = [t.call(l, PROC, a, b) for l, a, b in calls]
    o = CpuStretch("orc", 321)
    o.configure(2, 512, 128)
    pos = 0
    for (l, a, b), y in zip(calls, ys):
        i = l.index(0)
        ref = o.process(t.x[0][:, pos:pos + a[i]], b[i])
        pos += a[i]
        assert np.array_equal(y[i, :, :b[i]], ref), np.abs(y[i, :, :b[i]] - ref).max()


# ------------------------------------------------------------------ H100
@pytest.mark.gpu
def test_tenth_of_a_large_batch_with_turnover_on_the_gpu(cuda_lib):
    """1024 stereo presetDefault slots, 10 % listed (a random list, in random order) over 20 calls, with flushes and
    output seeks in the middle: the twin-engine equality on the H100, bit for bit."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C = 1024, 2
    rng = np.random.default_rng(17)

    def make():
        e = BatchStretch(S)
        e.presetDefault(C, SR)
        return e

    H = 1440
    n_out = 8 * H
    n_in = int(round(n_out / 0.8))
    lst = rng.permutation(S)[:S // 10]
    audio = signals.batch("harmonic", lst.size, C, 20 * n_in + 8000, 48000)
    t = Twins(make, dict(zip(lst, audio)), S)
    assert t.sub.intervalSamples() == H
    turn = lst[::7]
    for k in range(20):
        ops = np.full(lst.size, PROC, np.int32)
        ni = np.full(lst.size, n_in, np.int32)
        no = np.full(lst.size, n_out, np.int32)
        if k == 9:
            ops[np.isin(lst, turn)] = FLUSH
            ni[ops == FLUSH], no[ops == FLUSH] = 0, 3 * H
        elif k == 10:
            ops[np.isin(lst, turn)] = OSEEK
            ni[ops == OSEEK], no[ops == OSEEK] = 6000, 0
        t.call(lst, ops, ni, no, rates=1.0, check=k in (0, 5, 9, 10, 19))  # (records of 1024 slots: a few checkpoints)
        if k == 4:
            lst = rng.permutation(lst)  # a changed list from here on
    assert t.sub.unserved_random_blocks() == 0


@pytest.mark.gpu
def test_torch_tensor_list_call_on_the_current_stream(cuda_lib):
    """A torch CUDA tensor through run(..., streams=) runs on torch's current stream (b200s_run_streams_device) and equals
    the host-buffer list call."""
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C = 64, 2
    lst = np.array([40, 3, 17, 63, 0, 22, 9, 51])
    engines = [BatchStretch(S), BatchStretch(S)]
    for e in engines:
        e.presetDefault(C, SR)
    H = engines[0].intervalSamples()
    x = signals.batch("harmonic", lst.size, C, 3 * 10 * H, 48000).astype(np.float32)
    side = torch.cuda.Stream()
    host, dev = [], []
    with torch.cuda.stream(side):
        for k in range(3):
            a = np.ascontiguousarray(x[:, :, k * 10 * H:(k + 1) * 10 * H])
            host.append(engines[0].run(PROC, a, 8 * H, streams=lst))
            y = engines[1].run(PROC, torch.from_numpy(a).cuda(), 8 * H, streams=lst)
            dev.append(y.cpu().numpy())
    for a, b in zip(host, dev):
        assert np.array_equal(a, b)
