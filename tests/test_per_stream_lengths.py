"""Per-stream input / output lengths (b200s_process_per_stream*): one call whose streams each read and write their own
number of samples.

Under the CPU emulator (exact arithmetic, the oracle's FFT swapped in) every stream must be bit-identical to its own
one-stream oracle driven with that stream's lengths, over calls whose lengths change from call to call.  On the H100
(-m gpu) every stream must be bit-identical to the same stream in a uniform batch run with its lengths, the exact mode
must equal the emulator's float build, per-stream calls must allocate nothing after reserve(), and chained asynchronous
calls must equal synchronous ones.
"""
import ctypes

import numpy as np
import pytest

import signals

SR = 48000.0
PLAIN = (0, 0, 0, False, 0)


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


def _ragged_inputs(x, plan, pad=4, fill=0.75):
    """Per call: the [S][C][stride] input slab (stream s's next n_in[s] samples of x[s], then `fill` up to the stride, which
    the engine must not read; the stride is a multiple of 4, so that aligned lengths take the bulk-copy staging) and the
    counts.  plan: list of (n_in[S], n_out[S])."""
    S, C = x.shape[:2]
    pos = np.zeros(S, int)
    calls = []
    for n_in, n_out in plan:
        n_in, n_out = np.asarray(n_in), np.asarray(n_out)
        stride = (int(n_in.max()) + pad + 3) // 4 * 4
        buf = np.full((S, C, stride), fill, np.float32)
        for s in range(S):
            buf[s, :, :n_in[s]] = x[s, :, pos[s]:pos[s] + n_in[s]]
        pos += n_in
        calls.append((buf, n_in, n_out))
    assert np.all(pos <= x.shape[-1])
    return calls


def _run_ragged(g, x, plan, out_pad=0):
    """Drive a batch engine with per-stream lengths; returns each stream's output [C][sum of its n_out] and checks the zero
    tails (output rows are max(n_out) + out_pad long)."""
    S, C = x.shape[:2]
    ys = [[] for _ in range(S)]
    for buf, n_in, n_out in _ragged_inputs(x, plan):
        out = np.full((S, C, int(n_out.max()) + out_pad), np.nan, np.float32)
        y = np.array(g.process(buf, n_out, out=out, inputSamples=n_in))
        for s in range(S):
            assert not np.any(y[s, :, n_out[s]:]), "stream %d: the output tail is not zero" % s
            ys[s].append(y[s, :, :n_out[s]])
    return [np.concatenate(v, axis=-1) for v in ys]


def _oracle():
    """A one-stream oracle with the emulator engines' seed: (0, n) calls stretch without limit, so their blocks draw random
    time factors."""
    from oracle.hdrref import CpuStretch

    return CpuStretch("orc", 321)


def _run_oracle(o, xs, plan, s):
    outs, pos = [], 0
    for n_in, n_out in plan:
        outs.append(o.process(xs[:, pos:pos + n_in[s]], int(n_out[s])))
        pos += n_in[s]
    return np.concatenate(outs, axis=-1)


def _check_vs_oracles(ys, make, cfg, prm, x, plan):
    for s in range(len(ys)):
        o = make()
        cfg(o)
        _set_one(o, prm[s])
        ref = _run_oracle(o, x[s], plan, s)
        assert ys[s].shape == ref.shape, (s, ys[s].shape, ref.shape)
        assert np.array_equal(ys[s], ref), "stream %d: max diff %g" % (s, np.abs(ys[s] - ref).max())


# ------------------------------------------------------------------ CPU emulator, against the oracle
# configure(2, 512, 128), six streams; per call (n_in, n_out) of each stream
SIX_PRM = [PLAIN, (3, 0.25, 0, False, 0), PLAIN, (0, 0, 3, False, 0), PLAIN, (-5, 0, 0, True, 200 / SR)]
SIX_PLAN = [  # s0 beyond 2x | s1 (0, n) calls | s2 silent, then (0, 0) | s3 lengths not multiples of 4 | s4 silent | s5 0.5x
    ([128, 400, 400, 401, 300, 640], [320, 320, 320, 318, 320, 320]),
    ([120, 0, 400, 397, 250, 600], [300, 300, 320, 333, 300, 300]),
    ([140, 350, 600, 402, 300, 700], [350, 280, 480, 290, 350, 350]),
    ([100, 0, 600, 399, 200, 500], [250, 250, 480, 301, 250, 250]),
    ([128, 420, 0, 400, 260, 640], [320, 336, 0, 317, 320, 320]),
    ([0, 300, 300, 303, 0, 0], [0, 240, 300, 300, 0, 0]),
    ([130, 0, 500, 401, 200, 640], [325, 0, 400, 320, 320, 320]),
    ([128, 400, 400, 400, 200, 640], [320, 320, 320, 320, 320, 320]),
]


def _six_inputs():
    x = signals.batch("harmonic", 6, 2, 5000, 48000)
    x[2, :, 800:2000] = 0.0  # stream 2: two silent calls (1200 samples >= 2 * 512), then (0, 0) enters the bypass
    rng = np.random.default_rng(5)
    x[4] = (1e-9 * rng.uniform(-1, 1, x[4].shape)).astype(np.float32)  # below the noise floor: the bypass copies its input
    return x


def test_six_streams_with_own_lengths_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Beyond 2x (random path), (0, n), (0, 0) after a long silence (the bands are cleared), lengths that are not multiples
    of 4, a silent stream whose bypass wraps its own input, mapped and formant streams: lengths change every call."""
    cfg = lambda o: o.configure(2, 512, 128)  # noqa: E731
    x = _six_inputs()
    g = _emu(emu_libs["exact"], 6)
    cfg(g)
    _set_batch(g, SIX_PRM)
    ys = _run_ragged(g, x, SIX_PLAN, out_pad=5)
    assert g.unserved_random_blocks() == 0
    assert np.abs(ys[4]).max() > 0 and np.abs(ys[4]).max() < 1e-8  # the bypass: the stream's own input, wrapped
    _check_vs_oracles(ys, _oracle, cfg, SIX_PRM, x, SIX_PLAN)


def test_stereo_preset_per_stream_ratios_and_output_lengths_bit_exact_vs_oracle(emu_libs, oracle_port):
    """presetDefault stereo, 32-block calls (k_analyse2<3072>, k_chain_direct4, k_synth2): per-stream ratios with the same
    output length, then per-stream output lengths (zero tails checked), one of them with an unaligned input length."""
    cfg = lambda o: o.presetDefault(2, 48000.0)  # noqa: E731
    H = 1440
    n = 32 * H
    prm = [PLAIN, PLAIN, (4, 8000 / SR, 0, False, 0), PLAIN]
    plan = [
        ([int(round(n / r)) for r in (0.8, 1.25, 1.0, 0.67)], [n] * 4),
        ([36000, 28801, 0, 57600], [n, 20 * H + 7, 0, 32 * H]),
        ([12000, 14400, 23040, 1440], [9 * H, 5 * H, 16 * H, 0]),
    ]
    x = signals.batch("harmonic", 4, 2, sum(max(p[0]) for p in plan), 48000)
    g = _emu(emu_libs["exact"], 4)
    cfg(g)
    _set_batch(g, prm)
    ys = _run_ragged(g, x, plan, out_pad=3)
    _check_vs_oracles(ys, _oracle, cfg, prm, x, plan)


def test_cheaper_split_mono_per_stream_lengths_bit_exact_vs_oracle(emu_libs, oracle_port):
    """presetCheaper mono with split computation (k_analyse2<2560>, the split ring of k_synth2), per-stream lengths."""
    cfg = lambda o: o.presetCheaper(1, 48000.0)  # noqa: E731
    H = 1920
    prm = [PLAIN] * 3
    plan = [
        ([12 * H, 8 * H, 10 * H + 1], [10 * H, 10 * H, 10 * H]),
        ([9 * H, 0, 4 * H], [6 * H + 3, 4 * H, 8 * H]),
        ([7 * H, 12 * H, 0], [7 * H, 9 * H, 0]),
    ]
    x = signals.batch("harmonic", 3, 1, sum(max(p[0]) for p in plan), 48000)
    g = _emu(emu_libs["exact"], 3)
    cfg(g)
    ys = _run_ragged(g, x, plan)
    _check_vs_oracles(ys, _oracle, cfg, prm, x, plan)


def test_equal_per_stream_lengths_equal_the_uniform_call(emu_libs):
    """Float emulator: per-stream calls whose streams all have the call's lengths give the uniform call's output bit for bit,
    with the same kernel launches."""
    S, C = 3, 2
    x = signals.batch("harmonic", S, C, 3000, 48000)
    outs, launches = [], []
    for per in (False, True):
        g = _emu(emu_libs["float"], S, exact_math=False)
        g.configure(C, 512, 128)
        n0 = g.kernel_launches()
        ys = []
        for i, ci, co in signals.chunks(x.shape[-1], 0.8, 500):
            a = x[:, :, i:i + ci]
            ys.append(np.array(g.process(a, np.full(S, co), inputSamples=np.full(S, ci)) if per else g.process(a, co)))
        outs.append(np.concatenate(ys, axis=-1))
        launches.append(g.kernel_launches() - n0)
    assert np.array_equal(outs[0], outs[1])
    assert launches[0] == launches[1]


def test_one_stream_beyond_2x_leaves_no_unserved_random_block(emu_libs, oracle_port):
    """Only stream 1 of four stretches beyond 2x, and in one call it idles with (0, 0) while the others run at 1x: the
    random path is launched whenever it may be needed, and that stream matches its oracle."""
    cfg = lambda o: o.configure(1, 512, 128)  # noqa: E731
    plan = [([400, 120, 400, 400], [400, 300, 400, 400]),
            ([400, 0, 400, 400], [400, 0, 400, 400]),
            ([400, 130, 400, 400], [400, 330, 400, 400]),
            ([400, 100, 400, 400], [400, 400, 400, 400])]
    x = signals.batch("harmonic", 4, 1, 1600, 48000)
    g = _emu(emu_libs["exact"], 4)
    cfg(g)
    ys = _run_ragged(g, x, plan)
    assert g.unserved_random_blocks() == 0
    _check_vs_oracles(ys, _oracle, cfg, [PLAIN] * 4, x, plan)


def test_per_stream_arguments_are_validated(emu_libs):
    """NULL arrays, negative strides, negative lengths and lengths beyond the stride are refused before anything is
    enqueued, naming the stream; Python refuses wrong shapes with ValueError."""
    from signalsmith_stretch_b200 import StretchError

    S, C = 3, 2
    g = _emu(emu_libs["float"], S)
    g.configure(C, 512, 128)
    lib, h = g._lib, g._h
    ip = ctypes.POINTER(ctypes.c_int)
    buf = np.zeros((S, C, 256), np.float32)
    out = np.zeros((S, C, 256), np.float32)
    ok = np.array([100, 200, 256], np.int32)
    n0 = g.kernel_launches()
    for fn in ("b200s_process_per_stream", "b200s_process_per_stream_async"):
        f = getattr(lib, fn)
        assert f(h, buf.ctypes.data, 256, None, out.ctypes.data, 256, ok.ctypes.data_as(ip)) == -1
        assert f(h, buf.ctypes.data, 256, ok.ctypes.data_as(ip), out.ctypes.data, 256, None) == -1
        assert f(h, buf.ctypes.data, -1, ok.ctypes.data_as(ip), out.ctypes.data, 256, ok.ctypes.data_as(ip)) == -1
        assert f(h, buf.ctypes.data, 256, ok.ctypes.data_as(ip), out.ctypes.data, -4, ok.ctypes.data_as(ip)) == -1
    assert lib.b200s_process_per_stream_device(h, buf.ctypes.data, 256, None, out.ctypes.data, 256, None) == -1
    assert lib.b200s_process_per_stream(None, buf.ctypes.data, 256, ok.ctypes.data_as(ip), out.ctypes.data, 256, ok.ctypes.data_as(ip)) == -1
    for bad_in, bad_out, stream in (([100, -1, 0], [10, 10, 10], 1), ([100, 257, 0], [10, 10, 10], 1),
                                    ([0, 0, 0], [10, 10, 300], 2), ([0, 0, 0], [-3, 0, 0], 0)):
        a, b = np.array(bad_in, np.int32), np.array(bad_out, np.int32)
        rc = lib.b200s_process_per_stream(h, buf.ctypes.data, 256, a.ctypes.data_as(ip), out.ctypes.data, 256, b.ctypes.data_as(ip))
        assert rc == -1
        assert ("stream %d" % stream) in lib.b200s_last_error(h).decode()
    assert g.kernel_launches() == n0  # nothing was enqueued
    with pytest.raises(StretchError, match="stream 1"):
        g.process_per_stream_host_ptr(buf.ctypes.data, 256, [0, 300, 0], out.ctypes.data, 256, [0, 0, 0], wait=True)
    for call in (lambda: g.process(buf, [10, 10]), lambda: g.process(buf, 10, inputSamples=[1, 2, 3, 4]),
                 lambda: g.process(buf, [10, 10, 10], inputSamples=[1, 2, 300]),
                 lambda: g.process(buf, [10, -1, 10]), lambda: g.process(buf, np.zeros((S, 1), int)),
                 lambda: g.process(buf, [10, 20, 30], out=np.zeros((S, C, 20), np.float32)),
                 lambda: g.process(buf, [1.5, 2, 3])):
        with pytest.raises(ValueError):
            call()
    assert g.kernel_launches() == n0
    # a valid call after the refused ones: the output has max(outputSamples) samples per row
    y = g.process(buf, [10, 0, 30], inputSamples=[256, 0, 17])
    assert y.shape == (S, C, 30) and not np.any(y[:, :, 30:]) and not np.any(y[0, :, 10:])


# ------------------------------------------------------------------ H100
def _gpu_mix(S, seed=99):
    """Seeded per-stream ratios and output lengths (presetDefault stereo, 48 kHz): a few distinct (ratio, length) pairs so
    that the uniform batches stay few."""
    rng = np.random.default_rng(seed)
    H = 1440
    ratios = np.array([0.67, 0.8, 1.0, 1.25, 1.5])
    r = ratios[rng.integers(0, len(ratios), S)]
    n_out = np.where(rng.random(S) < 0.5, 32 * H, 20 * H)
    return r, n_out


@pytest.mark.gpu
def test_per_stream_lengths_equal_uniform_batches_on_the_gpu(cuda_lib, oracle_port):
    """64 stereo presetDefault streams with seeded per-stream ratios and output lengths, fast arithmetic, two calls: each
    stream is bit-identical to the same stream in a uniform batch run with its lengths, and within the usual short-horizon
    tolerances of its oracle."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C = 64, 2
    r, n_out = _gpu_mix(S)
    n_in = np.array([int(round(n_out[s] / r[s])) for s in range(S)])
    plan = [(n_in, n_out), (n_in, n_out)]
    x = signals.batch("harmonic", S, C, 2 * int(n_in.max()), 48000)
    g = BatchStretch(S)
    g.presetDefault(C, SR)
    ys = _run_ragged(g, x, plan)
    groups = {}
    for s in range(S):
        groups.setdefault((int(n_in[s]), int(n_out[s])), []).append(s)
    assert len(groups) > 3
    for (ni, no), idx in groups.items():
        u = BatchStretch(len(idx))
        u.presetDefault(C, SR)
        yu = np.concatenate([np.array(u.process(x[idx][:, :, k * ni:(k + 1) * ni], no)) for k in range(2)], axis=-1)
        for j, s in enumerate(idx):
            assert np.array_equal(ys[s], yu[j]), "stream %d (%d, %d): max diff %g" % (s, ni, no, np.abs(ys[s] - yu[j]).max())
    H = g.intervalSamples()
    per = []
    for s in range(S):
        o = oracle_port()
        o.presetDefault(C, SR)
        ref = o.process(x[s][:, :n_in[s]], int(n_out[s]))
        lat = g.outputLatency() + int(g.inputLatency() * r[s])
        per.append(rms((ys[s][:, :n_out[s]] - ref)[:, :lat + 8 * H]))
    per = np.array(per)
    assert np.median(per) <= 1e-4, per
    assert per.max() <= 1e-3, per


@pytest.mark.gpu
def test_exact_mode_ragged_batch_bit_identical_to_emulator(cuda_lib, emu_libs):
    """Exact arithmetic: a small ragged presetDefault batch (idle slot, (0, n), an unaligned length, differing output
    lengths) gives the emulator's float build bit for bit."""
    from signalsmith_stretch_b200 import BatchStretch

    H = 1440
    plan = [([14400, 11520, 0, 9001], [12 * H, 8 * H, 0, 7 * H + 1]),
            ([8640, 0, 14400, 11520], [8 * H, 6 * H, 10 * H, 9 * H]),
            ([11520, 12000, 7200, 10000], [9 * H + 3, 10 * H, 5 * H, 8 * H])]
    x = signals.batch("harmonic", 4, 2, sum(max(p[0]) for p in plan), 48000)
    outs = []
    for e in (BatchStretch(4), BatchStretch(4, lib_path=emu_libs["float"])):
        e.presetDefault(2, SR)
        e.set_tuning(3, 1)
        outs.append(_run_ragged(e, x, plan, out_pad=2))
    for s in range(4):
        a, b = outs[0][s], outs[1][s]
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (s, np.abs(a - b).max())
    assert np.abs(outs[0][0]).max() > 0.05


@pytest.mark.gpu
def test_per_stream_calls_allocate_nothing_after_reserve(cuda_lib):
    """After reserve() with the strides, per-stream calls whose lengths change every call allocate nothing (within 2x
    stretch: beyond it the random path's rows are allocated on first use, as for the uniform call)."""
    from signalsmith_stretch_b200 import BatchStretch

    S, C = 16, 2
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    H = e.intervalSamples()
    in_stride, out_stride = 12 * H, 9 * H
    e.reserve(in_stride, out_stride)
    rng = np.random.default_rng(3)
    x = signals.batch("harmonic", S, C, in_stride, 48000)
    before = e.device_allocations()
    for k in range(5):
        n_out = rng.integers(0, out_stride + 1, S)
        n_out[0] = out_stride
        n_in = rng.integers(n_out, in_stride + 1)
        n_in[1], n_out[1] = (0, 0) if k % 2 else (in_stride, 0)  # an idle slot, then (n, 0)
        e.process(x, n_out, inputSamples=n_in)
    e.synchronize()
    assert e.device_allocations() == before


@pytest.mark.gpu
def test_chained_async_per_stream_calls_equal_synchronous_calls(cuda_lib):
    """Chained b200s_process_per_stream_async calls (pinned buffers, equal strides, lengths that change every call, the
    host-buffer stream groups pipelining without a join) equal the synchronous calls bit for bit."""
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C, calls = 48, 2, 6
    rng = np.random.default_rng(11)
    e0 = BatchStretch(1)
    e0.presetDefault(C, SR)
    H = e0.intervalSamples()
    in_stride, out_stride = 10 * H, 8 * H
    lens = [(rng.integers(0, in_stride + 1, S).astype(np.int32), rng.integers(0, out_stride + 1, S).astype(np.int32)) for _ in range(calls)]
    x = signals.batch("harmonic", S, C, calls * in_stride, 48000)
    slabs = [np.ascontiguousarray(x[:, :, k * in_stride:(k + 1) * in_stride]) for k in range(calls)]
    sync = BatchStretch(S)
    sync.presetDefault(C, SR)
    ref = [sync.process(slabs[k], lens[k][1], out=np.empty((S, C, out_stride), np.float32), inputSamples=lens[k][0]) for k in range(calls)]
    e = BatchStretch(S)
    e.presetDefault(C, SR)
    e.reserve(in_stride, out_stride)
    pin_in = [torch.from_numpy(slabs[k]).pin_memory() for k in range(calls)]
    pin_out = [torch.empty((S, C, out_stride), dtype=torch.float32).pin_memory() for _ in range(calls)]
    for k in range(calls):
        pin_out[k].fill_(float("nan"))
    for k in range(calls):
        e.process_per_stream_host_ptr(pin_in[k].data_ptr(), in_stride, lens[k][0], pin_out[k].data_ptr(), out_stride, lens[k][1])
    e.synchronize()
    for k in range(calls):
        got = pin_out[k].numpy()
        assert np.array_equal(got, ref[k]), (k, np.nanmax(np.abs(got - ref[k])))
