"""GPU parity tests: the CUDA path, called through the C ABI (include/b200_stretch.h), against the
oracle and the committed golden vectors.  `pytest -m gpu` on an H100.

Tolerances (float32 path; the only arithmetic that differs from the oracle is the FFT rounding):
  * identity configuration (no transposition, rate 1): <= 1e-6 RMS at any length;
  * short free-running horizon (first 8 blocks after the latency): <= 1e-4 RMS  (north_star);
  * whole fixture (16 blocks): <= 1e-3 RMS, the reference's own regression criterion
    (-60 dB, cmd/main-dev.cpp:215-232) -- the algorithm is chaotic beyond a few blocks
    (SURVEY.md section 0.4: two builds of the reference diverge the same way).
"""
import os

import numpy as np
import pytest

import signals

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rms(a):
    return float(np.sqrt(np.mean(np.square(a, dtype=np.float64))))


@pytest.fixture(scope="module")
def gpu(cuda_lib):
    import torch

    assert torch.cuda.is_available(), "these tests need a GPU"
    from signalsmith_stretch_b200 import BatchStretch

    return lambda batch: BatchStretch(batch)


def _oracle_batch(oracle_port, cfg, x, ratio, chunk):
    outs = []
    for s in range(x.shape[0]):
        o = oracle_port()
        cfg(o)
        outs.append(signals.run_single(o, x[s], ratio, chunk))
    return np.stack(outs)


@pytest.mark.parametrize("name", list(signals.CONFIGS))
def test_golden_vectors_from_the_reference(gpu, name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg, C, sr, ratio, _ = signals.CONFIGS[name]
    e = gpu(3)  # the same stream three times: also checks batch lanes agree bit-exactly
    cfg(e)
    x = np.repeat(g["x"][None], 3, axis=0)
    y = signals.run_batch(e, x, float(g["ratio"]), int(g["chunk"]))
    assert np.array_equal(y[0], y[1]) and np.array_equal(y[0], y[2])
    H = e.intervalSamples()
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    for key in ("hdr", "wasm"):
        if key not in g:
            continue
        d = y[0] - g[key]
        if name == "identity":
            assert rms(d) <= 1e-6, key
        else:
            assert rms(d[:, : lat + 8 * H]) <= 1e-4, (key, rms(d[:, : lat + 8 * H]))
            assert rms(d) <= 1e-3, (key, rms(d))


@pytest.mark.parametrize("name", list(signals.CONFIGS))
def test_free_run_vs_oracle_batch(gpu, oracle_port, name):
    """8 different streams per config, one long chunk per call (the bench's call pattern)."""
    cfg, C, sr, ratio, kind = signals.CONFIGS[name]
    S = 8
    e = gpu(S)
    cfg(e)
    H, B = e.intervalSamples(), e.blockSamples()
    n_out = 12 * H + B
    n_in = int(round(n_out / ratio))
    x = signals.batch(kind, S, C, n_in, sr)
    y = signals.run_batch(e, x, ratio, n_out)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, n_out)
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    d = y - ref
    if name == "identity":
        assert rms(d) <= 1e-6
    else:
        # per stream: the hard decisions of the algorithm (peak picking, max channel) can flip on a
        # 1e-7 FFT rounding difference and the feedback then amplifies it (SURVEY.md section 0.4), so the
        # short-horizon gate is on the median stream; every stream must stay within the reference's own
        # whole-file criterion.  The step-by-step gate without amplification is the teacher-forced test.
        per = np.array([rms(d[s][:, : lat + 8 * H]) for s in range(S)])
        assert np.median(per) <= 1e-4, per
        assert per.max() <= 1e-3 and rms(d) <= 1e-3, (per, rms(d))


@pytest.mark.parametrize("ratio", [1.5, 0.75])
def test_stereo_preset_cheaper_plain_vs_oracle(gpu, oracle_port, ratio):
    """presetCheaper stereo without transposition: K = 2560 = 16*16*10 paired FFT, L = 3 (odd lane skew) in the packed
    stereo chain (fast arithmetic), split computation (ring of block + interval samples) in the vector overlap-add."""
    def cfg(o):
        o.presetCheaper(2, 48000.0)

    S = 4
    e = gpu(S)
    cfg(e)
    H, B = e.intervalSamples(), e.blockSamples()
    n_out = 12 * H + B
    x = signals.batch("harmonic", S, 2, int(round(n_out / ratio)), 48000)
    y = signals.run_batch(e, x, ratio, 6 * H)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, 6 * H)
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    d = y - ref
    per = np.array([rms(d[s][:, : lat + 8 * H]) for s in range(S)])
    assert np.median(per) <= 1e-4, per
    assert per.max() <= 1e-3 and rms(d) <= 1e-3, (per, rms(d))


def test_automatic_formant_pitch_vs_oracle(gpu, oracle_port):
    """setFormantBase(0): the per-block pitch estimate (estimateFrequency :929-966, k_pitch) and its smoothing state,
    carried over calls -- stereo, +12 semitones with formant compensation, several calls per stream."""
    def cfg(o):
        o.presetDefault(2, 48000.0)
        o.setTransposeSemitones(12, 0)
        o.setFormantFactor(1, True)
        o.setFormantBase(0)

    S = 4
    e = gpu(S)
    cfg(e)
    H, B = e.intervalSamples(), e.blockSamples()
    n_out = 12 * H + B
    x = signals.batch("harmonic", S, 2, n_out, 48000)
    y = signals.run_batch(e, x, 1.0, 4 * H)  # four blocks per call: the estimate's state crosses calls
    ref = _oracle_batch(oracle_port, cfg, x, 1.0, 4 * H)
    lat = e.outputLatency() + e.inputLatency()
    d = y - ref
    per = np.array([rms(d[s][:, : lat + 8 * H]) for s in range(S)])
    assert np.median(per) <= 1e-4, per
    assert per.max() <= 1e-3 and rms(d) <= 1e-3, (per, rms(d))


@pytest.mark.parametrize("name", [n for n in signals.CONFIGS if n != "identity"])
def test_teacher_forced_block_by_block(gpu, oracle_port, name):
    """T1 of SURVEY.md section 8(c): before every call the oracle's complete signal state (history,
    pending overlap-add, spectra, prediction energy) is imported into the GPU engine, both then
    process the same 2 blocks; errors cannot accumulate across calls.  Gate: EVERY call <= 1e-5 RMS on the
    harmonic fixtures (2e-5 with formants: the envelope's running max / min decisions sit on the FFT rounding).
    The one exception is the pure sine sweep (config 1): most of its bins are at rounding-noise level, where a hard
    decision can flip inside a single block -- the reference's own two builds (header vs shipped binary) disagree by
    more than 1e-4 over 2-block windows of that very fixture, which is asserted below from the golden file; there the
    gate is median <= 1e-5, every call <= 2e-4."""
    cfg, C, sr, ratio, kind = signals.CONFIGS[name]
    e, o = gpu(1), oracle_port()
    cfg(e)
    cfg(o)
    H, B = e.intervalSamples(), e.blockSamples()
    n_calls, co = 14, 2 * H
    ci = int(round(co / ratio))
    x = signals.batch(kind, 1, C, ci * n_calls, sr)
    errs = []
    for k in range(n_calls):
        st = o.signal_state()
        for key in ("history", "pending", "pendingWp", "input", "prevInput", "output", "predEnergy"):
            e.set_state(key, st[key][None])
        xin = x[:, :, k * ci:(k + 1) * ci]
        yo = o.process(xin[0], co)
        yg = np.asarray(e.process(xin, co))[0]
        errs.append(rms(yg - yo))
    if kind == "sweep":
        g = np.load(os.path.join(GOLD, name + ".npz"))
        lat = e.outputLatency() + int(e.inputLatency() * ratio)
        dd = g["hdr"] - g["wasm"]
        ref_vs_ref = max(rms(dd[:, lat + k * co: lat + (k + 1) * co]) for k in range((dd.shape[-1] - lat) // co))
        assert ref_vs_ref > 1e-4, ref_vs_ref  # the reference disagrees with itself by more than the north-star tolerance here
        assert np.median(errs) <= 1e-5 and max(errs) <= 2e-4, errs
    else:
        assert max(errs) <= (2e-5 if name == "config4_formant" else 1e-5), errs


def test_identity_full_size_is_a_pure_delay(gpu):
    """Size-independent property at BASELINE batch scale: 1024 stereo streams, 1 s calls."""
    S, C, sr = 1024, 2, 48000
    e = gpu(S)
    e.presetDefault(C, float(sr))
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((S, C, 2 * sr)) * 0.25).astype(np.float32)
    y = signals.run_batch(e, x, 1.0, sr)
    lat = e.inputLatency() + e.outputLatency()
    assert rms(y[:, :, lat:] - x[:, :, :-lat]) <= 1e-6
    assert np.abs(y[:, :, :lat]).max() <= 1e-5


def test_chunk_size_invariance_bit_exact(gpu):
    """SURVEY.md section 8(c) KAT 6: the reference is bit-exactly chunk-invariant at rate 1."""
    x = signals.batch("harmonic", 4, 1, 30000, 48000)
    ys = []
    for chunk in (64, 480, 5000, 30000):
        e = gpu(4)
        signals.cfg_config3(e)
        ys.append(signals.run_batch(e, x, 1.0, chunk))
    for y in ys[1:]:
        assert np.array_equal(ys[0], y)


def test_split_computation_is_a_delay_by_one_interval(gpu):
    x = signals.batch("harmonic", 2, 1, 30000, 48000)
    a, b = gpu(2), gpu(2)
    a.presetCheaper(1, 48000.0, False)
    b.presetCheaper(1, 48000.0, True)
    for e in (a, b):
        e.setTransposeSemitones(5, 0)
    ya, yb = signals.run_batch(a, x, 1.0, 6000), signals.run_batch(b, x, 1.0, 6000)
    H = a.intervalSamples()
    assert b.outputLatency() == a.outputLatency() + H
    assert rms(yb[:, :, H:] - ya[:, :, :-H]) <= 1e-4


def test_api_sequence_vs_oracle(gpu, oracle_port):
    """seek / silence bypass / flush / reset / outputSeek / exact, presetDefault size."""
    x = signals.harmonic(60000, 48000)[None]

    def seq(o, wrap, unwrap):
        o.presetDefault(1, 48000.0)
        o.setTransposeSemitones(3, 0)
        outs = []
        o.seek(wrap(x[:, :3000]), 1.0)
        outs.append(unwrap(o.process(wrap(x[:, 3000:7800]), 4800)))
        z = np.zeros((1, 30000), np.float32)
        outs.append(unwrap(o.process(wrap(z[:, :12000]), 12000)))
        outs.append(unwrap(o.process(wrap(z[:, :4000]), 4000)))
        outs.append(unwrap(o.process(wrap(z[:, :4000]), 5000)))
        outs.append(unwrap(o.process(wrap(x[:, 8000:17600]), 9000)))
        outs.append(unwrap(o.flush(1000, 1.0)))
        outs.append(unwrap(o.process(wrap(x[:, 20000:24800]), 4800)))
        outs.append(unwrap(o.flush(5000, 1.1)))
        o.reset()
        outs.append(unwrap(o.process(wrap(x[:, 20000:24800]), 2400)))
        o.outputSeek(wrap(x[:, : o.outputSeekLength(1.3)]))
        outs.append(unwrap(o.process(wrap(x[:, 5000:11240]), 4800)))
        ok, e = o.exact(wrap(x[:, :40000]), 50000)
        assert ok
        outs.append(unwrap(e))
        return outs

    ref = seq(oracle_port(), lambda a: a, lambda a: a)
    got = seq(gpu(1), lambda a: a[None], lambda a: np.asarray(a)[0])
    for i, (r, g_) in enumerate(zip(ref, got)):
        assert r.shape == g_.shape
        # calls of <= 0.2 s: short horizon; exact() renders a full second: the reference's own
        # whole-file criterion (-60 dB) applies (SURVEY.md section 0.4)
        tol = 2e-4 if r.shape[1] <= 12000 else 1e-3
        assert rms(r - g_) <= tol, (i, rms(r - g_))
    # the bypass calls copy input to output exactly
    assert np.array_equal(ref[2], got[2]) and np.array_equal(ref[3], got[3])


def test_device_pointer_api_matches_host_api(gpu):
    import torch

    x = signals.batch("harmonic", 4, 2, 20000, 48000)
    a, b = gpu(4), gpu(4)
    for e in (a, b):
        signals.cfg_config2(e)
    ya = signals.run_batch(a, x, 0.8, 8000)
    outs = []
    for i, ci, co in signals.chunks(20000, 0.8, 8000):
        xin = torch.from_numpy(np.ascontiguousarray(x[:, :, i:i + ci])).cuda()
        torch.cuda.synchronize()
        yo = b.process(xin, co)
        b.synchronize()
        outs.append(yo.cpu().numpy())
    assert np.array_equal(ya, np.concatenate(outs, axis=2))


def test_fast_div_sqrt_are_correctly_rounded(gpu):
    """The branch-free division / square root of the chain kernel (kernels.cuh fdivq/fsqrtq) must equal
    the IEEE round-to-nearest intrinsics bit for bit: 2^27 operand pairs, exponents 2^-60 .. 2^60, plus 2^27 pairs from the
    edge classes (zero, subnormal, tiny and huge numerators, divisors up to FLT_MAX and +-inf, subnormal, zero and
    infinite square-root arguments)."""
    e = gpu(1)
    bad_div, bad_sqrt = e.selftest_divsqrt(1 << 27, 12345)
    assert bad_div == 0 and bad_sqrt == 0, (bad_div, bad_sqrt)


@pytest.mark.gpu
@pytest.mark.parametrize("blocks_per_call", [7, 40])
def test_chain_kernel_generations_agree_bit_exactly(gpu, blocks_per_call):
    """The direct chain kernels (scalar lane-per-block, lane-per-(block,channel) multi-warp, paired (f2)
    stereo, packed with the decoupled skew) implement the same arithmetic: on identical spectra their outputs must be identical bit for bit
    (guards the packed kernel against compiler contraction of multiply-add pairs).  40 blocks per call also
    exercises the second group / the warp hand-off."""
    cfg, C, sr, ratio, kind = signals.CONFIGS["config2_stereo_0p8x"]
    outs = []
    from signalsmith_stretch_b200 import StretchError

    gens = []
    for gen in (1, 2, 3, 4, 5, 6):
        e = gpu(5)
        cfg(e)
        try:
            e.set_tuning(0, gen)
        except StretchError:  # generations 1, 3, 5 are superseded: only in builds with -DB200S_KEEP_OLD_KERNELS
            continue
        gens.append(gen)
        e.set_tuning(3, 1)  # exact arithmetic: generation 4 defaults to the fast (fused) mode
        H = e.intervalSamples()
        n_out = 3 * blocks_per_call * H
        x = signals.batch(kind, 5, C, int(round(n_out / ratio)), sr)
        outs.append(signals.run_batch(e, x, ratio, blocks_per_call * H))
    assert {2, 4, 6} <= set(gens), gens
    for gen, out in zip(gens[1:], outs[1:]):
        assert np.array_equal(outs[0], out), "generation %d differs from generation %d: max %g" % (gen, gens[0], np.abs(outs[0] - out).max())


@pytest.mark.gpu
@pytest.mark.parametrize("preset,ratio", [("presetDefault", 0.8), ("presetCheaper", 2.0)])
def test_mono_stream_pairs_agree_with_one_stream_per_warp_bit_exactly(gpu, preset, ratio):
    """Mono plain path: two streams per warp on the packed wavefront (k_chain_direct6<.., DUAL>, tuning key 5; stream 4 of the
    five, and the pair (2, 3) while stream 3 is silent, run alone through the same kernel) against every stream on
    k_chain_direct2, exact arithmetic: identical bit for bit.  40 blocks per call: a second group of lanes."""
    outs = []
    for dual in (0, 1):
        e = gpu(5)
        getattr(e, preset)(1, 48000.0)
        e.set_tuning(3, 1)
        e.set_tuning(5, dual)
        H = e.intervalSamples()
        n_out = 3 * 40 * H
        x = signals.batch("harmonic", 5, 1, int(round(n_out / ratio)), 48000)
        x[3, :, x.shape[-1] // 3: x.shape[-1] // 2] = 0.0
        outs.append(signals.run_batch(e, x, ratio, 40 * H))
    assert np.abs(outs[0]).max() > 0.1
    assert np.array_equal(outs[0], outs[1]), "max %g" % np.abs(outs[0] - outs[1]).max()


@pytest.mark.gpu
def test_fast_and_exact_chain_arithmetic_agree_over_a_short_horizon(gpu):
    """Default (fast: fused multiply-add, SFU reciprocal / rsqrt) against exact (the reference's unfused IEEE order)
    arithmetic of the stereo direct chain on the same spectra: float rounding apart over the first blocks (the
    recurrence is chaotic beyond, SURVEY.md section 0.4), same level throughout."""
    cfg, C, sr, ratio, kind = signals.CONFIGS["config2_stereo_0p8x"]
    outs = []
    for exact in (1, 0):
        e = gpu(4)
        cfg(e)
        e.set_tuning(3, exact)
        H = e.intervalSamples()
        n_out = 24 * H
        x = signals.batch(kind, 4, C, int(round(n_out / ratio)), sr)
        outs.append(signals.run_batch(e, x, ratio, 12 * H))
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    assert not np.array_equal(outs[0], outs[1])
    head = slice(lat, lat + 8 * H)
    assert rms(outs[0][..., head] - outs[1][..., head]) <= 1e-5
    assert rms(outs[0] - outs[1]) <= 1e-3
    assert abs(20 * np.log10(rms(outs[0]) / rms(outs[1]))) <= 0.1


@pytest.mark.gpu
def test_async_pipelined_host_calls_equal_blocking_calls(gpu):
    """b200s_process_async: consecutive host-buffer calls chained over the stream groups (no join between calls, the
    copies of one call overlapping the kernels of its neighbours) give bit for bit what blocking calls give."""
    import torch

    cfg, C, sr, ratio, kind = signals.CONFIGS["config2_stereo_0p8x"]
    S, calls = 48, 4
    outs = []
    for use_async in (False, True):
        e = gpu(S)
        cfg(e)
        H = e.intervalSamples()
        n_out = 6 * H
        n_in = int(round(n_out / ratio))
        x = signals.batch(kind, S, C, n_in * calls, sr)
        xs = [torch.from_numpy(np.ascontiguousarray(x[:, :, k * n_in:(k + 1) * n_in])).pin_memory() for k in range(calls)]
        ys = [torch.zeros((S, C, n_out), dtype=torch.float32).pin_memory() for _ in range(calls)]
        for k in range(calls):
            if use_async:
                e.process_host_ptr_async(xs[k].data_ptr(), n_in, ys[k].data_ptr(), n_out)
            else:
                e.process_host_ptr(xs[k].data_ptr(), n_in, ys[k].data_ptr(), n_out)
        e.synchronize()
        outs.append(np.concatenate([y.numpy().copy() for y in ys], axis=2))
    assert np.abs(outs[0]).max() > 0.01
    assert np.array_equal(outs[0], outs[1])


@pytest.mark.gpu
def test_paired_fft_kernels_match_scalar_fft_kernels(gpu):
    """Paired in-place packed FFT kernels vs the first-generation scalar Stockham kernels: same transform,
    different rounding -- identity configuration agrees to float precision."""
    outs = []
    for v1 in (1, 0):
        e = gpu(3)
        e.presetDefault(2, 48000.0)
        e.set_tuning(1, v1)
        x = signals.batch("harmonic", 3, 2, 48000, 48000)
        outs.append(signals.run_batch(e, x, 1.0, 7200))
    assert rms(outs[0] - outs[1]) <= 2e-7


@pytest.mark.gpu
def test_pcm16_boundary_equals_float_path_with_the_tools_conversions(gpu):
    """b200s_process_pcm16 (int16 over PCIe, conversions on the device) == the float call fed sample / 32768 with its
    output rounded to nearest (halves away from zero) and clamped; several calls, stream groups chained."""
    cfg, C, sr, ratio, kind = signals.CONFIGS["config2_stereo_0p8x"]
    S = 48
    outs = []
    for pcm in (True, False):
        e = gpu(S)
        cfg(e)
        H = e.intervalSamples()
        n_out = 6 * H
        n_in = int(round(n_out / ratio))
        x = signals.batch(kind, S, C, 3 * n_in, sr)
        x16 = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
        ys = []
        for k in range(3):
            chunk = np.ascontiguousarray(x16[:, :, k * n_in:(k + 1) * n_in])
            if pcm:
                ys.append(e.process_pcm16(chunk, n_out))
            else:
                v = e.process(chunk.astype(np.float32) * np.float32(1 / 32768), n_out) * np.float32(32768)
                ys.append(np.clip(np.sign(v) * np.floor(np.abs(v) + np.float32(0.5)), -32768, 32767).astype(np.int16))
        outs.append(np.concatenate(ys, axis=2))
    assert np.abs(outs[0]).max() > 300
    assert np.array_equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------
# parity at the benchmark's shape (BASELINE configs at batch scale, 32 blocks per call, default arithmetic)
# ------------------------------------------------------------------------------------------------
def _pool_input(S, C, n, sr, sampled):
    """[S][C][n]: 32 distinct harmonic streams at the `sampled` indices (seed = index), every other stream a copy of
    one of them (generating 1024 x 172 800 x 11 sines per test would cost more than the test itself)."""
    pool = {s: np.stack([signals.harmonic(n, sr, s, c) for c in range(C)]) for s in sampled}
    keys = list(sampled)
    return np.stack([pool[s] if s in pool else pool[keys[s % len(keys)]] for s in range(S)])


BENCH_SHAPES = [
    # (name, batch, calls): three 32-block calls, i.e. every lane of the frame wavefront busy, state carried twice
    ("config2_stereo_0p8x", 1024, 3),
    ("config3_7st_ton8k", 256, 3),
    ("config4_formant", 256, 3),
]


@pytest.mark.parametrize("name,S,calls", BENCH_SHAPES, ids=[b[0] for b in BENCH_SHAPES])
def test_benchmark_shape_vs_oracle(gpu, oracle_port, name, S, calls):
    """BASELINE configs[1] at its real batch (1024 stereo streams, 0.8x, 32 blocks per call) and configs[2] / [3] at
    batch 256, default (fast) arithmetic: 32 sampled streams against the oracle.  <= 1e-4 RMS over the first 8 blocks
    after the latency, <= 1e-3 over the whole 2.9 s (the reference's own criterion, cmd/main-dev.cpp:215-232)."""
    cfg, C, sr, ratio, kind = signals.CONFIGS[name]
    e = gpu(S)
    cfg(e)
    H = e.intervalSamples()
    n_out = 32 * H
    n_in = int(round(n_out / ratio))
    sampled = [(S // 32) * i + (i % (S // 32)) for i in range(32)]
    x = _pool_input(S, C, n_in * calls, sr, sampled)
    y = signals.run_batch(e, x, ratio, n_out)
    assert y.shape == (S, C, n_out * calls)
    ref = _oracle_batch(oracle_port, cfg, x[sampled], ratio, n_out)
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    d = y[sampled] - ref
    head = np.array([rms(d[i][:, : lat + 8 * H]) for i in range(len(sampled))])
    whole = np.array([rms(d[i]) for i in range(len(sampled))])
    mid = np.array([rms(d[i][:, : lat + 16 * H]) for i in range(len(sampled))])
    if name == "config4_formant":
        # formant envelope: running max / min decisions per bin (:986-1007) sit on the FFT's rounding, and a flipped one moves
        # a whole band's energy ratio; the median stays within 1e-4 while single streams can exceed it.  Same
        # median / worst-stream gate as the 8-stream free-run test above.
        assert np.median(head) <= 1e-4 and head.max() <= 1e-3, (head.max(), np.median(head))
    else:
        assert head.max() <= 1e-4, (head.max(), np.median(head))
    # 16 blocks: the horizon of the reference's own regression fixtures and criterion (-60 dB, cmd/main-dev.cpp:215-232)
    assert mid.max() <= 1e-3, (mid.max(), np.median(mid))
    # the whole 2.9 s (96 blocks): the recurrence is chaotic (SURVEY.md section 0.4, BASELINE.md section 2: the reference's
    # output moves by 3e-4 ... 8e-3 RMS within 1-10 s under a 1e-7 input perturbation), so SURVEY.md 8(c) T3 gates the
    # long horizon on level match and bounds the raw difference by that self-divergence.  The oracle against the
    # reference's own shipped binary (a different build of the same code) is asserted below to be just as far apart on one
    # of these streams.
    assert whole.max() <= 1e-2, (whole.max(), np.median(whole))
    lvl = np.array([20 * np.log10(rms(y[s]) / rms(ref[i])) for i, s in enumerate(sampled)])
    assert np.abs(lvl).max() <= 0.1, lvl
    if name == "config2_stereo_0p8x":  # the shipped binary's output on stream 0, sampled (tests/golden/make_golden.py)
        st = signals.REFERENCE_STRIDE
        rw = np.load(os.path.join(GOLD, "reference_outputs.npz"))["bench_shape_wasm"]
        assert sampled[0] == 0 and rw.shape == ref[0][:, ::st].shape
        ref_vs_ref = rms(rw - ref[0][:, ::st])
        print("reference (shipped binary) vs oracle over %d blocks: %.2e RMS; GPU vs oracle: %.2e" % (32 * calls, ref_vs_ref, whole[0]))
        assert ref_vs_ref >= 1e-3, ref_vs_ref  # (3.96e-3 measured: the reference does not meet 1e-3 against itself at this horizon)
    # copies of the same input in different batch lanes agree bit for bit
    twin = next(s for s in range(S) if s not in sampled and s % len(sampled) == 0)
    assert np.array_equal(y[twin], y[sampled[0]])


@pytest.mark.parametrize("which", ["monotone", "folding"])
def test_set_freq_map_table_vs_oracle(gpu, oracle_port, which):
    """setFreqMap through the C ABI on the GPU (row f3): a monotone piecewise-linear map and one that folds back
    (non-monotone output map, :896-911), presetDefault stereo, several calls."""
    tab = signals.PWL_MONOTONE if which == "monotone" else signals.PWL_FOLDING

    def cfg(o):
        o.presetDefault(2, 48000.0)
        o.setFreqMapTable(*tab)

    S = 4
    e = gpu(S)
    cfg(e)
    H, B = e.intervalSamples(), e.blockSamples()
    n_out = 12 * H + B
    x = signals.batch("harmonic", S, 2, n_out, 48000)
    y = signals.run_batch(e, x, 1.0, 6 * H)
    ref = _oracle_batch(oracle_port, cfg, x, 1.0, 6 * H)
    lat = e.outputLatency() + e.inputLatency()
    d = y - ref
    per = np.array([rms(d[s][:, : lat + 8 * H]) for s in range(S)])
    assert np.median(per) <= 1e-4, per
    assert per.max() <= 1e-3 and rms(d) <= 1e-3, (per, rms(d))


@pytest.mark.parametrize("name", ["config2_stereo_0p8x", "config4_formant"])
def test_no_device_allocation_in_process_after_reserve(gpu, name):
    """The reference's real-time contract (cmd/main-dev.cpp:158-163: no allocation inside process()): after
    b200s_reserve() with the call sizes -- parameters set first -- process() performs no cudaMalloc."""
    import torch

    cfg, C, sr, ratio, kind = signals.CONFIGS[name]
    S = 16
    e = gpu(S)
    cfg(e)
    H = e.intervalSamples()
    n_out = 8 * H
    n_in = int(round(n_out / ratio))
    e.reserve(n_in, n_out)
    x = signals.batch(kind, S, C, 3 * n_in, sr)
    before = e.device_allocations()
    for k in range(3):  # host-buffer API
        e.process(x[:, :, k * n_in:(k + 1) * n_in], n_out)
    xd = torch.from_numpy(np.ascontiguousarray(x[:, :, :n_in])).cuda()
    torch.cuda.synchronize()
    e.process(xd, n_out)  # device-pointer API
    e.process(x[:, :, : n_in // 2], n_out // 2)  # smaller calls fit too
    e.synchronize()
    assert e.device_allocations() == before
    assert before > 0


@pytest.mark.parametrize("name,ratio", [("config2_stereo_0p8x", 2.5), ("config3_7st_ton8k", 3.0)])
def test_random_time_factors_beyond_2x_vs_oracle(gpu, oracle_port, name, ratio):
    """Stretching beyond 2x (:639-640): per-bin random time factors from std::default_random_engine(seed), same seed on
    both sides -- plain stereo (interleaved spectra: the direct chain leaves the stream to k_prep + k_chain) and mono
    with a frequency map; short horizon and the reference's whole-fixture criterion.  (oracle_port builds the oracle; the
    oracle objects are created here with the engine's seed.)"""
    from oracle.hdrref import CpuStretch
    from signalsmith_stretch_b200 import BatchStretch

    cfg, C, sr, _, kind = signals.CONFIGS[name]
    S, seed = 4, 20260923
    e = BatchStretch(S, seed=seed)
    cfg(e)
    H, B = e.intervalSamples(), e.blockSamples()
    n_out = 12 * H + B
    x = signals.batch(kind, S, C, int(round(n_out / ratio)), sr)
    y = signals.run_batch(e, x, ratio, 6 * H)
    ref = []
    for s in range(S):
        o = CpuStretch("orc", seed)
        cfg(o)
        ref.append(signals.run_single(o, x[s], ratio, 6 * H))
    d = y - np.stack(ref)
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    per = np.array([rms(d[s][:, : lat + 8 * H]) for s in range(S)])
    if name == "config2_stereo_0p8x":
        assert np.median(per) <= 1e-4, per
        assert per.max() <= 1e-3 and rms(d) <= 1e-3, (per, rms(d))
    else:
        # 3x with a frequency map: every bin's twists reach up to 3 L bins away with a random offset, and the FFT's rounding
        # is amplified accordingly (per stream up to ~1e-3 over 8 blocks; the same kernels with the
        # oracle's FFT are bit-exact, tests/test_host_logic.py).  The reference's own regression criterion (-60 dB) is only
        # applied up to 1.6x stretch (cmd/main-dev.cpp:98); gate: that criterion on the median stream, level match on all.
        assert np.median(per) <= 1e-3 and per.max() <= 5e-3, per
        lvl = [20 * np.log10(rms(y[s]) / rms(ref[s])) for s in range(S)]
        assert np.abs(lvl).max() <= 0.1, lvl
    # a different seed gives a different (equally valid) output: the draws really are in the path
    e2 = BatchStretch(S, seed=seed + 1)
    cfg(e2)
    y2 = signals.run_batch(e2, x, ratio, 6 * H)
    assert rms(y2 - y) > 1e-3


def test_live_batch_vs_oracle(gpu, oracle_port):
    """The live caller (web/web-wrapper.js:215-332) on the GPU: 8 streams with their own rates, seek + process(0, 128)
    per quantum through b200s_seek_rates / b200s_process, against one oracle object per stream driven by the same loop."""
    from signalsmith_stretch_b200.live import LiveBatch

    class One:  # a one-stream oracle object behind the calls LiveBatch makes
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

    sr, S, C, quantum = 48000.0, 8, 2, 128
    audio = signals.batch("harmonic", S, C, 48000, 48000)
    e = gpu(S)
    e.presetDefault(C, sr)
    live = LiveBatch(e, sr)
    refs = []
    for s in range(S):
        o = oracle_port()
        o.presetDefault(C, sr)
        r = LiveBatch(One(o), sr)
        r.add_buffers(0, audio[s])
        r.start(0, when=0.0, offset=0.01 * s, rate=0.7 + 0.1 * s)
        refs.append(r)
        live.add_buffers(s, audio[s])
        live.start(s, when=0.0, offset=0.01 * s, rate=0.7 + 0.1 * s)
    nq = (e.outputLatency() + e.inputLatency() + 8 * e.intervalSamples()) // quantum
    y = np.concatenate([live.process(quantum) for _ in range(nq)], axis=-1)
    ref = np.stack([np.concatenate([r.process(quantum)[0] for _ in range(nq)], axis=-1) for r in refs])
    per = np.array([rms(y[s] - ref[s]) for s in range(S)])
    assert np.abs(ref).max() > 0.05
    assert np.median(per) <= 1e-4 and per.max() <= 1e-3, per
