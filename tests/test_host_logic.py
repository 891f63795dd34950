"""CPU-only checks of the product's host logic and kernel logic.

* the nvcc-built library loads here (no GPU), exports every symbol include/b200_stretch.h declares,
  and fails loudly (no CPU fallback) when asked for an engine;
* the SAME CUDA sources, run under the thread-per-CUDA-thread emulator (tests/cuda_emu), are
  compared with the oracle: with the oracle's FFT swapped in, everything else (device block
  scheduler, spectral prep, frame-wavefront phase chain, overlap-add, seek/flush/reset/outputSeek/
  exact) must be BIT-EXACT; with the real shared-memory FFT the short-horizon error is bounded;
* the multi-GPU sharding helper under gloo, world_size 2.
"""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import signals

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rms(a):
    return float(np.sqrt(np.mean(np.square(a, dtype=np.float64))))


# ------------------------------------------------------------------ the shipped library
def test_library_exports_every_declared_symbol(cuda_lib):
    import signalsmith_stretch_b200 as pkg

    header = open(os.path.join(ROOT, "include", "b200_stretch.h")).read()
    declared = sorted(set(re.findall(r"\b(b200s_[a-z0-9_]+)\s*\(", header)))
    assert declared == sorted(pkg.ABI_SYMBOLS)
    lib = ctypes.CDLL(cuda_lib)
    for name in declared:
        assert hasattr(lib, name), name


def test_no_cpu_fallback(cuda_lib):
    """Without a GPU the product must refuse to create an engine (not silently run on the CPU)."""
    import torch

    import signalsmith_stretch_b200 as pkg

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(pkg.StretchError, match="no usable CUDA device"):
        pkg.BatchStretch(2)
    with pytest.raises(pkg.StretchError, match="not found"):
        pkg.BatchStretch(2, lib_path="/nonexistent/libb200stretch.so")


def test_product_sources_never_touch_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "signalsmith_stretch_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle/" not in src and "import oracle" not in src and "from oracle" not in src, f


# ------------------------------------------------------------------ kernels under the emulator
def _emu(path, batch, exact_math=True, gen=0, pairs=False):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(batch, lib_path=path)
    e.set_tuning(3, 1 if exact_math else 0)  # the bit-exact checks run the phase chain in the reference's own arithmetic
    if gen:
        e.set_tuning(0, gen)  # generation of the stereo direct chain kernel (0 = the default)
    if pairs:
        e.set_tuning(5, 1)  # mono plain path: two streams per warp on the packed wavefront (k_chain_direct6<.., DUAL>)
    return e


def _oracle_batch(oracle_port, cfg, x, ratio, chunk):
    outs = []
    for s in range(x.shape[0]):
        o = oracle_port()
        cfg(o)
        outs.append(signals.run_single(o, x[s], ratio, chunk))
    return np.stack(outs)


SMALL = [
    ("identity", lambda o: o.configure(1, 512, 128), 1, 1.0, 1000),
    ("radix3_K192_+5st", lambda o: (o.configure(1, 384, 96), o.setTransposeSemitones(5, 0)), 1, 1.0, 1000),
    ("radix5_K160_-4st_tonality", lambda o: (o.configure(1, 320, 80), o.setTransposeSemitones(-4, 0.2)), 1, 1.0, 777),
    ("stereo_0.8x", lambda o: o.configure(2, 512, 128), 2, 0.8, 640),
    ("stereo_1.5x_+3st", lambda o: (o.configure(2, 512, 128), o.setTransposeSemitones(3, 0.25)), 2, 1.5, 900),
    ("split_400_160", lambda o: (o.configure(1, 400, 160, True), o.setTransposeSemitones(2, 0)), 1, 1.0, 500),
    ("formant_comp_stereo", lambda o: (o.configure(2, 512, 128), o.setTransposeSemitones(12, 0), o.setFormantFactor(1, True), o.setFormantBase(200 / 48000)), 2, 1.0, 640),
    ("formant_+3st_1.25x", lambda o: (o.configure(1, 512, 128), o.setTransposeSemitones(-3, 0.2), o.setFormantSemitones(3, False), o.setFormantBase(300 / 48000)), 1, 1.25, 640),
    # setFormantBase(0): automatic pitch estimate per block (estimateFrequency :929-966, k_pitch), state carried over calls
    ("formant_auto_pitch_stereo", lambda o: (o.configure(2, 512, 128), o.setTransposeSemitones(5, 0), o.setFormantFactor(1, True), o.setFormantBase(0)), 2, 1.0, 640),
    ("formant_auto_pitch_+4st_0.8x", lambda o: (o.configure(1, 384, 96), o.setFormantSemitones(4, False), o.setFormantBase(0)), 1, 0.8, 500),
    # long vertical steps that do not divide the 12-step unrolling of k_chain_t (its FIFOs are then shifted, not rotated)
    ("L5_mapped_stereo", lambda o: (o.configure(2, 500, 100), o.setTransposeSemitones(4, 0.2)), 2, 1.0, 700),
    ("L8_mapped_mono_1.25x", lambda o: (o.configure(1, 512, 64), o.setTransposeSemitones(-3, 0)), 1, 1.25, 640),
    ("L2_mapped_formants", lambda o: (o.configure(1, 512, 256), o.setTransposeSemitones(5, 0), o.setFormantFactor(1, True), o.setFormantBase(150 / 48000)), 1, 1.0, 1024),
]


@pytest.mark.parametrize("name,cfg,C,ratio,chunk", SMALL, ids=[c[0] for c in SMALL])
def test_kernel_logic_bit_exact_vs_oracle(emu_libs, oracle_port, name, cfg, C, ratio, chunk):
    x = signals.batch("harmonic", 2, C, 4000, 48000)
    g = _emu(emu_libs["exact"], 2)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


LONG_CALLS = [
    # (name, configure, channels, out/in, input samples, chunk): blocks per call chosen so that the direct chain
    # kernel runs with several warps per stream (hand-off ring between warps) and with more than one round
    ("stereo_0.8x_2warps", lambda o: o.configure(2, 512, 128), 2, 0.8, 9000, 3000),   # 24 blocks: 2 warps of 16
    ("stereo_0.8x_2rounds", lambda o: o.configure(2, 512, 128), 2, 0.8, 14000, 9000),  # 71 blocks: 4 warps, 2 rounds
    ("mono_1.25x_3warps", lambda o: o.configure(1, 384, 96), 1, 1.25, 9000, 8000),     # 84 blocks: 3 warps of 32
]


@pytest.mark.parametrize("name,cfg,C,ratio,n,chunk", LONG_CALLS, ids=[c[0] for c in LONG_CALLS])
def test_long_calls_multi_warp_chain_bit_exact_vs_oracle(emu_libs, oracle_port, name, cfg, C, ratio, n, chunk):
    x = signals.batch("harmonic", 2, C, n, 48000)
    g = _emu(emu_libs["exact"], 2)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


PRESET_CALLS = [
    # preset sizes run on the paired-FFT kernels (stft2.cuh); with the oracle's FFT swapped in, their staging,
    # job pairing and fused overlap-add sweep must reproduce the oracle bit for bit
    ("default_stereo_0.8x", lambda o: o.presetDefault(2, 48000.0), 2, 0.8, 12800, 5760),  # aligned 16-byte staging, two calls
    ("default_mono_1.25x_odd", lambda o: o.presetDefault(1, 48000.0), 1, 1.25, 12000, 4999),  # unaligned chunks, odd block counts
    ("cheaper_mono_split", lambda o: o.presetCheaper(1, 48000.0), 1, 1.0, 14000, 6000),
    # the benchmark's call shape: 32 blocks per call, i.e. all 32 lanes of the packed stereo wavefront, two calls
    ("default_stereo_0.8x_32_blocks_per_call", lambda o: o.presetDefault(2, 48000.0), 2, 0.8, 2 * 57600, 46080),
    # presetCheaper stereo without transposition: K = 2560, L = 3 (odd lane skew), split computation in the vector overlap-add
    ("cheaper_stereo_1.5x", lambda o: o.presetCheaper(2, 48000.0), 2, 1.5, 16000, 11520),
    # more than 32 blocks per call: a second group of lanes whose first block takes its predecessor from the rows the
    # first group wrote (stereo), several warps per stream handing over through shared memory (mono)
    ("default_stereo_1.25x_40_blocks_per_call", lambda o: o.presetDefault(2, 48000.0), 2, 1.25, 2 * 46080, 57600),
    ("default_mono_0.8x_40_blocks_per_call", lambda o: o.presetDefault(1, 48000.0), 1, 0.8, 2 * 72000, 57600),
]


@pytest.mark.parametrize("name,cfg,C,ratio,n,chunk", PRESET_CALLS, ids=[c[0] for c in PRESET_CALLS])
def test_preset_pair_kernels_bit_exact_vs_oracle(emu_libs, oracle_port, name, cfg, C, ratio, n, chunk):
    x = signals.batch("harmonic", 1, C, n, 48000)
    g = _emu(emu_libs["exact"], 1)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


FULL_SIZE = [
    # the BASELINE configurations at their real sizes (K = 3072), several calls, two streams
    ("config1_mono_44k_+12st_ton8k", lambda o: (o.presetDefault(1, 44100.0), o.setTransposeSemitones(12, 8000 / 44100)), 1, 1.0, 30000, 10584),
    ("config3_mono_+7st_ton8k", lambda o: (o.presetDefault(1, 48000.0), o.setTransposeSemitones(7, 8000 / 48000)), 1, 1.0, 30000, 11520),
    ("config4_stereo_+12st_formant_comp_200Hz", lambda o: (o.presetDefault(2, 48000.0), o.setTransposeSemitones(12, 0), o.setFormantFactor(1, True), o.setFormantBase(200 / 48000)), 2, 1.0, 30000, 11520),
    ("config4_auto_pitch", lambda o: (o.presetDefault(2, 48000.0), o.setTransposeSemitones(12, 0), o.setFormantFactor(1, True), o.setFormantBase(0)), 2, 1.0, 30000, 11520),
    ("config5_cheaper_mono_2x_-5st", lambda o: (o.presetCheaper(1, 48000.0), o.setTransposeSemitones(-5, 0.1)), 1, 2.0, 20000, 15360),
]


@pytest.mark.parametrize("name,cfg,C,ratio,n,chunk", FULL_SIZE, ids=[c[0] for c in FULL_SIZE])
def test_baseline_configurations_full_size_bit_exact_vs_oracle(emu_libs, oracle_port, name, cfg, C, ratio, n, chunk):
    x = signals.batch("harmonic", 2, C, n, 48000)
    g = _emu(emu_libs["exact"], 2)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


FREQ_MAPS = [
    ("pwl_monotone_K256", lambda o: (o.configure(2, 512, 128), o.setFreqMapTable(*signals.PWL_MONOTONE)), 2, 1.0, 4000, 640),
    ("pwl_folding_K256_0.8x", lambda o: (o.configure(1, 512, 128), o.setFreqMapTable(*signals.PWL_FOLDING)), 1, 0.8, 4000, 640),
    ("pwl_folding_default_stereo", lambda o: (o.presetDefault(2, 48000.0), o.setFreqMapTable(*signals.PWL_FOLDING)), 2, 1.0, 20000, 5760),
    ("pwl_monotone_formant_comp", lambda o: (o.configure(2, 512, 128), o.setFreqMapTable(*signals.PWL_MONOTONE), o.setFormantFactor(1, True), o.setFormantBase(200 / 48000)), 2, 1.0, 4000, 640),
]


@pytest.mark.parametrize("name,cfg,C,ratio,n,chunk", FREQ_MAPS, ids=[c[0] for c in FREQ_MAPS])
def test_set_freq_map_table_bit_exact_vs_oracle(emu_libs, oracle_port, name, cfg, C, ratio, n, chunk):
    """setFreqMap (:120-122) through b200s_set_freq_map_table: the per-peak mapFreq (:874), the formant target map
    (:1020) and -- with a map that folds back -- the non-monotone output-map replay, on the CUDA kernels."""
    x = signals.batch("harmonic", 2, C, n, 48000)
    g = _emu(emu_libs["exact"], 2)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


def test_tabulated_smooth_map_error_is_small(emu_libs, oracle_port):
    """The facade tabulates a callable on 2049 points (include/signalsmith-stretch/signalsmith-stretch.h): for a smooth
    map (the oracle's quadratic stand-in) the piecewise-linear table deviates by < 1e-7 of the sample rate, and the
    output stays within the short-horizon tolerance of the analytic map."""
    a, b = 1.2, 0.5
    fin = np.linspace(0.0, 0.5, 2049).astype(np.float32)
    fout = (np.float32(a) * fin + np.float32(b) * fin * fin).astype(np.float32)
    mid = ((fin[1:].astype(np.float64) + fin[:-1]) / 2)
    assert np.abs((fout[1:].astype(np.float64) + fout[:-1]) / 2 - (a * mid + b * mid * mid)).max() < 1e-7
    x = signals.batch("harmonic", 1, 2, 6000, 48000)

    def cfg_tab(o):
        o.configure(2, 512, 128)
        o.setFreqMapTable(fin, fout)

    def cfg_quad(o):
        o.configure(2, 512, 128)
        o.setFreqMapQuadratic(a, b)

    g = _emu(emu_libs["exact"], 1)
    cfg_tab(g)
    y = signals.run_batch(g, x, 1.0, 640)
    ref = _oracle_batch(oracle_port, cfg_quad, x, 1.0, 640)
    lat = g.outputLatency() + g.inputLatency()
    assert rms((y - ref)[..., : lat + 8 * 128]) <= 1e-4


RANDOM_STRETCH = [
    # beyond 2x stretch the reference draws a random time factor per bin and direction (:639-640,:749,:769) from
    # std::default_random_engine(seed): k_plan advances the stream's engine state per block, k_prep forms the twists
    # with the per-bin draws (one modular multiplication each), the generic chain consumes them
    ("mono_K256_3x", lambda o: o.configure(1, 512, 128), 1, 3.0, 2000, 1500, 77),
    ("stereo_K256_2.5x", lambda o: o.configure(2, 512, 128), 2, 2.5, 2000, 1280, 12345),
    ("stereo_K256_2.5x_+3st_mapped", lambda o: (o.configure(2, 512, 128), o.setTransposeSemitones(3, 0.25)), 2, 2.5, 2000, 1280, 5),
    ("default_stereo_2.5x_interleaved_spectra", lambda o: o.presetDefault(2, 48000.0), 2, 2.5, 9216, 11520, 3),
    ("cheaper_mono_4x", lambda o: o.presetCheaper(1, 48000.0), 1, 4.0, 6000, 7680, 2**31 + 9),
]


@pytest.mark.parametrize("name,cfg,C,ratio,n,chunk,seed", RANDOM_STRETCH, ids=[c[0] for c in RANDOM_STRETCH])
def test_random_time_factors_beyond_2x_bit_exact_vs_oracle(emu_libs, name, cfg, C, ratio, n, chunk, seed):
    from oracle.hdrref import CpuStretch
    from signalsmith_stretch_b200 import BatchStretch

    x = signals.batch("harmonic", 2, C, n, 48000)
    g = BatchStretch(2, seed=seed, lib_path=emu_libs["exact"])
    g.set_tuning(3, 1)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = []
    for s in range(2):
        o = CpuStretch("orc", seed)
        cfg(o)
        ref.append(signals.run_single(o, x[s], ratio, chunk))
    ref = np.stack(ref)
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


def test_random_path_mixed_with_clean_calls_bit_exact_vs_oracle(emu_libs):
    """Calls below and beyond 2x in one stream (the engine state advances only in random blocks; the first block after a
    ratio change mixes both intervals), a seek at a slow rate (its time factor goes to the next block, :164,:312), and
    flush with playbackRate 0 (input interval 0, every block random); two streams of one batch where only ONE is silent
    for a while, so that their schedules -- and their engine states -- diverge."""
    from oracle.hdrref import CpuStretch
    from signalsmith_stretch_b200 import BatchStretch

    x = signals.batch("harmonic", 2, 2, 30000, 48000)
    x[1, :, 6000:16000] = 0  # stream 1 falls silent (bypass after two blocks of silence) while stream 0 keeps stretching

    def seq(o, wrap, unwrap, s):
        o.configure(2, 512, 128)
        outs, pos = [], 0

        def run(n_in, n_out):
            nonlocal pos
            outs.append(unwrap(o.process(wrap(s[..., pos:pos + n_in]), n_out)))
            pos += n_in

        run(1024, 1024)
        run(400, 1280)      # 3.2x
        run(1024, 1024)     # back to 1x: the first block's interval mixes the two ratios
        o.seek(wrap(s[..., pos:pos + 700]), 0.3)
        pos += 700
        run(600, 1536)      # 2.56x after a seek at rate 0.3
        run(2000, 2000)
        run(512, 1536)      # 3x
        run(3000, 3000)
        run(3000, 3000)
        run(640, 1600)
        outs.append(unwrap(o.flush(900, 0.0)))
        run(1024, 1024)
        return np.concatenate(outs, axis=-1)

    g = BatchStretch(2, seed=4242, lib_path=emu_libs["exact"])
    g.set_tuning(3, 1)
    y = seq(g, lambda a: a, lambda a: np.array(a), x)  # (copies: the binding reuses its output array)
    for st in range(2):
        o = CpuStretch("orc", 4242)
        r = seq(o, lambda a: a, lambda a: a, x[st])
        assert np.array_equal(y[st], r), "stream %d: max diff %g" % (st, np.abs(y[st] - r).max())


def test_parameters_change_between_calls_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Switching between the kernel paths from call to call -- plain stereo (packed direct chain on interleaved spectra,
    state carried through k_plan / k_commit in both layouts), frequency map (k_prep + generic chain), formants with
    automatic pitch, back to plain, a time-stretch change -- must carry every piece of state across: same sequence on
    the oracle, bit for bit."""
    x = signals.batch("harmonic", 1, 2, 8 * 5760, 48000)

    def seq(o, wrap, unwrap):
        o.presetDefault(2, 48000.0)
        outs, pos = [], 0

        def run(n_in, n_out):
            nonlocal pos
            outs.append(unwrap(o.process(wrap(x[0][:, pos:pos + n_in]), n_out)))
            pos += n_in

        run(5760, 5760)
        run(7200, 5760)              # 0.8x: re-analysis every block
        o.setTransposeSemitones(3, 0.2)
        run(5760, 5760)              # mapped
        o.setFormantFactor(1.2, True)
        o.setFormantBase(0)
        run(5760, 5760)              # mapped + formants, automatic pitch
        run(2880, 5760)              # 2x stretch with formants
        o.setTransposeSemitones(0, 0)
        o.setFormantFactor(1, False)
        run(5760, 5760)              # plain again: interleaved state rebuilt from the planar one
        run(7200, 5760)
        return np.concatenate(outs, axis=1)

    ref = seq(oracle_port(), lambda a: a, lambda a: a)
    got = seq(_emu(emu_libs["exact"], 1), lambda a: a[None], lambda a: np.asarray(a)[0])
    assert np.array_equal(ref, got), "max diff %g" % np.abs(ref - got).max()


def test_silence_bypass_and_energy_scan_at_preset_size_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Stereo preset path through silence: the energy scan of k_plan (which stops at the first loud tile), the silence
    counter, the first bypass call that zeroes the spectra (also their interleaved copies), bypass copies, and the
    restart -- including a chunk that is silent except for its last samples (the scan must not stop early there)."""
    x = signals.batch("harmonic", 1, 2, 6 * 5760, 48000)[0]
    z = np.zeros((2, 5760), np.float32)
    late = z.copy()
    late[:, -7:] = 0.25  # loud only at the very end of the chunk

    def seq(o, wrap, unwrap):
        o.presetDefault(2, 48000.0)
        outs = []
        for chunk in (x[:, :5760], x[:, 5760:11520], z, z, z, z[:, :2880], late, z, x[:, 11520:17280], x[:, 17280:23040]):
            outs.append(unwrap(o.process(wrap(chunk), 5760)))
        return np.concatenate(outs, axis=1)

    ref = seq(oracle_port(), lambda a: a, lambda a: a)
    got = seq(_emu(emu_libs["exact"], 1), lambda a: a[None], lambda a: np.asarray(a)[0])
    assert np.array_equal(ref, got), "max diff %g" % np.abs(ref - got).max()


def test_streams_with_different_schedules_in_one_batch_bit_exact_vs_oracle(emu_libs, oracle_port):
    """One launch sequence, diverging streams: stream 1 falls silent (silence counter, then bypass: no analysis jobs, no
    blocks) and comes back while streams 0 and 2 keep going -- the persistent analysis kernel has to skip the job slots
    of the bypassed stream (items looked up two ahead), every kernel its empty block list."""
    S, C, calls, n = 3, 2, 9, 5760
    x = signals.batch("harmonic", S, C, calls * n, 48000)
    x[1, :, 2 * n:7 * n] = 0.0  # stream 1: silent for five calls
    g = _emu(emu_libs["exact"], S)
    g.presetDefault(C, 48000.0)
    y = signals.run_batch(g, x, 1.0, n)
    ref = _oracle_batch(oracle_port, lambda o: o.presetDefault(C, 48000.0), x, 1.0, n)
    for s_ in range(S):
        assert np.array_equal(y[s_], ref[s_]), "stream %d: max diff %g" % (s_, np.abs(y[s_] - ref[s_]).max())


def test_randomised_configurations_bit_exact_vs_oracle(emu_libs, oracle_port):
    """Differential fuzz, fixed seed: random sizes (generic kernels) and presets at several sample rates (paired-FFT
    kernels, K = 3072 / 2560 / other), mono / stereo, split or not, time ratios, transposition with and without
    tonality limit, formants with fixed and automatic pitch, aligned and odd chunk sizes -- bit for bit against the
    oracle.  (Ratios whose time factor exceeds 2 are left out: the reference draws random numbers there, DESIGN.md 6.)"""
    rng = np.random.default_rng(2024)
    for it in range(36):
        preset = it % 3 == 2
        C = int(rng.integers(1, 3))
        split = bool(rng.integers(0, 2))
        ratio = float(rng.choice([0.5, 0.75, 0.8, 1.0, 1.25, 1.5, 1.8]))
        semis = float(rng.choice([0, 0, 3, -4, 7, 12]))
        ton = float(rng.choice([0, 0.1, 0.25]))
        form = int(rng.choice([0, 0, 1, 2, 3]))
        if preset:
            sr = float(rng.choice([32000, 40000, 44100, 48000]))
            cheaper = bool(rng.integers(0, 2))
            H = int(sr * (0.04 if cheaper else 0.03))
            chunk = int(rng.choice([H * 4, H * 3 + 5, H * 2 + 1, 4 * (H // 2)]))
            conf = lambda o: (o.presetCheaper if cheaper else o.presetDefault)(C, sr, split)  # noqa: E731
        else:
            sr = 48000.0
            block = int(rng.choice([256, 320, 384, 400, 512, 640, 768, 1000, 1024]))
            interval = int(block // rng.choice([3, 4, 5, 6]))
            chunk = int(rng.choice([interval * 2, interval * 3 + 7, 480, 1000, block * 2]))
            conf = lambda o: o.configure(C, block, interval, split)  # noqa: E731

        def cfg(o):
            conf(o)
            o.setTransposeSemitones(semis, ton)
            if form == 1:
                o.setFormantFactor(1, True)
                o.setFormantBase(200 / sr)
            elif form == 2:
                o.setFormantSemitones(3, False)
                o.setFormantBase(300 / sr)
            elif form == 3:
                o.setFormantSemitones(-2, True)
                o.setFormantBase(0)

        n_out = chunk * int(rng.integers(2, 4))
        x = signals.batch("harmonic", 1, C, int(round(n_out / ratio)) + 8, int(sr))
        g = _emu(emu_libs["exact"], 1)
        cfg(g)
        y = signals.run_batch(g, x, ratio, chunk)
        ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
        assert np.array_equal(y, ref), (it, preset, C, sr, split, ratio, semis, ton, form, chunk, float(np.abs(y - ref).max()))


@pytest.mark.parametrize("gen", [4, 6])
@pytest.mark.parametrize("idx", [0, 3, 4, 5])
def test_stereo_chain_generations_bit_exact_vs_oracle(emu_libs, oracle_port, gen, idx):
    """Both packed stereo chain kernels (k_chain_direct4 and its leaner successor k_chain_direct6, which forms the twists
    one / two bins behind the preliminary prediction, keeps products instead of factors in its FIFOs and hands the finals
    from lane to lane through shared memory), selected explicitly: aligned calls, all 32 lanes busy, odd lane skew (L = 3),
    and more than 32 blocks per call (a second group of lanes continuing from the rows the first group wrote)."""
    name, cfg, C, ratio, n, chunk = PRESET_CALLS[idx]
    assert C == 2
    x = signals.batch("harmonic", 2, C, n, 48000)
    g = _emu(emu_libs["exact"], 2, gen=gen)
    cfg(g)
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
    assert np.array_equal(y, ref), "%s gen %d: max diff %g" % (name, gen, np.abs(y - ref).max())


def test_stereo_chain_generation6_with_diverging_streams_and_silence(emu_libs, oracle_port):
    S, C, calls, n = 3, 2, 7, 5760
    x = signals.batch("harmonic", S, C, calls * n, 48000)
    x[1, :, 2 * n:5 * n] = 0.0
    g = _emu(emu_libs["exact"], S, gen=6)
    g.presetDefault(C, 48000.0)
    y = signals.run_batch(g, x, 0.8, int(n * 0.8))
    ref = _oracle_batch(oracle_port, lambda o: o.presetDefault(C, 48000.0), x, 0.8, int(n * 0.8))
    assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


MONO_PAIRS = [
    # mono plain calls with two streams per warp on the packed wavefront (k_chain_direct6<.., DUAL>, tuning key 5); the odd
    # stream of the batch and pairs whose schedules differ run alone through the same kernel.  (block, interval) -> L = 1 .. 8
    ("L1", 256, 256, 0.8), ("L2", 512, 256, 1.25), ("L3", 384, 128, 0.8), ("L4", 512, 128, 0.5), ("L5", 500, 100, 1.6), ("L8", 512, 64, 0.8),
]


@pytest.mark.parametrize("name,B,H,ratio", MONO_PAIRS, ids=[c[0] for c in MONO_PAIRS])
def test_mono_stream_pairs_on_the_packed_chain_bit_exact_vs_oracle(emu_libs, oracle_port, name, B, H, ratio):
    S = 5  # two pairs and an odd stream
    x = signals.batch("harmonic", S, 1, 12 * B, 48000)
    x[3, :, 3 * B:7 * B] = 0.0  # stream 3 falls silent for a while: the pair (2, 3) stops sharing its schedule
    g = _emu(emu_libs["exact"], S, pairs=True)
    g.configure(1, B, H)
    chunk = 40 * H + 17  # more than 32 blocks per call: a second group of lanes
    y = signals.run_batch(g, x, ratio, chunk)
    ref = _oracle_batch(oracle_port, lambda o: o.configure(1, B, H), x, ratio, chunk)
    for s_ in range(S):
        assert np.array_equal(y[s_], ref[s_]), "stream %d: max diff %g" % (s_, np.abs(y[s_] - ref[s_]).max())


def test_mono_stream_pairs_at_preset_size_bit_exact_vs_oracle(emu_libs, oracle_port):
    for cfg, ratio, n, chunk in ((lambda o: o.presetDefault(1, 48000.0), 0.8, 2 * 57600, 46080), (lambda o: o.presetCheaper(1, 48000.0), 2.0, 30000, 20000)):
        x = signals.batch("harmonic", 2, 1, n, 48000)
        g = _emu(emu_libs["exact"], 2, pairs=True)
        cfg(g)
        y = signals.run_batch(g, x, ratio, chunk)
        ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
        assert np.array_equal(y, ref), "max diff %g" % np.abs(y - ref).max()


def test_fast_chain_arithmetic_of_generation6_and_of_mono_pairs_stays_within_tolerance(emu_libs, oracle_port):
    cases = [(PRESET_CALLS[3], 6), (PRESET_CALLS[4], 6), (("default_mono_0.8x", lambda o: o.presetDefault(1, 48000.0), 1, 0.8, 2 * 57600, 46080), 0)]
    for (name, cfg, C, ratio, n, chunk), gen in cases:
        x = signals.batch("harmonic", 2, C, n, 48000)
        g = _emu(emu_libs["exact"], 2, exact_math=False, gen=gen, pairs=(C == 1))
        cfg(g)
        y = signals.run_batch(g, x, ratio, chunk)
        ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
        assert not np.array_equal(y, ref), name
        H = g.intervalSamples()
        head = g.outputLatency() + int(g.inputLatency() * ratio) + 8 * H
        assert rms((y - ref)[..., :head]) <= 2e-6, (name, rms((y - ref)[..., :head]))
        assert rms(y - ref) <= 1e-3, (name, rms(y - ref))


def test_fast_chain_arithmetic_stays_within_tolerance(emu_libs, oracle_port):
    """The default (fast: fused multiply-add, reciprocal / rsqrt) arithmetic of the stereo direct chain against the
    oracle, FFT substituted: not bit-exact by construction, but within float rounding over a short horizon -- also with
    all 32 lanes of the wavefront busy (32 blocks per call) and with the odd lane skew of presetCheaper."""
    for name, cfg, C, ratio, n, chunk in (PRESET_CALLS[0], PRESET_CALLS[3], PRESET_CALLS[4]):
        x = signals.batch("harmonic", 1, C, n, 48000)
        g = _emu(emu_libs["exact"], 1, exact_math=False)
        cfg(g)
        y = signals.run_batch(g, x, ratio, chunk)
        ref = _oracle_batch(oracle_port, cfg, x, ratio, chunk)
        assert not np.array_equal(y, ref), name  # the fast path really ran
        H = g.intervalSamples()
        head = g.outputLatency() + int(g.inputLatency() * ratio) + 8 * H
        assert rms((y - ref)[..., :head]) <= 2e-6, (name, rms((y - ref)[..., :head]))  # float rounding over the first blocks
        assert rms(y - ref) <= 1e-3, (name, rms(y - ref))  # chaotic beyond (SURVEY.md section 0.4): the reference's own -60 dB criterion


def test_api_sequence_bit_exact_vs_oracle(emu_libs, oracle_port):
    """seek / silence bypass / flush / reset / outputSeek / exact through the batched ABI."""
    x = signals.harmonic(6000, 48000)[None]

    def seq(o, wrap, unwrap):
        o.configure(1, 512, 128)
        o.setTransposeSemitones(3, 0)
        outs = []
        o.seek(wrap(x[:, :300]), 1.0)
        outs.append(unwrap(o.process(wrap(x[:, 300:780]), 480)))
        z = np.zeros((1, 3000), np.float32)
        outs.append(unwrap(o.process(wrap(z[:, :1200]), 1200)))  # counts silence
        outs.append(unwrap(o.process(wrap(z[:, :400]), 400)))    # first bypass call: state zeroed
        outs.append(unwrap(o.process(wrap(z[:, :400]), 500)))    # bypass, in != out
        outs.append(unwrap(o.process(wrap(x[:, 800:1760]), 900)))
        outs.append(unwrap(o.flush(100, 1.0)))
        outs.append(unwrap(o.process(wrap(x[:, 2000:2480]), 480)))
        outs.append(unwrap(o.flush(500, 1.1)))
        o.reset()
        outs.append(unwrap(o.process(wrap(x[:, 2000:2480]), 240)))
        o.outputSeek(wrap(x[:, : o.outputSeekLength(1.3)]))
        outs.append(unwrap(o.process(wrap(x[:, 500:1124]), 480)))
        ok, e = o.exact(wrap(x[:, :4000]), 5000)
        assert ok
        outs.append(unwrap(e))
        ok, e = o.exact(wrap(x[:, :100]), 5000)  # too short: zero output, false (:471-479)
        assert not ok and not np.any(e)
        return np.concatenate(outs, axis=1)

    ref = seq(oracle_port(), lambda a: a, lambda a: a)
    got = seq(_emu(emu_libs["exact"], 1), lambda a: a[None], lambda a: np.asarray(a)[0])
    assert np.array_equal(ref, got), "max diff %g" % np.abs(ref - got).max()


def test_async_host_calls_equal_blocking_calls(emu_libs):
    """b200s_process_async (pipelined host-buffer calls over chained stream groups) gives what blocking calls give."""
    import ctypes

    x = signals.batch("harmonic", 4, 1, 1024, 48000)
    outs = []
    for use_async in (False, True):
        g = _emu(emu_libs["float"], 4)
        g.set_tuning(2, 2)  # two stream groups of two streams
        g.configure(1, 256, 64)
        g.setTransposeSemitones(3, 0)
        ys = [np.zeros((4, 1, 256), np.float32) for _ in range(4)]
        for k in range(4):
            xi = np.ascontiguousarray(x[:, :, 256 * k:256 * (k + 1)])
            if use_async:
                g.process_host_ptr_async(xi.ctypes.data, 256, ys[k].ctypes.data, 256)
                keep = xi  # noqa: F841  (the emulator copies synchronously; on a GPU the buffer must outlive the call)
            else:
                g.process_host_ptr(xi.ctypes.data, 256, ys[k].ctypes.data, 256)
        g.synchronize()
        outs.append(np.concatenate(ys, axis=2))
    assert np.array_equal(outs[0], outs[1])


def test_pcm16_boundary_equals_float_path_with_the_tools_conversions(emu_libs):
    """b200s_process_pcm16: int16 in / out with the conversions on the device == the float call fed sample / 32768,
    its output rounded to nearest (halves away from zero) and clamped -- what the reference's tool does around the path."""
    x = signals.batch("harmonic", 4, 2, 3 * 640, 48000)
    x16 = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    outs = []
    for pcm in (True, False):
        g = _emu(emu_libs["float"], 4)
        g.set_tuning(2, 2)  # two stream groups
        g.configure(2, 512, 128)
        g.setTransposeSemitones(-2, 0.3)
        ys = []
        for k in range(3):
            chunk = np.ascontiguousarray(x16[:, :, 640 * k:640 * (k + 1)])
            if pcm:
                ys.append(g.process_pcm16(chunk, 640))
            else:
                v = g.process((chunk.astype(np.float32) * np.float32(1 / 32768)), 640) * np.float32(32768)
                ys.append(np.clip(np.sign(v) * np.floor(np.abs(v) + np.float32(0.5)), -32768, 32767).astype(np.int16))
        outs.append(np.concatenate(ys, axis=2))
    assert np.abs(outs[0]).max() > 300
    assert np.array_equal(outs[0], outs[1])


def test_api_sequence_at_preset_size_stereo_bit_exact_vs_oracle(emu_libs, oracle_port):
    """seek / process / flush / reset / outputSeek / exact on the stereo preset kernels (paired FFT, packed chain, ring
    in shared memory): the state these calls touch lives in the layouts of the preset path."""
    x = signals.batch("harmonic", 1, 2, 60000, 48000)[0]

    def seq(o, wrap, unwrap):
        o.presetDefault(2, 48000.0)
        outs = []
        o.seek(wrap(x[:, :3000]), 1.25)
        outs.append(unwrap(o.process(wrap(x[:, 3000:10200]), 5760)))
        outs.append(unwrap(o.process(wrap(x[:, 10200:13800]), 2880)))
        outs.append(unwrap(o.flush(1000, 1.0)))
        outs.append(unwrap(o.process(wrap(x[:, 14000:19760]), 5760)))
        outs.append(unwrap(o.flush(7000, 1.2)))
        o.reset()
        outs.append(unwrap(o.process(wrap(x[:, 20000:22880]), 2880)))
        o.outputSeek(wrap(x[:, 23000:23000 + o.outputSeekLength(0.8)]))
        outs.append(unwrap(o.process(wrap(x[:, 30000:34608]), 5760)))
        ok, e = o.exact(wrap(x[:, 35000:55000]), 16000)
        assert ok
        outs.append(unwrap(e))
        return np.concatenate(outs, axis=1)

    ref = seq(oracle_port(), lambda a: a, lambda a: a)
    got = seq(_emu(emu_libs["exact"], 1), lambda a: a[None], lambda a: np.asarray(a)[0])
    assert np.array_equal(ref, got), "max diff %g" % np.abs(ref - got).max()


def test_streams_are_independent_and_chunking_is_invariant(emu_libs):
    """A stream's output does not depend on its neighbours in the batch nor on the call chunking."""
    x = signals.batch("harmonic", 3, 1, 3000, 48000)
    cfg = lambda o: (o.configure(1, 384, 96), o.setTransposeSemitones(4, 0.2))  # noqa: E731
    g3 = _emu(emu_libs["float"], 3)
    cfg(g3)
    y3 = signals.run_batch(g3, x, 1.0, 3000)
    g1 = _emu(emu_libs["float"], 1)
    cfg(g1)
    y1 = signals.run_batch(g1, x[1:2], 1.0, 250)
    assert np.array_equal(y3[1:2], y1)


def test_shared_memory_fft_accuracy(emu_libs, oracle_port):
    """Real float Stockham FFT (radix 4/2 + 3 or 5) vs the oracle's double FFT: identity config is a
    pure delay to 1e-6 for every radix mix, presets included."""
    for cfg, C, n in ((lambda o: o.configure(1, 384, 96), 1, 2000),      # K=192 = 3*4^3
                      (lambda o: o.configure(1, 320, 80), 1, 2000),      # K=160 = 5*4^2*2
                      (lambda o: o.configure(1, 256, 64), 1, 2000),      # K=128 = 4^3*2
                      (lambda o: o.presetDefault(1, 48000.0), 1, 5760 + 1440 * 2),   # K=3072: paired in-place FFT, mono pairs
                      (lambda o: o.presetDefault(2, 48000.0), 2, 5760 + 1440 * 3),   # K=3072: channel pairs, odd block count
                      (lambda o: o.presetCheaper(2, 48000.0), 2, 4800 + 1920 * 3),   # K=2560 = 16*16*10, split computation
                      (lambda o: o.presetDefault(1, 44100.0), 1, 5292 + 1323 * 2)):  # K=3072 with an odd history length (unaligned staging)
        x = signals.batch("harmonic", 1, C, n, 48000)
        g = _emu(emu_libs["float"], 1)
        cfg(g)
        y = signals.run_batch(g, x, 1.0, n)
        ref = _oracle_batch(oracle_port, cfg, x, 1.0, n)
        assert rms(y - ref) <= 1e-6


def test_unsupported_features_fail_loudly(emu_libs):
    from signalsmith_stretch_b200 import StretchError

    g = _emu(emu_libs["float"], 1)
    with pytest.raises(StretchError):
        g.process(np.zeros((1, 1, 10), np.float32), 10)  # not configured
    with pytest.raises(StretchError, match="channels"):
        g.configure(3, 512, 128)
    with pytest.raises(StretchError, match="unknown key"):
        g.set_tuning(99, 0)
    # 192 kHz presets: K = 12288 bands, beyond the shared-memory FFT (the largest size, 6144, is 96 kHz): refused with
    # B200S_EUNSUPPORTED (-4) before anything is launched
    g.presetDefault(1, 96000.0)
    before = g.kernel_launches()
    for preset in ("presetDefault", "presetCheaper"):
        with pytest.raises(StretchError, match="error -4"):
            getattr(g, preset)(1, 192000.0)
    assert g.kernel_launches() == before and g.bands() == 6144


def test_file_mode_caller_against_the_oracle(emu_libs, oracle_port, tmp_path):
    """cmd/stretch_cli.cpp (WAV in, the reference tool's outputSeek / process / flush stages through the C++ facade,
    16-bit WAV out), linked against the emulator build of the library: the file it writes is the oracle's output,
    driven through the same stages and rounded to 16 bits, sample for sample."""
    import struct

    exe = os.path.join(os.path.dirname(emu_libs["exact"]), "stretch_cli_emu")
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(ROOT, "cmd", "stretch_cli.cpp"),
                    emu_libs["exact"], "-Wl,-rpath," + os.path.dirname(emu_libs["exact"])], check=True)
    sr, n, C, semitones, time = 48000, 20000, 1, 4.0, 1.25
    x = signals.batch("harmonic", 1, C, n, sr)[0]
    x = (np.round(x * 32768) / 32768).astype(np.float32)
    src, dst = str(tmp_path / "in.wav"), str(tmp_path / "out.wav")
    data = np.ascontiguousarray(np.round(x.T * 32768).astype("<i2")).tobytes()  # a 16-bit PCM file, as the reference tool reads
    with open(src, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, 1, C, sr, sr * C * 2, C * 2, 16))
        f.write(b"data" + struct.pack("<I", len(data)) + data)
    r = subprocess.run([exe, src, dst, "--semitones=%g" % semitones, "--time=%g" % time], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    d = open(dst, "rb").read()
    assert d[:4] == b"RIFF" and d[8:12] == b"WAVE" and struct.unpack("<H", d[22:24])[0] == C and struct.unpack("<I", d[24:28])[0] == sr
    y = np.frombuffer(d[44:], dtype="<i2").reshape(-1, C).T
    o = oracle_port()
    o.presetDefault(C, float(sr))
    o.setTransposeSemitones(semitones, 8000.0 / sr)
    o.setFormantSemitones(0.0, False)
    o.setFormantBase(100.0 / sr)
    n_out = int(round(n * time))
    seek = o.outputSeekLength(np.float32(1 / time))
    out_index = n_out - o.intervalSamples()
    in_index = int(round((out_index + o.outputLatency()) / time)) + o.inputLatency()
    xp = np.zeros((C, max(in_index, seek)), np.float32)
    xp[:, :n] = x
    o.outputSeek(xp[:, :seek])
    ref = np.concatenate([o.process(xp[:, seek:in_index], out_index), o.flush(n_out - out_index)], axis=1)
    v = ref * np.float32(32768.0)
    q = np.clip(np.sign(v) * np.floor(np.abs(v) + np.float32(0.5)), -32768, 32767).astype(np.int16)  # std::round: halves away from zero
    assert y.shape == q.shape
    assert np.array_equal(y, q), "max diff %d LSB" % np.abs(y.astype(np.int32) - q).max()


# ------------------------------------------------------------------ sharding, gloo world_size 2
def test_shard_range_partitions_the_batch():
    from signalsmith_stretch_b200.shard import shard_range

    for batch in (1, 7, 8, 1024, 8192):
        for world in (1, 2, 3, 8):
            cover = []
            for r in range(world):
                lo, hi = shard_range(batch, r, world)
                cover += list(range(lo, hi))
            assert cover == list(range(batch))


def test_gloo_two_ranks_reduce_the_throughput_counter():
    script = r"""
import os, sys
sys.path.insert(0, %r)
import torch.distributed as dist
from signalsmith_stretch_b200.shard import shard_range, reduce_throughput
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%%s" %% os.environ["PORT"], rank=int(os.environ["RANK"]), world_size=2)
lo, hi = shard_range(9, dist.get_rank(), 2)
total, tmax = reduce_throughput((hi - lo) * 1000, 1.0 + dist.get_rank(), dist)
assert total == 9000 and tmax == 2.0, (total, tmax)
dist.destroy_process_group()
print("ok")
""" % ROOT
    import socket

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [subprocess.Popen([sys.executable, "-c", script], env=dict(os.environ, RANK=str(r), PORT=str(port)),
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    for p in procs:
        out, err = p.communicate(timeout=120)
        assert p.returncode == 0 and "ok" in out, err


# ------------------------------------------------------------------ the live / streaming caller (web/web-wrapper.js:215-332)
class _OneStream:
    """Adapter: a one-stream oracle object behind the BatchStretch calls LiveBatch makes (batch of 1)."""

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


@pytest.mark.parametrize("bank", [None, "numpy"], ids=["host_windows", "device_bank"])
def test_live_batch_seek_every_quantum_bit_exact_vs_oracle(emu_libs, oracle_port, bank):
    """SURVEY.md 8(f) rank 4: the reference's live wrapper seeks every audio quantum with the current time-map
    segment's rate and renders `process(0, quantum)` (web-wrapper.js:314-315).  LiveBatch does that for a batch with
    one b200s_seek_rates + one b200s_process per quantum; three streams with their own rates / offsets / loop / stop
    times against three oracle objects driven by the same loop, bit for bit."""
    from signalsmith_stretch_b200.live import LiveBatch

    sr, S, C, quantum = 48000.0, 3, 2, 128
    audio = signals.batch("harmonic", S, C, 12000, 48000)
    g = _emu(emu_libs["exact"], S)
    g.configure(C, 512, 128)
    # bank: the streams' audio in a "device" bank (host memory under the emulator), windows cut by the seek kernel
    # (b200s_live_seek); None: windows gathered on the host and uploaded (b200s_seek_rates)
    live = LiveBatch(g, sr, bank=bank)
    refs = []
    for s in range(S):
        o = oracle_port()
        o.configure(C, 512, 128)
        refs.append(LiveBatch(_OneStream(o), sr))

    def both(fn):
        fn(live, lambda s: s)
        for s, r in enumerate(refs):
            fn(r, lambda _s, s=s: 0 if _s == s else None)

    def setup(lv, idx):
        for s in range(S):
            i = idx(s)
            if i is None:
                continue
            lv.add_buffers(i, audio[s])
        for s, kw in enumerate([dict(rate=0.8, offset=0.01), dict(rate=1.0, offset=0.0), dict(rate=1.3, offset=0.02)]):
            i = idx(s)
            if i is not None:
                lv.start(i, when=0.004 * s, **kw)
        i = idx(2)
        if i is not None:  # stream 2 loops between 50 ms and 110 ms of its input
            lv.schedule(i, dict(outputTime=0.03, loopStart=0.05, loopEnd=0.11), adjust_previous=False)

    both(setup)
    outs, ref_outs = [], [[] for _ in range(S)]
    for qn in range(40):
        if qn == 25:  # stream 0 stops; stream 1 slows down now and is steered to input 0.1 s at output 0.2 s (adjustPrevious)
            both(lambda lv, idx: [lv.stop(idx(0)) if idx(0) is not None else None,
                                  lv.schedule(idx(1), dict(rate=0.6)) if idx(1) is not None else None,
                                  lv.schedule(idx(1), dict(outputTime=0.2, input=0.1), adjust_previous=True) if idx(1) is not None else None])
        outs.append(live.process(quantum))
        for s, r in enumerate(refs):
            ref_outs[s].append(r.process(quantum)[0])
    y = np.concatenate(outs, axis=-1)
    for s in range(S):
        r = np.concatenate(ref_outs[s], axis=-1)
        if s == 0:  # the stopped stream: compared while it plays (documented difference of a batch call afterwards)
            n = 25 * quantum
            assert np.array_equal(y[s][:, :n], r[:, :n]), "stream 0: max diff %g" % np.abs(y[s][:, :n] - r[:, :n]).max()
        else:
            assert np.array_equal(y[s], r), "stream %d: max diff %g" % (s, np.abs(y[s] - r).max())
    assert np.abs(y).max() > 0.05


def test_live_time_map_semantics():
    """The time-map bookkeeping of LiveBatch against the worklet's rules (web/web-wrapper.js:45-108,227-231,271-279),
    on a stub engine: inheritance from the earliest replaced point, backwards extrapolation, stop = rate 0 from there on,
    adjustPrevious re-aiming, loop wrap, and the window positions handed to the seek."""
    from signalsmith_stretch_b200.live import LiveBatch

    class Stub:
        batch = 2

        def __init__(self):
            self.calls = []

        def channels(self):
            return 1

        def inputLatency(self):
            return 300

        def outputLatency(self):
            return 200

        def seek(self, win, rates):
            self.calls.append(("seek", win.copy(), np.array(rates)))

        def process(self, x, n):
            self.calls.append(("process", x.shape[-1], n))
            return np.zeros((2, 1, n), np.float32)

    sr = 1000.0
    e = Stub()
    lv = LiveBatch(e, sr)  # host mode (the stub has no bank)
    ramp = np.arange(5000, dtype=np.float32)
    lv.add_buffers(0, ramp)
    lv.add_buffers(1, ramp)
    a = lv.start(0, when=0.1, offset=2.0, rate=0.5)
    assert (a["output"], a["input"], a["rate"], a["active"]) == (0.1, 2.0, 0.5, True)
    b = lv.schedule(0, dict(outputTime=0.05, rate=2.0))  # replaces the point at 0.1: inherits from it, input extrapolated back
    assert b["active"] is True and abs(b["input"] - (2.0 + (0.05 - 0.1) * 0.5)) < 1e-12 and b["rate"] == 2.0
    assert [pt["output"] for pt in lv.time_maps[0]] == [0.05]  # (the worklet prunes up to the NEW point's time, :98-101)
    c = lv.stop(0, when=1.0)  # position at the stop: 1.975 + 0.95 * 2
    assert abs(c["input"] - (1.975 + 0.95 * 2.0)) < 1e-12 and c["active"] is False
    d = lv.schedule(0, dict(outputTime=2.0))  # a stopped segment stands still
    assert abs(d["input"] - c["input"]) < 1e-12
    # (the worklet prunes the map up to the NEW point's output time, :98-101, so a point scheduled for the future becomes the
    #  map's first entry at once and is looked up -- extrapolated backwards -- until its time comes: mirrored, quirk included)
    assert [pt["output"] for pt in lv.time_maps[0]] == [2.0] and lv.time_maps[0][0]["active"] is False
    # stream 1: play from 0 at rate 1, then a point "input 3.0 at output 2.0" with adjustPrevious
    lv.start(1, when=0.0, offset=0.0, rate=1.0)
    p = lv.schedule(1, dict(outputTime=2.0, input=3.0), adjust_previous=True)
    assert p["rate"] == 1.0 and [pt["output"] for pt in lv.time_maps[1]] == [2.0]
    # a quantum at current time 0: output time = 0.2 (output latency).  Stream 0 is stopped (silent window, rate 1); stream 1
    # is on the line through (output 2.0, input 3.0) with rate 1: input 1.2 s, + input latency, window = the 500 samples before
    lv.process(100)
    kind, win, rates = e.calls[0]
    assert kind == "seek" and e.calls[1] == ("process", 0, 100)
    assert not win[0].any() and rates[0] == 1.0
    end1 = int(np.floor((3.0 + (0.2 - 2.0) * 1.0 + 0.3) * sr + 0.5))
    assert end1 == 1500 and np.array_equal(win[1, 0], ramp[end1 - 500:end1]) and rates[1] == 1.0
    # loop: stream 1 loops [0.4, 0.6) s of its input; once past the end, the position wraps back by the loop length
    lv.schedule(1, dict(loopStart=1.3, loopEnd=1.5))
    for _ in range(6):
        lv.process(100)
    seg = lv.time_maps[1][0]
    pos = lv._in[1] + (lv.current_time + 0.2 - seg["output"]) * seg["rate"]
    assert 1.3 <= pos < 1.5 + 0.1
