"""CPU counterparts of tests/test_gpu_stages.py, on the emulator builds of the CUDA sources (tests/cuda_emu).

* the analysis spectra of the real float FFT kernels against the oracle's double FFT, per bin, after every call
  (tests/stages.py), at the small sizes the emulator runs quickly and at the preset sizes of 48 kHz;
* the branch-free division / square root of the exact phase chain (kernels.cuh fdivq / fsqrtq) on the edge operands,
  with the emulator modelling the PTX special values of rcp.approx.ftz / rsqrt.approx.ftz;
* loud, near-silent and spectrally extreme inputs through every exact chain path, bit for bit against the oracle
  (the oracle's FFT swapped in).  On int16-level input |phase|^2 overflows to +inf in the chain, where the reference
  gets energy / inf = 0; the division must do the same, not produce NaN.
"""
import numpy as np
import pytest

import signals
import stages

# (name, configure, channels): every FFT family the emulator can run in seconds
STAGE_SIZES = [
    ("K160_radix5", lambda o: o.configure(1, 320, 80), 1),
    ("K192_radix3", lambda o: o.configure(2, 384, 96), 2),
    ("K384_split", lambda o: o.configure(1, 768, 192, True), 1),
    ("K640", lambda o: o.configure(2, 1280, 320), 2),
    ("K1024_from_1000", lambda o: o.configure(1, 2000, 500), 1),
    ("default_48k_K3072_stereo", lambda o: o.presetDefault(2, 48000.0), 2),
    ("cheaper_48k_K2560_mono_split", lambda o: o.presetCheaper(1, 48000.0), 1),
]
STAGE_KINDS = ("harmonic_1", "dc", "nyquist", "impulse_train", "harmonic_32768")


def _engine(path, S, cfg, seed=0):
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(S, seed=seed, lib_path=path)
    e.set_tuning(3, 1)
    cfg(e)
    return e


def _stage_input(C, calls, H, sr=48000):
    n = calls * H
    return np.concatenate([signals.edge(k, 1, C, n, sr) for k in STAGE_KINDS], axis=0)


@pytest.mark.parametrize("name,cfg,C", STAGE_SIZES, ids=[c[0] for c in STAGE_SIZES])
def test_float_fft_analysis_spectra_per_bin_vs_double_fft(emu_libs, oracle_port, name, cfg, C):
    """The shared-memory float FFT kernels (the same sources the GPU runs), per bin against the oracle's double FFT after
    every call: no round trip for errors to cancel in.  Harmonic, DC, Nyquist, impulse train and int16 level."""
    e = _engine(emu_libs["float"], len(STAGE_KINDS), cfg)
    H, B = e.intervalSamples(), e.blockSamples()
    calls = B // H + 3
    x = _stage_input(C, calls, H)
    oracles = []
    for _ in STAGE_KINDS:
        o = oracle_port()
        cfg(o)
        oracles.append(o)
    worst = stages.check(stages.run(e, oracles, x, H, calls))
    print("%s: worst spectrum rms %.2e max %.2e, pending %.2e" % (name, *worst))


def test_fast_div_sqrt_are_correctly_rounded_on_the_edge_operands(emu_libs):
    """k_selftest_divsqrt under the emulator: the sequences of fdivq / fsqrtq (seeded by the modelled rcp / rsqrt) against
    IEEE division and square root on the normal range and on the edge classes: zero, subnormal, tiny and huge
    numerators, divisors up to FLT_MAX and +-inf, subnormal / zero / infinite square-root arguments."""
    from signalsmith_stretch_b200 import BatchStretch

    e = BatchStretch(1, lib_path=emu_libs["float"])
    assert e.selftest_divsqrt(1 << 21, 99) == (0, 0)


# (name, configure, channels, out/in ratio, seed): the exact chain paths
EDGE_CONFIGS = [
    ("mono_+7st_tonality_chain_t", lambda o: (o.configure(1, 512, 128), o.setTransposeSemitones(7, 0.2)), 1, 1.0, 0),
    ("stereo_plain_exact_direct", lambda o: o.configure(2, 512, 128), 2, 0.8, 0),
    ("stereo_formant_comp", lambda o: (o.configure(2, 512, 128), o.setTransposeSemitones(12, 0), o.setFormantFactor(1, True), o.setFormantBase(200 / 48000)), 2, 1.0, 0),
    ("stereo_random_2.5x", lambda o: o.configure(2, 512, 128), 2, 2.5, 77),
    ("default_mono_+7st_tonality", lambda o: (o.presetDefault(1, 48000.0), o.setTransposeSemitones(7, 8000 / 48000)), 1, 1.0, 0),
    ("default_stereo_plain_exact_packed", lambda o: o.presetDefault(2, 48000.0), 2, 0.8, 0),
]
EDGE_KINDS = ("harmonic_1e-6", "harmonic_3000", "harmonic_32768", "loud_and_tiny", "loud_and_zero", "dc", "nyquist", "impulses")


@pytest.mark.parametrize("name,cfg,C,ratio,seed", EDGE_CONFIGS, ids=[c[0] for c in EDGE_CONFIGS])
def test_extreme_inputs_bit_exact_vs_oracle(emu_libs, name, cfg, C, ratio, seed):
    from oracle.hdrref import CpuStretch

    kinds = [k for k in EDGE_KINDS if C == 2 or not k.startswith("loud_and")]
    probe = _engine(emu_libs["exact"], 1, cfg)
    H, B = probe.intervalSamples(), probe.blockSamples()
    n_out = 6 * H + B
    n_in = int(round(n_out / ratio))
    x = np.concatenate([signals.edge(k, 1, C, n_in, 48000) for k in kinds], axis=0)
    e = _engine(emu_libs["exact"], len(kinds), cfg, seed)
    y = signals.run_batch(e, x, ratio, 3 * H)
    for s, k in enumerate(kinds):
        o = CpuStretch("orc", seed)
        cfg(o)
        ref = signals.run_single(o, x[s], ratio, 3 * H)
        assert np.all(np.isfinite(ref)), k
        assert np.all(np.isfinite(y[s])), "%s: %d non-finite output samples" % (k, int(np.sum(~np.isfinite(y[s]))))
        assert np.array_equal(y[s], ref), "%s: max diff %g" % (k, np.abs(y[s] - ref).max())
