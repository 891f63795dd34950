"""GPU tests stage by stage and at the edges of the input range.  `pytest -m gpu` on an H100.

A. The analysis spectra of every FFT family (paired 3072 / 2560, both generations at the preset sizes, the generic kernels
   at every other preset size from 8 to 96 kHz, configure() sizes with a radix-2 or odd last stage), per bin against the
   oracle's double FFT after every call (bounds in tests/stages.py: no feedback, so they hold at any horizon).
B. The GPU's analysis spectra equal the emulator's float build bit for bit (the FFT uses only .rn intrinsics and
   __fmaf_rn, the library is built with --fmad=false, the emulator with -ffp-contract=off, the tables come from the same
   host code), and so does the whole path in exact arithmetic (tuning key 3), whose division / square root is correctly
   rounded on the device.  The fast mode uses the SFU approximations and is not bit-identical by construction.
C. Loud (int16-level), near-silent, zero, DC, Nyquist and impulse inputs through the plain fast stereo path, the
   transposed mono path (k_chain_t), formant compensation, 96 kHz stereo (k_chain_direct2, exact) and the random path:
   finite output, the short-horizon gate relative to the input level, level match.
"""
import numpy as np
import pytest

import signals
import stages

pytestmark = pytest.mark.gpu


def rms(a):
    return float(np.sqrt(np.mean(np.square(a, dtype=np.float64))))


@pytest.fixture(scope="module")
def gpu(cuda_lib):
    import torch

    assert torch.cuda.is_available(), "these tests need a GPU"
    from signalsmith_stretch_b200 import BatchStretch

    return lambda batch, seed=0: BatchStretch(batch, seed=seed)


# ------------------------------------------------------------------ A. analysis spectra against the double FFT
# (name, configure, channels, scalar FFT generation forced (tuning key 1))
FFT_FAMILIES = [
    ("paired_3072_stereo_48k", lambda o: o.presetDefault(2, 48000.0), 2, 0),
    ("paired_3072_mono_44k", lambda o: o.presetDefault(1, 44100.0), 1, 0),
    ("paired_2560_stereo_split_48k", lambda o: o.presetCheaper(2, 48000.0), 2, 0),
    ("scalar_3072_stereo_48k", lambda o: o.presetDefault(2, 48000.0), 2, 1),
    ("scalar_2560_mono_split_48k", lambda o: o.presetCheaper(1, 48000.0), 1, 1),
    ("generic_512_mono_8k", lambda o: o.presetDefault(1, 8000.0), 1, 0),
    ("generic_1024_stereo_16k", lambda o: o.presetDefault(2, 16000.0), 2, 0),
    ("generic_1536_mono_22k", lambda o: o.presetDefault(1, 22050.0), 1, 0),
    ("generic_1280_stereo_split_22k", lambda o: o.presetCheaper(2, 22050.0), 2, 0),
    ("generic_2048_stereo_32k", lambda o: o.presetDefault(2, 32000.0), 2, 0),
    ("generic_5120_mono_split_96k", lambda o: o.presetCheaper(1, 96000.0), 1, 0),
    ("generic_6144_stereo_88k", lambda o: o.presetDefault(2, 88200.0), 2, 0),
    ("generic_6144_stereo_96k", lambda o: o.presetDefault(2, 96000.0), 2, 0),
    ("configure_160_radix5", lambda o: o.configure(1, 320, 80), 1, 0),
    ("configure_192_radix3_stereo", lambda o: o.configure(2, 384, 96), 2, 0),
    ("configure_384_split", lambda o: o.configure(1, 768, 192, True), 1, 0),
    ("configure_640_stereo", lambda o: o.configure(2, 1280, 320), 2, 0),
    ("configure_1000_to_1024", lambda o: o.configure(1, 2000, 500), 1, 0),
]
STAGE_KINDS = ("harmonic_1", "dc", "nyquist", "impulse_train", "harmonic_32768")


def _stage_run(e, cfg, C, sr, oracle_port):
    H, B = e.intervalSamples(), e.blockSamples()
    calls = B // H + 3  # the window fills, then three more blocks
    x = np.concatenate([signals.edge(k, 1, C, calls * H, sr) for k in STAGE_KINDS], axis=0)
    oracles = []
    for _ in STAGE_KINDS:
        o = oracle_port()
        cfg(o)
        oracles.append(o)
    return stages.run(e, oracles, x, H, calls)


@pytest.mark.parametrize("name,cfg,C,v1", FFT_FAMILIES, ids=[f[0] for f in FFT_FAMILIES])
def test_analysis_spectra_per_bin_vs_double_fft(gpu, oracle_port, name, cfg, C, v1):
    e = gpu(len(STAGE_KINDS))
    cfg(e)
    e.set_tuning(1, v1)
    e.set_tuning(3, 1)  # pending is compared too: identity configuration, exact chain arithmetic
    worst = stages.check(_stage_run(e, cfg, C, 48000, oracle_port))
    print("%s (K = %d): worst spectrum rms %.2e max %.2e, pending %.2e" % (name, e.bands(), *worst))


# ------------------------------------------------------------------ B. GPU and emulator bit-identical
# (not the scalar generation forced at 3072 / 2560: the emulator build keeps the superseded specialisations k_analyse<3072> /
# <2560> (B200S_KEEP_OLD_KERNELS) where the shipped library runs the generic k_analyse<0>, so the two run different kernels
# there -- equal in value, but not in the sign of every zero)
BIT_IDENTICAL = [f for f in FFT_FAMILIES if f[0] in ("paired_3072_stereo_48k", "paired_2560_stereo_split_48k", "generic_512_mono_8k",
                                                     "configure_160_radix5", "configure_192_radix3_stereo", "configure_1000_to_1024")]


@pytest.mark.parametrize("name,cfg,C,v1", BIT_IDENTICAL, ids=[f[0] for f in BIT_IDENTICAL])
def test_analysis_spectra_bit_identical_to_emulator(gpu, emu_libs, oracle_port, name, cfg, C, v1):
    from signalsmith_stretch_b200 import BatchStretch

    runs = []
    for e in (gpu(len(STAGE_KINDS)), BatchStretch(len(STAGE_KINDS), lib_path=emu_libs["float"])):
        cfg(e)
        e.set_tuning(1, v1)
        e.set_tuning(3, 1)
        runs.append(_stage_run(e, cfg, C, 48000, oracle_port))
    for k, ((g, _), (m, _)) in enumerate(zip(*runs)):
        for key in ("input", "prevInput", "pending"):
            assert np.array_equal(g[key].view(np.uint32), m[key].view(np.uint32)), (k, key, np.abs(g[key] - m[key]).max())


@pytest.mark.parametrize("C,ratio", [(1, 1.25), (2, 0.8)])
def test_exact_mode_output_bit_identical_to_emulator(gpu, emu_libs, C, ratio):
    """The whole path in exact arithmetic: the chain's fdivq / fsqrtq are IEEE on the device (k_selftest_divsqrt) and
    IEEE in the emulator, everything else is explicit .rn arithmetic."""
    from signalsmith_stretch_b200 import BatchStretch

    def cfg(o):
        o.configure(C, 512, 128)
        o.setTransposeSemitones(3 if C == 1 else 0, 0.2 if C == 1 else 0)

    x = np.concatenate([signals.batch("harmonic", 2, C, 4000, 48000), signals.edge("harmonic_32768", 1, C, 4000, 48000)])
    outs = []
    for e in (gpu(3), BatchStretch(3, lib_path=emu_libs["float"])):
        cfg(e)
        e.set_tuning(3, 1)
        outs.append(signals.run_batch(e, x, ratio, 640))
    assert np.all(np.isfinite(outs[0])) and np.abs(outs[0]).max() > 0.1
    assert np.array_equal(outs[0], outs[1]), np.abs(outs[0] - outs[1]).max()


# ------------------------------------------------------------------ C. extreme and edge inputs against the oracle
EDGE_CONFIGS = [
    # (name, configure, channels, sample rate, out/in ratio, seed)
    ("plain_stereo_fast", lambda o: o.presetDefault(2, 48000.0), 2, 48000, 0.8, 0),
    ("mono_+7st_tonality_chain_t", lambda o: (o.presetDefault(1, 48000.0), o.setTransposeSemitones(7, 8000 / 48000)), 1, 48000, 1.0, 0),
    ("stereo_formant_comp", signals.cfg_config4, 2, 48000, 1.0, 0),
    ("stereo_96k_plain_exact_direct2", lambda o: o.presetDefault(2, 96000.0), 2, 96000, 1.0, 0),
    ("stereo_random_2.5x", lambda o: o.presetDefault(2, 48000.0), 2, 48000, 2.5, 20261015),
]
EDGE_KINDS = ("harmonic_1e-6", "harmonic_1", "harmonic_3000", "harmonic_32768", "loud_and_tiny", "loud_and_zero", "dc", "nyquist", "impulses")


@pytest.mark.parametrize("name,cfg,C,sr,ratio,seed", EDGE_CONFIGS, ids=[c[0] for c in EDGE_CONFIGS])
def test_extreme_inputs_vs_oracle(gpu, oracle_port, name, cfg, C, sr, ratio, seed):
    from oracle.hdrref import CpuStretch

    kinds = [k for k in EDGE_KINDS if C == 2 or not k.startswith("loud_and")]
    e = gpu(len(kinds), seed)
    cfg(e)
    H, B = e.intervalSamples(), e.blockSamples()
    n_out = 12 * H + B
    x = np.concatenate([signals.edge(k, 1, C, int(round(n_out / ratio)), sr) for k in kinds], axis=0)
    y = signals.run_batch(e, x, ratio, 6 * H)
    lat = e.outputLatency() + int(e.inputLatency() * ratio)
    head, lvl = {}, {}
    for s, k in enumerate(kinds):
        o = CpuStretch("orc", seed)
        cfg(o)
        ref = signals.run_single(o, x[s], ratio, 6 * H)
        assert np.all(np.isfinite(ref)), k
        bad = int(np.sum(~np.isfinite(y[s])))
        assert bad == 0, "%s: %d non-finite output samples (the oracle's are finite)" % (k, bad)
        # per channel, relative to that channel's input level (the near-silent channel next to a loud one included)
        for c in range(C):
            level = rms(x[s, c])
            if level == 0:
                assert not np.any(y[s, c]) and not np.any(ref[c]), k  # an exactly zero channel stays exactly zero
                continue
            head[(k, c)] = rms((y[s, c] - ref[c])[: lat + 8 * H]) / level
            lvl[(k, c)] = 20 * np.log10(rms(y[s, c]) / rms(ref[c]))
    print(name, {key: "%.1e / %+.3f dB" % (head[key], lvl[key]) for key in head})
    # The median over the stream-channels: a single stream can go its own way within 8 blocks on a flipped hard decision
    # (peak picking, max channel) -- sparse impulses, whose blocks between the impulses hold only rounding-level bins, do
    # (H100: up to 1.3x their input level over 8 blocks, at matching level); the same inputs are bit-exact against the oracle
    # under the emulator with the oracle's FFT (tests/test_host_stages.py).  Beyond 2x the random time factors amplify the
    # FFT's rounding further (tests/test_gpu_parity.py::test_random_time_factors_beyond_2x_vs_oracle): there the
    # reference's own -60 dB criterion applies to the median.
    assert np.median(list(head.values())) <= (1e-3 if ratio > 2 else 1e-4), head
    # Level match over the whole output.  Exception: the Nyquist tone on the random path -- one partial at the band edge,
    # whose level after the overlap-add depends on the random phase realisation that a flipped decision changes (H100:
    # -1.4 dB, while every harmonic, DC, impulse and mixed-level stream of that run stays within 0.001 dB).
    assert all(abs(v) <= 0.1 for (k, c), v in lvl.items() if not (ratio > 2 and k == "nyquist")), lvl


def test_192k_is_unsupported_without_a_launch(gpu):
    """192 kHz presets ask for K = 12288 bands, beyond the shared-memory FFT (<= 6144): refused with B200S_EUNSUPPORTED,
    before anything is launched, and the engine keeps its previous configuration."""
    from signalsmith_stretch_b200 import StretchError

    e = gpu(1)
    e.presetDefault(2, 96000.0)
    before = e.kernel_launches()
    for preset in ("presetDefault", "presetCheaper"):
        with pytest.raises(StretchError, match="error -4"):
            getattr(e, preset)(2, 192000.0)
    assert e.kernel_launches() == before
    assert e.bands() == 6144
