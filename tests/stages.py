"""Stage-by-stage comparison of a BatchStretch with the oracle (tests/test_gpu_stages.py, tests/test_host_stages.py).

After every call both sides expose the input history, the last block's analysis spectra (Band::input / prevInput) and
the overlap-add state (pending output and window products).  An analysis spectrum is a pure function of the input
history: no phase feedback, no chaos.  So, unlike the output audio, it can be held after any number of calls to a bound
of the float FFT's own rounding against the oracle's double-precision FFT.
"""
import numpy as np

# Analysis spectra, per stream-channel, against the double FFT: rms(dX) <= SPEC_RMS * rms(X) and
# max|dX| <= SPEC_MAX * max|X|.  Measured on an H100 (and bit-identically in the emulator's float build) over every FFT
# family of tests/test_gpu_stages.py: <= 1.9e-7 rms and <= 2.2e-7 max; a twiddle or radix stage a few times less
# accurate than it should be fails these.
SPEC_RMS = 5e-7
SPEC_MAX = 1e-6
# pending output under the identity configuration, through the analysis and the synthesis FFT (measured <= 2.2e-6)
PEND_RMS = 5e-6


def _rel(d, ref, how):
    """Per stream-channel error of d relative to ref: 'rms' or 'max'.  Zero where both are zero, inf where only ref is."""
    d = np.abs(d.astype(np.complex128) if np.iscomplexobj(d) else d.astype(np.float64))
    r = np.abs(ref.astype(np.complex128) if np.iscomplexobj(ref) else ref.astype(np.float64))
    if how == "rms":
        num, den = np.sqrt(np.mean(d * d, axis=-1)), np.sqrt(np.mean(r * r, axis=-1))
    else:
        num, den = d.max(axis=-1), r.max(axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(num == 0, 0.0, num / np.where(den == 0, 0.0, den))


def oracle_states(oracles):
    st = [o.signal_state() for o in oracles]
    return {k: np.stack([s[k] for s in st]) for k in ("history", "pending", "pendingWp", "input", "prevInput")}


def engine_states(e):
    return {k: np.array(e.get_state(k)) for k in ("history", "pending", "pendingWp", "input", "prevInput")}


def run(e, oracles, x, chunk, calls):
    """Feed x [S][C][n] to the engine and to one oracle per stream, `calls` calls of `chunk` samples at rate 1; return
    the list of (engine states, oracle states) after every call."""
    out = []
    for k in range(calls):
        xin = np.ascontiguousarray(x[:, :, k * chunk:(k + 1) * chunk])
        e.process(xin, chunk)
        for s, o in enumerate(oracles):
            o.process(xin[s], chunk)
        out.append((engine_states(e), oracle_states(oracles)))
    return out


def check(states, pending=True):
    """Assert the stage bounds on every call; return the worst (spectrum rms, spectrum max, pending rms) seen."""
    worst = [0.0, 0.0, 0.0]
    for k, (g, o) in enumerate(states):
        assert np.array_equal(g["history"], o["history"]), "call %d: input history differs" % k
        for key in ("input", "prevInput"):
            assert np.all(np.isfinite(g[key].view(np.float32))), (k, key)
            er, em = _rel(g[key] - o[key], o[key], "rms"), _rel(g[key] - o[key], o[key], "max")
            worst[0], worst[1] = max(worst[0], float(er.max())), max(worst[1], float(em.max()))
            assert er.max() <= SPEC_RMS and em.max() <= SPEC_MAX, (k, key, er.max(), em.max())
        if pending:
            ep = _rel(g["pending"] - o["pending"], o["pending"], "rms")
            worst[2] = max(worst[2], float(ep.max()))
            assert ep.max() <= PEND_RMS, (k, ep.max())
            assert np.array_equal(g["pendingWp"], o["pendingWp"]), "call %d: window products differ" % k
    return worst
