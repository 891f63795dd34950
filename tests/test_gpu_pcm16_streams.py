"""The 16-bit PCM list calls on the H100: chained wait = 0 calls through pinned buffers equal the float twin bit for bit.

One engine runs b200s_run_streams_pcm16 with wait = 0, its twin b200s_run_streams_async with the same lists fed
x16 / 32768; the twin's output is converted as b200s_process_pcm16 converts it (test_pcm16_streams.to_pcm16).  The copies
and kernels of consecutive calls overlap on the device here, which the emulator cannot show.
"""
import numpy as np
import pytest

import signals
from test_pcm16_streams import to_float, to_pcm16

SR = 48000.0
PROC, OSEEK, FLUSH = 1, 3, 4


@pytest.mark.gpu
def test_chained_list_calls_with_a_turnover_equal_the_float_twin(cuda_lib):
    """256 stereo presetDefault slots: four chained calls over 10 % of the slots, a turnover call (a FLUSH on one slot, an
    OUTPUT_SEEK on another: it joins), four chained calls over every slot in shuffled order; the whole sequence twice, with
    no device allocation in the second round.  Outputs and every slot's record equal the float twin's."""
    import torch

    from signalsmith_stretch_b200 import BatchStretch

    S, C = 256, 2
    rng = np.random.default_rng(23)
    engines = []
    for _ in range(2):
        e = BatchStretch(S)
        e.presetDefault(C, SR)
        engines.append(e)
    pcm, flt = engines
    H = pcm.intervalSamples()
    n_out = 8 * H
    n_in = int(round(n_out / 0.8))
    tenth, every = rng.permutation(S)[:S // 10].astype(np.int32), rng.permutation(S).astype(np.int32)
    x = signals.batch("harmonic", S, C, 2 * 9 * n_in, 48000)
    x16 = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    del x
    pos = np.zeros(S, int)

    def pinned(a):
        return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()

    def sequence():
        calls = [(tenth, None)] * 4 + [(tenth, "turnover")] + [(every, None)] * 4
        bufs = []
        for lst, kind in calls:
            ops = np.full(lst.size, PROC, np.int32)
            ni, no = np.full(lst.size, n_in, np.int32), np.full(lst.size, n_out, np.int32)
            if kind:
                ops[1], ni[1], no[1] = FLUSH, 0, 3 * H
                ops[2], ni[2], no[2] = OSEEK, 6000, 0
            src = np.zeros((lst.size, C, n_in), np.int16)
            for i, s in enumerate(lst):
                src[i, :, :ni[i]] = x16[s, :, pos[s]:pos[s] + ni[i]]
                pos[s] += ni[i]
            b = {"in16": pinned(src), "inf": pinned(to_float(src)),
                 "out16": pinned(np.full((lst.size, C, n_out), 0x7fff, np.int16)),
                 "outf": pinned(np.full((lst.size, C, n_out), np.nan, np.float32))}
            pcm.run_pcm16_host_ptr(ops, b["in16"].data_ptr(), n_in, ni, b["out16"].data_ptr(), n_out, no, playback_rates=1.0,
                                   streams=lst, wait=False)
            flt.run_streams_host_ptr(lst, ops, b["inf"].data_ptr(), n_in, ni, b["outf"].data_ptr(), n_out, no, playback_rates=1.0,
                                     wait=False)
            bufs.append(b)
        pcm.synchronize()
        flt.synchronize()
        for k, b in enumerate(bufs):
            yf = b["outf"].numpy()
            assert not np.isnan(yf).any(), k
            y, want = b["out16"].numpy(), to_pcm16(yf)
            assert np.array_equal(y, want), "call %d: %d samples differ" % (k, int((y != want).sum()))
            assert np.abs(y).max() > 300, k
        assert pcm.export_streams(range(S)).tobytes() == flt.export_streams(range(S)).tobytes()

    sequence()
    allocs = pcm.device_allocations()
    sequence()
    assert pcm.device_allocations() == allocs
    assert pcm.unserved_random_blocks() == 0
