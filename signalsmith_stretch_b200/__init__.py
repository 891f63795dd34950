"""signalsmith_stretch_b200 -- host-side mirror of the reference API over the H100 C-ABI library.

The product is `libb200stretch.so` (hand-written sm_90a CUDA behind the `extern "C"` ABI declared
in include/b200_stretch.h).  This module is a thin ctypes binding whose method names, argument
meaning and defaults follow `signalsmith::stretch::SignalsmithStretch<float>`
(/root/reference/signalsmith-stretch.h:34-491), batched: buffers are `[batch][channels][samples]`.

There is NO CPU fallback: importing is cheap, but constructing a `BatchStretch` raises
`StretchError` if the CUDA library is missing or no GPU is usable.
"""
import ctypes
import os

import numpy as np

__all__ = ["BatchStretch", "StretchError", "library_path", "build_library", "ABI_SYMBOLS"]

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB_NAME = "libb200stretch.so"

# every symbol include/b200_stretch.h declares
ABI_SYMBOLS = [
    "b200s_create", "b200s_destroy", "b200s_last_error", "b200s_version", "b200s_set_stream", "b200s_synchronize", "b200s_set_sub_batches", "b200s_set_tuning",
    "b200s_preset_default", "b200s_preset_cheaper", "b200s_configure", "b200s_reset", "b200s_reserve",
    "b200s_batch", "b200s_channels", "b200s_block_samples", "b200s_interval_samples", "b200s_input_latency",
    "b200s_output_latency", "b200s_split_computation", "b200s_seek_length", "b200s_output_seek_length",
    "b200s_fft_samples", "b200s_bands",
    "b200s_set_transpose_factor", "b200s_set_transpose_semitones", "b200s_set_formant_factor",
    "b200s_set_formant_semitones", "b200s_set_formant_base", "b200s_set_freq_map_table", "b200s_set_freq_map_table_per_stream",
    "b200s_set_transpose_factor_per_stream", "b200s_set_transpose_semitones_per_stream", "b200s_set_formant_factor_per_stream",
    "b200s_set_formant_semitones_per_stream", "b200s_set_formant_base_per_stream",
    "b200s_seek", "b200s_seek_rates", "b200s_live_seek", "b200s_output_seek", "b200s_process", "b200s_process_async", "b200s_process_pcm16", "b200s_flush", "b200s_exact",
    "b200s_seek_device", "b200s_process_device", "b200s_flush_device",
    "b200s_process_per_stream", "b200s_process_per_stream_async", "b200s_process_per_stream_device",
    "b200s_run_per_stream", "b200s_run_per_stream_async", "b200s_run_per_stream_device",
    "b200s_run_streams", "b200s_run_streams_async", "b200s_run_streams_device",
    "b200s_run_per_stream_pcm16", "b200s_run_streams_pcm16",
    "b200s_timer_start", "b200s_timer_stop", "b200s_kernel_launches", "b200s_device_allocations", "b200s_unserved_random_blocks", "b200s_profile_begin", "b200s_profile_end",
    "b200s_selftest_divsqrt",
    "b200s_state_size", "b200s_get_state", "b200s_set_state",
    "b200s_stream_state_bytes", "b200s_copy_streams", "b200s_export_streams", "b200s_import_streams", "b200s_clone",
]

STATE = {"input": 0, "prevInput": 1, "output": 2, "predEnergy": 4, "history": 20, "pending": 21, "pendingWp": 22}


class StretchError(RuntimeError):
    pass


def library_path():
    return os.path.join(_HERE, _LIB_NAME)


def build_library(verbose=False):
    """Compile csrc/engine.cu for sm_90a into the in-tree shared library (nvcc cross-compiles without a GPU)."""
    import subprocess

    src = os.path.join(_HERE, "csrc", "engine.cu")
    out = library_path()
    deps = [src] + [os.path.join(_HERE, "csrc", f) for f in ("kernels.cuh", "fft.cuh", "common.cuh", "chain_direct.cuh", "chain_direct2.cuh", "fft2.cuh", "stft2.cuh", "chain_direct3.cuh", "chain_direct4.cuh", "chain_ws.cuh", "chain_t.cuh", "chain_direct6.cuh", "state_copy.cuh")]
    deps.append(os.path.join(_ROOT, "include", "b200_stretch.h"))
    deps.append(os.path.abspath(__file__))  # the nvcc command line below
    if os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    # --fmad=false: a plain `a * b + c` is rounded twice, as in the reference and the oracle (both built without
    # contraction); the multiply-adds the kernels want fused are written as __fmaf_rn and stay fused.  Implicit
    # contraction left the float rounding of the mapped and random paths far enough from the oracle's to flip the
    # algorithm's hard decisions within the first blocks of some streams.
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "--fmad=false", "-lineinfo", "-std=c++17",
           "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", out, src]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    if os.environ.get("B200S_EXTRA_NVCC"):  # profiling builds (e.g. -DB200S_CHAIN_PROBES); never set for the shipped library
        cmd[1:1] = os.environ["B200S_EXTRA_NVCC"].split()
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise StretchError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return out


def _bind(lib):
    vp, ci, cf, cd, cl, cll = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_double, ctypes.c_long, ctypes.c_longlong
    fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)
    sig = {
        "b200s_create": (ci, [ci, cl, ci, ctypes.POINTER(vp)]), "b200s_destroy": (None, [vp]),
        "b200s_last_error": (ctypes.c_char_p, [vp]), "b200s_version": (ci, [ip, ip, ip]),
        "b200s_set_stream": (ci, [vp, vp]), "b200s_synchronize": (ci, [vp]), "b200s_set_sub_batches": (ci, [vp, ci]), "b200s_set_tuning": (ci, [vp, ci, ci]),
        "b200s_preset_default": (ci, [vp, ci, cf, ci]), "b200s_preset_cheaper": (ci, [vp, ci, cf, ci]),
        "b200s_configure": (ci, [vp, ci, ci, ci, ci]), "b200s_reset": (ci, [vp]), "b200s_reserve": (ci, [vp, ci, ci]),
        "b200s_output_seek_length": (ci, [vp, cf]),
        "b200s_set_transpose_factor": (ci, [vp, cf, cf]), "b200s_set_transpose_semitones": (ci, [vp, cf, cf]),
        "b200s_set_formant_factor": (ci, [vp, cf, ci]), "b200s_set_formant_semitones": (ci, [vp, cf, ci]),
        "b200s_set_formant_base": (ci, [vp, cf]), "b200s_set_freq_map_table": (ci, [vp, fp, fp, ci]),
        "b200s_set_freq_map_table_per_stream": (ci, [vp, ip, ci, ip, fp, fp]),
        "b200s_set_transpose_factor_per_stream": (ci, [vp, fp, fp]), "b200s_set_transpose_semitones_per_stream": (ci, [vp, fp, fp]),
        "b200s_set_formant_factor_per_stream": (ci, [vp, fp, ip]), "b200s_set_formant_semitones_per_stream": (ci, [vp, fp, ip]),
        "b200s_set_formant_base_per_stream": (ci, [vp, fp]),
        "b200s_seek": (ci, [vp, vp, ci, cd]), "b200s_seek_rates": (ci, [vp, vp, ci, ctypes.POINTER(cd)]), "b200s_live_seek": (ci, [vp, vp, cll, ctypes.POINTER(cll), ci, ctypes.POINTER(cd)]), "b200s_output_seek": (ci, [vp, vp, ci]),
        "b200s_process": (ci, [vp, vp, ci, vp, ci]), "b200s_process_async": (ci, [vp, vp, ci, vp, ci]), "b200s_process_pcm16": (ci, [vp, vp, ci, vp, ci, ci]), "b200s_flush": (ci, [vp, vp, ci, cf]),
        "b200s_exact": (ci, [vp, vp, ci, vp, ci, ip]),
        "b200s_seek_device": (ci, [vp, vp, ci, cd]), "b200s_process_device": (ci, [vp, vp, ci, vp, ci]),
        "b200s_flush_device": (ci, [vp, vp, ci, cf]),
        "b200s_process_per_stream": (ci, [vp, vp, ci, ip, vp, ci, ip]), "b200s_process_per_stream_async": (ci, [vp, vp, ci, ip, vp, ci, ip]),
        "b200s_process_per_stream_device": (ci, [vp, vp, ci, ip, vp, ci, ip]),
        "b200s_run_per_stream": (ci, [vp, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd)]),
        "b200s_run_per_stream_async": (ci, [vp, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd)]),
        "b200s_run_per_stream_device": (ci, [vp, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd)]),
        "b200s_run_streams": (ci, [vp, ci, ip, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd)]),
        "b200s_run_streams_async": (ci, [vp, ci, ip, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd)]),
        "b200s_run_streams_device": (ci, [vp, ci, ip, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd)]),
        "b200s_run_per_stream_pcm16": (ci, [vp, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd), ci]),
        "b200s_run_streams_pcm16": (ci, [vp, ci, ip, ip, vp, ci, ip, vp, ci, ip, ctypes.POINTER(cd), ci]),
        "b200s_timer_start": (ci, [vp]), "b200s_timer_stop": (ci, [vp, fp]), "b200s_kernel_launches": (cll, [vp]), "b200s_device_allocations": (cll, [vp]), "b200s_unserved_random_blocks": (cll, [vp]),
        "b200s_profile_begin": (ci, [vp]), "b200s_profile_end": (ci, [vp, fp, ip, ci]),
        "b200s_selftest_divsqrt": (ci, [vp, cll, cll, ctypes.POINTER(cll), ctypes.POINTER(cll)]),
        "b200s_state_size": (ci, [vp, ci]), "b200s_get_state": (ci, [vp, ci, vp]), "b200s_set_state": (ci, [vp, ci, vp]),
        "b200s_stream_state_bytes": (ci, [vp]), "b200s_copy_streams": (ci, [vp, ip, vp, ip, ci]),
        "b200s_export_streams": (ci, [vp, ip, ci, vp]), "b200s_import_streams": (ci, [vp, ip, ci, vp]),
        "b200s_clone": (ci, [vp, ctypes.POINTER(vp)]),
    }
    for name in ("batch", "channels", "block_samples", "interval_samples", "input_latency", "output_latency",
                 "split_computation", "seek_length", "fft_samples", "bands"):
        sig["b200s_" + name] = (ci, [vp])
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


_LIBS = {}


def _load(path):
    if path not in _LIBS:
        if not os.path.exists(path):
            raise StretchError(
                "CUDA library %s not found: build it with signalsmith_stretch_b200.build_library() "
                "(there is no CPU fallback)" % path)
        _LIBS[path] = _bind(ctypes.CDLL(path))
    return _LIBS[path]


def _host(a, shape):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    if a.size != int(np.prod(shape)):
        raise ValueError("expected %s floats, got %s" % (shape, a.shape))
    return a.reshape(shape)


def _is_torch_cuda(t):
    return hasattr(t, "data_ptr") and hasattr(t, "is_cuda") and t.is_cuda


class BatchStretch:
    """A batch of independent streams; one `SignalsmithStretch<float>` per stream (signalsmith-stretch.h:34)."""

    version = (1, 3, 2)  # :36
    # per-stream operations of run() (B200S_OP_* of include/b200_stretch.h)
    OP_SKIP, OP_PROCESS, OP_SEEK, OP_OUTPUT_SEEK, OP_FLUSH, OP_RESET = range(6)

    def __init__(self, batch=1, seed=0, device=0, lib_path=None):
        self._lib = _load(lib_path or library_path())
        h = ctypes.c_void_p()
        rc = self._lib.b200s_create(int(batch), int(seed), int(device), ctypes.byref(h))
        if rc != 0:
            raise StretchError("b200s_create failed (%d): %s" % (rc, self._lib.b200s_last_error(None).decode()))
        self._h = h
        self.batch = int(batch)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200s_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def _ck(self, rc):
        if rc != 0:
            raise StretchError("b200_stretch error %d: %s" % (rc, self._lib.b200s_last_error(self._h).decode()))

    # ---- configuration (:49-104) ----
    def presetDefault(self, nChannels, sampleRate, splitComputation=False):
        self._ck(self._lib.b200s_preset_default(self._h, nChannels, sampleRate, int(splitComputation)))

    def presetCheaper(self, nChannels, sampleRate, splitComputation=True):
        self._ck(self._lib.b200s_preset_cheaper(self._h, nChannels, sampleRate, int(splitComputation)))

    def configure(self, nChannels, blockSamples, intervalSamples, splitComputation=False):
        self._ck(self._lib.b200s_configure(self._h, nChannels, blockSamples, intervalSamples, int(splitComputation)))

    def reset(self):
        self._ck(self._lib.b200s_reset(self._h))

    def reserve(self, maxInputSamples, maxOutputSamples):
        self._ck(self._lib.b200s_reserve(self._h, maxInputSamples, maxOutputSamples))

    def channels(self):
        return self._lib.b200s_channels(self._h)

    def blockSamples(self):
        return self._lib.b200s_block_samples(self._h)

    def intervalSamples(self):
        return self._lib.b200s_interval_samples(self._h)

    def inputLatency(self):
        return self._lib.b200s_input_latency(self._h)

    def outputLatency(self):
        return self._lib.b200s_output_latency(self._h)

    def splitComputation(self):
        return bool(self._lib.b200s_split_computation(self._h))

    def seekLength(self):
        return self._lib.b200s_seek_length(self._h)

    def outputSeekLength(self, playbackRate):
        return self._lib.b200s_output_seek_length(self._h, playbackRate)

    def fftSamples(self):
        return self._lib.b200s_fft_samples(self._h)

    def bands(self):
        return self._lib.b200s_bands(self._h)

    # ---- parameters (:107-135): every argument is a scalar (broadcast to every stream) or one value per stream ----
    def _per_stream(self, *args):
        """args: (value, dtype) pairs.  None when every value is a scalar (the broadcast setter applies); otherwise every
        value as a contiguous array of `batch` entries (a scalar is repeated), for the per-stream setter."""
        if all(np.ndim(v) == 0 for v, _ in args):
            return None
        out = []
        for v, dt in args:
            a = np.ascontiguousarray(np.broadcast_to(np.asarray(v, dt), (self.batch,)) if np.ndim(v) == 0 else np.asarray(v, dt))
            if a.shape != (self.batch,):
                raise ValueError("expected a scalar or %d values (one per stream), got shape %s" % (self.batch, np.shape(v)))
            out.append(a.ctypes.data_as(ctypes.POINTER(ctypes.c_int if dt == np.int32 else ctypes.c_float)))  # (keeps `a` alive)
        return out

    def setTransposeFactor(self, multiplier, tonalityLimit=0.0):
        a = self._per_stream((multiplier, np.float32), (tonalityLimit, np.float32))
        if a is None:
            self._ck(self._lib.b200s_set_transpose_factor(self._h, multiplier, tonalityLimit))
        else:
            self._ck(self._lib.b200s_set_transpose_factor_per_stream(self._h, a[0], a[1]))

    def setTransposeSemitones(self, semitones, tonalityLimit=0.0):
        a = self._per_stream((semitones, np.float32), (tonalityLimit, np.float32))
        if a is None:
            self._ck(self._lib.b200s_set_transpose_semitones(self._h, semitones, tonalityLimit))
        else:
            self._ck(self._lib.b200s_set_transpose_semitones_per_stream(self._h, a[0], a[1]))

    def setFormantFactor(self, multiplier, compensatePitch=False):
        a = self._per_stream((multiplier, np.float32), (compensatePitch, np.int32))
        if a is None:
            self._ck(self._lib.b200s_set_formant_factor(self._h, multiplier, int(compensatePitch)))
        else:
            self._ck(self._lib.b200s_set_formant_factor_per_stream(self._h, a[0], a[1]))

    def setFormantSemitones(self, semitones, compensatePitch=False):
        a = self._per_stream((semitones, np.float32), (compensatePitch, np.int32))
        if a is None:
            self._ck(self._lib.b200s_set_formant_semitones(self._h, semitones, int(compensatePitch)))
        else:
            self._ck(self._lib.b200s_set_formant_semitones_per_stream(self._h, a[0], a[1]))

    def setFormantBase(self, baseFreq=0.0):
        a = self._per_stream((baseFreq, np.float32))
        if a is None:
            self._ck(self._lib.b200s_set_formant_base(self._h, baseFreq))
        else:
            self._ck(self._lib.b200s_set_formant_base_per_stream(self._h, a[0]))

    @staticmethod
    def _tabulate(fn, points):
        fin = np.linspace(0.0, 0.5, points).astype(np.float32)
        return fin, np.array([fn(float(f)) for f in fin], np.float32)

    def setFreqMap(self, inputToOutput, points=2049, streams=None):
        """setFreqMap(std::function) (:120): the callable is tabulated on [0, 0.5] (piecewise linear).  With `streams`
        (a list of stream indices), or a list of callables (one per listed stream, or per stream of the batch; None = no
        map), the listed streams get their own maps and the others keep theirs."""
        if streams is None and not isinstance(inputToOutput, (list, tuple)):
            if inputToOutput is None:
                self._ck(self._lib.b200s_set_freq_map_table(self._h, None, None, 0))
                return
            self.setFreqMapTable(*self._tabulate(inputToOutput, points))
            return
        fns = inputToOutput if isinstance(inputToOutput, (list, tuple)) else [inputToOutput] * len(streams)
        self.setFreqMapTable([None if f is None else self._tabulate(f, points) for f in fns], streams=streams)

    def setFreqMapTable(self, fin, fout=None, streams=None):
        """The piecewise-linear map itself (b200s_set_freq_map_table): break points fin (ascending) -> fout.  Per stream
        (b200s_set_freq_map_table_per_stream): `streams` lists the streams that get the table (fin, fout), or fin is a
        list of (fin, fout) pairs, one per listed stream (or per stream of the batch when `streams` is None; None = no
        map).  Streams that are not listed keep their maps."""
        fp = ctypes.POINTER(ctypes.c_float)
        if streams is None and fout is not None:
            fin = np.ascontiguousarray(fin, np.float32)
            fout = np.ascontiguousarray(fout, np.float32)
            self._ck(self._lib.b200s_set_freq_map_table(self._h, fin.ctypes.data_as(fp), fout.ctypes.data_as(fp), len(fin)))
            return
        tables = list(fin) if fout is None else [(fin, fout)] * len(streams)
        streams = np.ascontiguousarray(range(self.batch) if streams is None else streams, np.int32)
        if len(tables) != len(streams):
            raise ValueError("%d tables for %d streams" % (len(tables), len(streams)))
        tables = [(np.zeros(0, np.float32),) * 2 if t is None else (np.asarray(t[0], np.float32), np.asarray(t[1], np.float32)) for t in tables]
        for a, b in tables:
            if a.shape != b.shape or a.ndim != 1:
                raise ValueError("freq_in and freq_out must be 1-D and of one length, got %s and %s" % (a.shape, b.shape))
        points = np.array([len(a) for a, _ in tables], np.int32)
        ain = np.ascontiguousarray(np.concatenate([a for a, _ in tables]) if tables else np.zeros(0), np.float32)
        aout = np.ascontiguousarray(np.concatenate([b for _, b in tables]) if tables else np.zeros(0), np.float32)
        ip = ctypes.POINTER(ctypes.c_int)
        self._ck(self._lib.b200s_set_freq_map_table_per_stream(self._h, streams.ctypes.data_as(ip), len(streams), points.ctypes.data_as(ip),
                                                               ain.ctypes.data_as(fp), aout.ctypes.data_as(fp)))

    # ---- the hot path ----
    def _shape(self, n, rows=None):
        c = self.channels()
        if c <= 0:
            raise StretchError("engine not configured: call presetDefault / presetCheaper / configure first")
        return (self.batch if rows is None else rows, c, n)

    def _adopt_torch_stream(self):
        """Device-pointer calls are enqueued on torch's CURRENT stream (b200s_set_stream), so they are ordered after the
        producers of `inputs` and before any torch op on the returned tensor, like a torch op.  (The engine's own side
        streams fork from and join that stream.)"""
        import torch

        st = torch.cuda.current_stream().cuda_stream
        if getattr(self, "_torch_stream", None) != st:
            self._ck(self._lib.b200s_set_stream(self._h, ctypes.c_void_p(st)))
            self._torch_stream = st

    def seek(self, inputs, playbackRate):
        if _is_torch_cuda(inputs):
            self._adopt_torch_stream()
            n = inputs.shape[-1]
            self._ck(self._lib.b200s_seek_device(self._h, inputs.data_ptr(), n, float(playbackRate)))
            return
        x = np.asarray(inputs, np.float32)
        n = x.shape[-1]
        x = _host(x, self._shape(n))
        if np.ndim(playbackRate) > 0:  # one rate per stream (b200s_seek_rates)
            r = np.ascontiguousarray(playbackRate, np.float64)
            if r.shape != (self.batch,):
                raise ValueError("expected %d playback rates" % self.batch)
            self._ck(self._lib.b200s_seek_rates(self._h, x.ctypes.data, n, r.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
            return
        self._ck(self._lib.b200s_seek(self._h, x.ctypes.data, n, float(playbackRate)))

    def live_seek(self, bank_ptr, bank_len, window_end, window, rates):
        """b200s_live_seek: seek windows cut from a device-resident audio bank (pointer), one end index and rate per stream."""
        we = np.ascontiguousarray(window_end, np.int64)
        r = np.ascontiguousarray(rates, np.float64)
        if we.shape != (self.batch,) or r.shape != (self.batch,):
            raise ValueError("expected %d window ends and rates" % self.batch)
        self._ck(self._lib.b200s_live_seek(self._h, ctypes.c_void_p(int(bank_ptr)), int(bank_len), we.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                           int(window), r.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))

    def outputSeek(self, inputs):
        x = np.asarray(inputs, np.float32)
        n = x.shape[-1]
        x = _host(x, self._shape(n))
        self._ck(self._lib.b200s_output_seek(self._h, x.ctypes.data, n))

    def _lengths(self, v, name, rows=None):
        """One sample count per stream (or per entry of a list of `rows` streams) as a contiguous int32 array (a scalar is
        repeated)."""
        rows = self.batch if rows is None else rows
        a = np.asarray(v)
        if a.ndim == 0:
            a = np.full(rows, int(a))
        if a.shape != (rows,):
            raise ValueError("%s: expected a scalar or %d values (one per stream), got shape %s" % (name, rows, np.shape(v)))
        if not np.issubdtype(a.dtype, np.integer):
            raise ValueError("%s: expected integer sample counts, got %s" % (name, a.dtype))
        return np.ascontiguousarray(a, np.int32)

    def process(self, inputs, outputSamples, out=None, inputSamples=None, streams=None):
        """inputs: [batch][channels][inputSamples] (numpy -> host API; torch CUDA tensor -> device API).

        outputSamples: an int, or one per stream; inputSamples: None (every stream reads all of `inputs`' last dimension)
        or one per stream.  With any per-stream array, stream s reads the first inputSamples[s] samples of its rows and
        writes the first outputSamples[s] of an output of max(outputSamples) samples per row, zeros after them
        (b200s_process_per_stream).  streams: only these streams process, as in run()."""
        if np.ndim(outputSamples) > 0 or inputSamples is not None or streams is not None:
            return self.run(self.OP_PROCESS, inputs, outputSamples, inputSamples=inputSamples, out=out, streams=streams)
        if _is_torch_cuda(inputs):
            import torch

            self._adopt_torch_stream()
            n_in = inputs.shape[-1]
            assert inputs.is_contiguous() and inputs.dtype == torch.float32
            if out is None:
                out = torch.empty(self._shape(outputSamples), dtype=torch.float32, device=inputs.device)
            self._ck(self._lib.b200s_process_device(self._h, inputs.data_ptr(), n_in, out.data_ptr(), outputSamples))
            return out
        x = np.asarray(inputs, np.float32)
        n_in = x.shape[-1]
        x = _host(x, self._shape(n_in))
        if out is None:
            out = np.empty(self._shape(max(outputSamples, 0)), np.float32)
        self._ck(self._lib.b200s_process(self._h, x.ctypes.data, n_in, out.ctypes.data, outputSamples))
        return out

    def _run_args(self, ops, in_stride, outputSamples, inputSamples, playbackRates, out, streams):
        """The checked arguments of run() / run_pcm16(): (rows, list or None, ops, n_in, n_out, rates or None, out_stride)."""
        lst = None if streams is None else self._stream_list(streams, "streams")
        rows = self.batch if lst is None else int(lst.size)
        op = self._lengths(ops, "ops", rows)
        if np.any((op < 0) | (op > 5)):
            raise ValueError("ops: every op must be one of OP_SKIP .. OP_RESET")
        n_out = self._lengths(outputSamples, "outputSamples", rows)
        if inputSamples is None:
            reads = (op == self.OP_PROCESS) | (op == self.OP_SEEK) | (op == self.OP_OUTPUT_SEEK)
            inputSamples = np.where(reads, in_stride, 0)
        n_in = self._lengths(inputSamples, "inputSamples", rows)
        rates = None
        if playbackRates is not None:
            rates = np.ascontiguousarray(np.broadcast_to(np.asarray(playbackRates, np.float64), (rows,)) if np.ndim(playbackRates) == 0
                                         else np.asarray(playbackRates, np.float64))
            if rates.shape != (rows,):
                raise ValueError("playbackRates: expected a scalar or %d values, got shape %s" % (rows, np.shape(playbackRates)))
        out_stride = int(n_out.max()) if rows else 0
        if out is not None:
            out_stride = int(out.shape[-1])
            if tuple(out.shape) != self._shape(out_stride, rows):
                raise ValueError("out: expected shape %s, got %s" % (self._shape(out_stride, rows), tuple(out.shape)))
        for name, a, stride in (("inputSamples", n_in, in_stride), ("outputSamples", n_out, out_stride)):
            bad = np.flatnonzero((a < 0) | (a > stride))
            if bad.size:
                raise ValueError("%s[%d] = %d is outside [0, %d]" % (name, bad[0], a[bad[0]], stride))
        return rows, lst, op, n_in, n_out, rates, out_stride

    def _run_call(self, fn_all, fn_list, lst, op, in_ptr, in_stride, n_in, out_ptr, out_stride, n_out, rates, *extra):
        ip, dp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)
        rp = None if rates is None else rates.ctypes.data_as(dp)
        args = (op.ctypes.data_as(ip), in_ptr, in_stride, n_in.ctypes.data_as(ip), out_ptr, out_stride, n_out.ctypes.data_as(ip), rp) + extra
        self._ck(fn_all(self._h, *args) if lst is None else fn_list(self._h, int(lst.size), lst.ctypes.data_as(ip), *args))

    def run(self, ops, inputs, outputSamples, inputSamples=None, playbackRates=None, out=None, streams=None):
        """Every stream runs its own operation (b200s_run_per_stream): ops, outputSamples, inputSamples and playbackRates are
        scalars (repeated for every stream) or one value per stream.  OP_PROCESS: process(inputs[s][:, :inputSamples[s]],
        outputSamples[s]); OP_SEEK: seek(inputs[s][:, :inputSamples[s]], playbackRates[s]); OP_OUTPUT_SEEK:
        outputSeek(inputs[s][:, :inputSamples[s]]); OP_FLUSH: flush(outputSamples[s], playbackRates[s]); OP_RESET: reset();
        OP_SKIP: nothing.  inputs: [batch][channels][stride] (numpy -> host API; torch CUDA tensor -> device API; None
        when no stream reads input); inputSamples defaults to the whole stride for the ops that read input and 0 for the
        others.  Returns [batch][channels][max(outputSamples)] (or `out`), zeros after each stream's own output.

        streams: a list of n slots (b200s_run_streams).  Only they run; every array then has one value per list entry and
        the buffers are [n][channels][stride], row i for stream streams[i].  The other streams are not touched."""
        torch_in = _is_torch_cuda(inputs)
        in_stride = 0 if inputs is None else int(inputs.shape[-1]) if torch_in else int(np.shape(inputs)[-1])
        rows, lst, op, n_in, n_out, rates, out_stride = self._run_args(ops, in_stride, outputSamples, inputSamples, playbackRates, out, streams)

        def call(fn_all, fn_list, in_ptr, out_ptr):
            self._run_call(fn_all, fn_list, lst, op, in_ptr, in_stride, n_in, out_ptr, out_stride, n_out, rates)

        if torch_in:
            import torch

            self._adopt_torch_stream()
            assert inputs.is_contiguous() and inputs.dtype == torch.float32
            if tuple(inputs.shape) != self._shape(in_stride, rows):
                raise ValueError("inputs: expected shape %s, got %s" % (self._shape(in_stride, rows), tuple(inputs.shape)))
            if out is None:
                out = torch.empty(self._shape(out_stride, rows), dtype=torch.float32, device=inputs.device)
            call(self._lib.b200s_run_per_stream_device, self._lib.b200s_run_streams_device, inputs.data_ptr(), out.data_ptr())
            return out
        x = None
        if inputs is not None:
            x = np.asarray(inputs, np.float32)
            if x.shape != self._shape(in_stride, rows):
                raise ValueError("inputs: expected shape %s, got %s" % (self._shape(in_stride, rows), x.shape))
            x = _host(x, self._shape(in_stride, rows))
        if out is None:
            out = np.empty(self._shape(out_stride, rows), np.float32)
        call(self._lib.b200s_run_per_stream, self._lib.b200s_run_streams, None if x is None else x.ctypes.data, out.ctypes.data)
        return out

    def run_pcm16(self, ops, inputs, outputSamples, inputSamples=None, playbackRates=None, out=None, streams=None):
        """run() with 16-bit PCM host buffers (b200s_run_per_stream_pcm16 / b200s_run_streams_pcm16): inputs is an int16
        array [rows][channels][stride] (or None), the result an int16 array [rows][channels][out_stride] (or `out`).  The
        output equals run() fed inputs / 32768, rounded to nearest (halves away from zero) and clamped to int16; both
        conversions run on the device.  There is no device-buffer form: a torch CUDA tensor raises TypeError."""
        if _is_torch_cuda(inputs) or _is_torch_cuda(out):
            raise TypeError("run_pcm16: 16-bit PCM is a host-buffer format; pass float32 CUDA tensors to run()")
        in_stride = 0 if inputs is None else int(np.shape(inputs)[-1])
        rows, lst, op, n_in, n_out, rates, out_stride = self._run_args(ops, in_stride, outputSamples, inputSamples, playbackRates, out, streams)
        x = None
        if inputs is not None:
            x = np.asarray(inputs)
            if x.dtype != np.int16:
                raise ValueError("inputs: expected int16 samples, got %s" % x.dtype)
            if x.shape != self._shape(in_stride, rows):
                raise ValueError("inputs: expected shape %s, got %s" % (self._shape(in_stride, rows), x.shape))
            x = np.ascontiguousarray(x)
        if out is None:
            out = np.empty(self._shape(out_stride, rows), np.int16)
        elif not (isinstance(out, np.ndarray) and out.dtype == np.int16 and out.flags.c_contiguous):
            raise ValueError("out: expected a contiguous int16 numpy array")
        self._run_call(self._lib.b200s_run_per_stream_pcm16, self._lib.b200s_run_streams_pcm16, lst, op, None if x is None else x.ctypes.data,
                       in_stride, n_in, out.ctypes.data, out_stride, n_out, rates, 1)
        return out

    def process_per_stream_host_ptr(self, in_ptr, in_stride, n_in, out_ptr, out_stride, n_out, wait=False):
        """Raw host pointers (pinned buffers [batch][channels][stride]) with per-stream counts n_in / n_out (`batch` ints
        each): b200s_process_per_stream, or b200s_process_per_stream_async unless `wait` (the buffers then belong to the
        engine until synchronize(); the counts are copied during the call)."""
        ip = ctypes.POINTER(ctypes.c_int)
        a, b = self._lengths(n_in, "n_in"), self._lengths(n_out, "n_out")
        fn = self._lib.b200s_process_per_stream if wait else self._lib.b200s_process_per_stream_async
        self._ck(fn(self._h, in_ptr, int(in_stride), a.ctypes.data_as(ip), out_ptr, int(out_stride), b.ctypes.data_as(ip)))

    def run_per_stream_host_ptr(self, ops, in_ptr, in_stride, n_in, out_ptr, out_stride, n_out, playback_rates=None, wait=False):
        """Raw host pointers (pinned buffers [batch][channels][stride]) with per-stream ops and counts (`batch` values each):
        b200s_run_per_stream, or b200s_run_per_stream_async unless `wait` (the buffers then belong to the engine until
        synchronize(); ops, counts and rates are copied during the call)."""
        ip = ctypes.POINTER(ctypes.c_int)
        o, a, b = self._lengths(ops, "ops"), self._lengths(n_in, "n_in"), self._lengths(n_out, "n_out")
        r = None if playback_rates is None else np.ascontiguousarray(np.broadcast_to(np.asarray(playback_rates, np.float64), (self.batch,)))
        rp = None if r is None else r.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        fn = self._lib.b200s_run_per_stream if wait else self._lib.b200s_run_per_stream_async
        self._ck(fn(self._h, o.ctypes.data_as(ip), in_ptr, int(in_stride), a.ctypes.data_as(ip), out_ptr, int(out_stride), b.ctypes.data_as(ip), rp))

    def run_streams_host_ptr(self, streams, ops, in_ptr, in_stride, n_in, out_ptr, out_stride, n_out, playback_rates=None, wait=False):
        """run_per_stream_host_ptr over a list of streams (b200s_run_streams / _async): pinned buffers [n][channels][stride],
        row i and the i-th value of ops, counts and rates for stream streams[i]."""
        ip = ctypes.POINTER(ctypes.c_int)
        lst = self._stream_list(streams, "streams")
        n = int(lst.size)
        o, a, b = self._lengths(ops, "ops", n), self._lengths(n_in, "n_in", n), self._lengths(n_out, "n_out", n)
        r = None if playback_rates is None else np.ascontiguousarray(np.broadcast_to(np.asarray(playback_rates, np.float64), (n,)))
        rp = None if r is None else r.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        fn = self._lib.b200s_run_streams if wait else self._lib.b200s_run_streams_async
        self._ck(fn(self._h, n, lst.ctypes.data_as(ip), o.ctypes.data_as(ip), in_ptr, int(in_stride), a.ctypes.data_as(ip), out_ptr,
                    int(out_stride), b.ctypes.data_as(ip), rp))

    def run_pcm16_host_ptr(self, ops, in_ptr, in_stride, n_in, out_ptr, out_stride, n_out, playback_rates=None, streams=None, wait=False):
        """Raw host pointers to pinned int16 buffers [rows][channels][stride]: b200s_run_per_stream_pcm16, or with `streams`
        b200s_run_streams_pcm16 (rows = len(streams)).  Unless `wait` the call returns once enqueued and the buffers belong
        to the engine until synchronize(); ops, counts and rates are copied during the call."""
        lst = None if streams is None else self._stream_list(streams, "streams")
        rows = self.batch if lst is None else int(lst.size)
        o, a, b = self._lengths(ops, "ops", rows), self._lengths(n_in, "n_in", rows), self._lengths(n_out, "n_out", rows)
        r = None if playback_rates is None else np.ascontiguousarray(np.broadcast_to(np.asarray(playback_rates, np.float64), (rows,)))
        self._run_call(self._lib.b200s_run_per_stream_pcm16, self._lib.b200s_run_streams_pcm16, lst, o, in_ptr, int(in_stride), a, out_ptr,
                       int(out_stride), b, r, 1 if wait else 0)

    def process_host_ptr(self, in_ptr, n_in, out_ptr, n_out):
        """Raw host pointers (e.g. pinned torch tensors): the end-to-end call bench.py times."""
        self._ck(self._lib.b200s_process(self._h, in_ptr, n_in, out_ptr, n_out))

    def process_host_ptr_async(self, in_ptr, n_in, out_ptr, n_out):
        """b200s_process_async: enqueue and return; buffers (pinned) belong to the engine until synchronize()."""
        self._ck(self._lib.b200s_process_async(self._h, in_ptr, n_in, out_ptr, n_out))

    def process_pcm16(self, inputs, outputSamples):
        """16-bit PCM in / out (int16 arrays [batch][channels][n]); conversion on the device."""
        x = np.ascontiguousarray(inputs, dtype=np.int16)
        n_in = x.shape[-1]
        out = np.empty(self._shape(max(outputSamples, 0)), np.int16)
        self._ck(self._lib.b200s_process_pcm16(self._h, x.ctypes.data, n_in, out.ctypes.data, outputSamples, 1))
        return out

    def process_pcm16_ptr(self, in_ptr, n_in, out_ptr, n_out, wait=False):
        self._ck(self._lib.b200s_process_pcm16(self._h, in_ptr, n_in, out_ptr, n_out, 1 if wait else 0))

    def flush(self, outputSamples, playbackRate=0.0):
        out = np.empty(self._shape(max(outputSamples, 0)), np.float32)
        self._ck(self._lib.b200s_flush(self._h, out.ctypes.data, outputSamples, playbackRate))
        return out

    def exact(self, inputs, outputSamples):
        x = np.asarray(inputs, np.float32)
        n_in = x.shape[-1]
        x = _host(x, self._shape(n_in))
        out = np.empty(self._shape(outputSamples), np.float32)
        ok = ctypes.c_int(0)
        self._ck(self._lib.b200s_exact(self._h, x.ctypes.data, n_in, out.ctypes.data, outputSamples, ctypes.byref(ok)))
        return bool(ok.value), out

    # ---- moving, duplicating and saving single streams (b200s_copy_streams / _export_streams / _import_streams / _clone) ----
    def _stream_list(self, streams, name):
        a = np.ascontiguousarray(np.atleast_1d(np.asarray(streams)))
        if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError("%s: expected a list of stream indices, got %s" % (name, np.shape(streams)))
        return np.ascontiguousarray(a, np.int32)

    def state_bytes(self):
        """Bytes of one stream's state record."""
        n = self._lib.b200s_stream_state_bytes(self._h)
        self._ck(min(n, 0))
        return n

    def copy_streams(self, dst_streams, src_streams, src=None):
        """Stream dst_streams[i] of this engine becomes a copy of stream src_streams[i] of `src` (default: this engine), as
        the reference's copy assignment would make it.  Asynchronous on both engines' streams; swaps and forks work."""
        src = self if src is None else src
        if src._lib is not self._lib:
            raise ValueError("copy_streams: both engines must come from the same library")
        d, s = self._stream_list(dst_streams, "dst_streams"), self._stream_list(src_streams, "src_streams")
        if d.size != s.size:
            raise ValueError("copy_streams: %d destinations for %d sources" % (d.size, s.size))
        ip = ctypes.POINTER(ctypes.c_int)
        self._ck(self._lib.b200s_copy_streams(self._h, d.ctypes.data_as(ip), src._h, s.ctypes.data_as(ip), int(d.size)))

    def export_streams(self, streams):
        """The listed streams' state records: uint8 [n, state_bytes()]."""
        s = self._stream_list(streams, "streams")
        out = np.empty((s.size, self.state_bytes()), np.uint8)
        self._ck(self._lib.b200s_export_streams(self._h, s.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), int(s.size), out.ctypes.data))
        return out

    def import_streams(self, streams, records):
        """Load records of export_streams() (this configuration) into the listed slots."""
        s = self._stream_list(streams, "streams")
        r = np.ascontiguousarray(records, np.uint8)
        if r.shape != (s.size, self.state_bytes()):
            raise ValueError("import_streams: expected records of shape %s, got %s" % ((s.size, self.state_bytes()), r.shape))
        self._ck(self._lib.b200s_import_streams(self._h, s.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), int(s.size), r.ctypes.data))

    def clone(self):
        """A new engine with this one's batch, device, seed, configuration, tuning, parameters and state of every stream."""
        h = ctypes.c_void_p()
        self._ck(self._lib.b200s_clone(self._h, ctypes.byref(h)))
        c = BatchStretch.__new__(BatchStretch)
        c._lib, c._h, c.batch = self._lib, h, self.batch
        return c

    # ---- plumbing ----
    def set_stream(self, cuda_stream):
        self._ck(self._lib.b200s_set_stream(self._h, ctypes.c_void_p(int(cuda_stream))))

    def set_tuning(self, key, value):
        """Implementation selectors (include/b200_stretch.h): 0 chain kernel generation, 1 scalar FFT kernels, 2 host pipeline groups."""
        self._ck(self._lib.b200s_set_tuning(self._h, int(key), int(value)))

    def set_sub_batches(self, n):
        self._ck(self._lib.b200s_set_sub_batches(self._h, n))

    def synchronize(self):
        self._ck(self._lib.b200s_synchronize(self._h))

    def timer_start(self):
        self._ck(self._lib.b200s_timer_start(self._h))

    def timer_stop(self):
        ms = ctypes.c_float(0)
        self._ck(self._lib.b200s_timer_stop(self._h, ctypes.byref(ms)))
        return ms.value

    def kernel_launches(self):
        return int(self._lib.b200s_kernel_launches(self._h))

    def unserved_random_blocks(self):
        return int(self._lib.b200s_unserved_random_blocks(self._h))

    def device_allocations(self):
        return int(self._lib.b200s_device_allocations(self._h))

    KERNELS = ("plan", "analyse", "prep", "chain", "synth", "commit")

    def profile_begin(self):
        self._ck(self._lib.b200s_profile_begin(self._h))

    def profile_end(self, phases=False):
        """{kernel: (total ms, launches)} for the process() calls since profile_begin(); phases=True adds "phases", the pre
        and post phases of run()."""
        names = self.KERNELS + (("phases",) if phases else ())
        ms = (ctypes.c_float * len(names))()
        cnt = (ctypes.c_int * len(names))()
        self._ck(self._lib.b200s_profile_end(self._h, ms, cnt, len(names)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(names)}

    def selftest_divsqrt(self, n=1 << 27, seed=1):
        a, b = ctypes.c_longlong(0), ctypes.c_longlong(0)
        self._ck(self._lib.b200s_selftest_divsqrt(self._h, n, seed, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def get_state(self, name):
        what = STATE[name]
        n = self._lib.b200s_state_size(self._h, what)
        buf = np.empty((self.batch, n), np.float32)
        self._ck(self._lib.b200s_get_state(self._h, what, buf.ctypes.data))
        C, K = self.channels(), self.bands()
        if name in ("input", "prevInput", "output"):
            return buf.view(np.complex64).reshape(self.batch, C, K)
        return buf.reshape(self.batch, C, -1)

    def set_state(self, name, value):
        what = STATE[name]
        n = self._lib.b200s_state_size(self._h, what)
        v = np.ascontiguousarray(value)
        if v.dtype == np.complex64:
            v = v.view(np.float32)
        v = np.ascontiguousarray(v, np.float32).reshape(self.batch, n)
        self._ck(self._lib.b200s_set_state(self._h, what, v.ctypes.data))
