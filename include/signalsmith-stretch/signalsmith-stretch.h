// include/signalsmith-stretch/signalsmith-stretch.h -- drop-in C++ facade over the GPU C ABI.
//
// Same include path (`#include "signalsmith-stretch/signalsmith-stretch.h"`, as cmd/main.cpp:5 of
// the reference does), same namespace, class name, template parameters, method names, argument
// order and defaults as /root/reference/signalsmith-stretch.h:34-491, so host code written
// against the reference compiles unchanged and runs its STFT phase-vocoder hot path on an H100:
//
//     signalsmith::stretch::SignalsmithStretch<float> stretch;
//     stretch.presetDefault(channels, sampleRate);
//     stretch.setTransposeSemitones(7, 8000 / sampleRate);
//     stretch.process(inputBuffers, inputSamples, outputBuffers, outputSamples);
//
// `Inputs` / `Outputs` are any type with `buf[channel][index]` (float**, std::vector<float*>,
// the reference's Wav proxy of doubles, ... README.md:46); like the reference's copyInput()
// (:220-226) the facade marshals element by element into planar float staging, then calls
// b200s_process().  One object = a batch of one stream; use the C ABI (or `BatchStretch` below)
// for batches.  Only Sample = float is GPU-backed.  Methods stay `void` (the reference has no error path at all), so a
// failure -- no usable GPU, an unsupported configuration, a CUDA error -- cannot be returned: it is FATAL.  The message
// goes to stderr and the process aborts, because host code written against the reference has no reason to poll an error
// flag and would otherwise write silence.  Define B200S_FACADE_SOFT_ERRORS before including this header to get the
// sticky lastError() string instead (outputs are then zero-filled on failure).  No CPU fallback.
#ifndef SIGNALSMITH_STRETCH_H
#define SIGNALSMITH_STRETCH_H

#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../b200_stretch.h"

namespace signalsmith { namespace stretch {

template <typename Sample = float, class RandomEngine = void>
struct SignalsmithStretch {
	static_assert(std::is_same<Sample, float>::value, "the GPU path computes in float (Sample = float)");
	static constexpr size_t version[3] = {1, 3, 2}; // reference :36

	SignalsmithStretch() : SignalsmithStretch(0) {}
	SignalsmithStretch(long seed) { check(b200s_create(1, seed, 0, &engine)); } // :38-39
	~SignalsmithStretch() { b200s_destroy(engine); }
	// Copyable and movable like the reference class (whose members the compiler copies): a copy continues exactly where
	// the original is -- parameters, state and random engine (b200s_clone).  A moved-from object holds no engine.
	SignalsmithStretch(const SignalsmithStretch &other) : channels(other.channels) {
		if (other.engine) check(b200s_clone(other.engine, &engine));
	}
	SignalsmithStretch &operator=(const SignalsmithStretch &other) {
		if (this != &other) {
			SignalsmithStretch copy(other);
			swap(copy);
		}
		return *this;
	}
	SignalsmithStretch(SignalsmithStretch &&other) noexcept { swap(other); }
	SignalsmithStretch &operator=(SignalsmithStretch &&other) noexcept {
		if (this != &other) {
			SignalsmithStretch gone(std::move(*this));
			swap(other);
		}
		return *this;
	}

	int inputLatency() const { return b200s_input_latency(engine); }   // :42
	int outputLatency() const { return b200s_output_latency(engine); } // :45
	void reset() { check(b200s_reset(engine)); }                       // :49

	void presetDefault(int nChannels, Sample sampleRate, bool splitComputation = false) { // :63
		check(b200s_preset_default(engine, nChannels, sampleRate, splitComputation));
		channels = nChannels;
	}
	void presetCheaper(int nChannels, Sample sampleRate, bool splitComputation = true) { // :66
		check(b200s_preset_cheaper(engine, nChannels, sampleRate, splitComputation));
		channels = nChannels;
	}
	void configure(int nChannels, int blockSamples, int intervalSamples, bool splitComputation = false) { // :71
		check(b200s_configure(engine, nChannels, blockSamples, intervalSamples, splitComputation));
		channels = nChannels;
	}
	int blockSamples() const { return b200s_block_samples(engine); }         // :96
	int intervalSamples() const { return b200s_interval_samples(engine); }   // :99
	bool splitComputation() const { return b200s_split_computation(engine); } // :102

	void setTransposeFactor(Sample multiplier, Sample tonalityLimit = 0) { check(b200s_set_transpose_factor(engine, multiplier, tonalityLimit)); }   // :107
	void setTransposeSemitones(Sample semitones, Sample tonalityLimit = 0) { check(b200s_set_transpose_semitones(engine, semitones, tonalityLimit)); } // :116
	// :120 -- a std::function cannot run on the device: it is tabulated on [0, 0.5] (2049 points,
	// piecewise linear), which is exact for the piecewise-linear maps the reference itself uses.
	void setFreqMap(std::function<Sample(Sample)> inputToOutput) {
		if (!inputToOutput) {
			check(b200s_set_freq_map_table(engine, nullptr, nullptr, 0));
			return;
		}
		const int n = 2049;
		std::vector<float> fin(n), fout(n);
		for (int i = 0; i < n; ++i) {
			fin[i] = 0.5f * float(i) / float(n - 1);
			fout[i] = inputToOutput(fin[i]);
		}
		check(b200s_set_freq_map_table(engine, fin.data(), fout.data(), n));
	}
	void setFormantFactor(Sample multiplier, bool compensatePitch = false) { check(b200s_set_formant_factor(engine, multiplier, compensatePitch)); }   // :124
	void setFormantSemitones(Sample semitones, bool compensatePitch = false) { check(b200s_set_formant_semitones(engine, semitones, compensatePitch)); } // :129
	void setFormantBase(Sample baseFreq = 0) { check(b200s_set_formant_base(engine, baseFreq)); }                                                         // :133

	template <class Inputs>
	void seek(Inputs &&inputs, int inputSamples, double playbackRate) { // :139
		gather(inputs, 0, inputSamples);
		check(b200s_seek(engine, stageIn.data(), inputSamples, playbackRate));
	}
	int seekLength() const { return b200s_seek_length(engine); } // :166

	template <class Inputs>
	void outputSeek(Inputs &&inputs, int inputLength) { // :172
		gather(inputs, 0, inputLength);
		check(b200s_output_seek(engine, stageIn.data(), inputLength));
	}
	int outputSeekLength(Sample playbackRate) const { return b200s_output_seek_length(engine, playbackRate); } // :205

	template <class Inputs, class Outputs>
	void process(Inputs &&inputs, int inputSamples, Outputs &&outputs, int outputSamples) { // :209
		gather(inputs, 0, inputSamples);
		stageOut.resize(size_t(channels) * size_t(outputSamples > 0 ? outputSamples : 1));
		check(b200s_process(engine, stageIn.data(), inputSamples, stageOut.data(), outputSamples));
		scatter(outputs, outputSamples);
	}

	template <class Outputs>
	void flush(Outputs &&outputs, int outputSamples, Sample playbackRate = 0) { // :426
		stageOut.resize(size_t(channels) * size_t(outputSamples > 0 ? outputSamples : 1));
		check(b200s_flush(engine, stageOut.data(), outputSamples, playbackRate));
		scatter(outputs, outputSamples);
	}

	template <class Inputs, class Outputs>
	bool exact(Inputs &&inputs, int inputSamples, Outputs &&outputs, int outputSamples) { // :467
		gather(inputs, 0, inputSamples);
		stageOut.resize(size_t(channels) * size_t(outputSamples > 0 ? outputSamples : 1));
		int ok = 0;
		check(b200s_exact(engine, stageIn.data(), inputSamples, stageOut.data(), outputSamples, &ok));
		scatter(outputs, outputSamples);
		return ok != 0;
	}

	// not in the reference: text of the last CUDA / argument error ("" if none)
	const std::string &lastError() const { return error; }

private:
	b200s_engine *engine = nullptr;
	int channels = 0;
	std::vector<float> stageIn, stageOut;
	std::string error;

	bool failed = false; // soft-error mode: the last call failed, scatter() writes zeros
	void swap(SignalsmithStretch &other) noexcept {
		std::swap(engine, other.engine);
		std::swap(channels, other.channels);
		stageIn.swap(other.stageIn);
		stageOut.swap(other.stageOut);
		error.swap(other.error);
		std::swap(failed, other.failed);
	}
	void check(int rc) {
		failed = rc != 0;
		if (!failed) return;
		error = engine ? b200s_last_error(engine) : b200s_last_error(nullptr);
#ifndef B200S_FACADE_SOFT_ERRORS
		std::fprintf(stderr, "signalsmith-stretch (GPU): fatal: %s (code %d)\n", error.c_str(), rc);
		std::abort();
#endif
	}
	template <class Inputs>
	void gather(Inputs &&inputs, int offset, int n) {
		stageIn.resize(size_t(channels) * size_t(n > 0 ? n : 1));
		for (int c = 0; c < channels; ++c) {
			auto &&channel = inputs[c];
			for (int i = 0; i < n; ++i) stageIn[size_t(c) * n + i] = float(channel[i + offset]);
		}
	}
	template <class Outputs>
	void scatter(Outputs &&outputs, int n) {
		for (int c = 0; c < channels; ++c) {
			auto &&channel = outputs[c];
			for (int i = 0; i < n; ++i) channel[i] = failed ? 0.f : stageOut[size_t(c) * n + i];
		}
	}
};

}} // namespace signalsmith::stretch
#endif
