// Polyphase resampling, scipy.signal.resample_poly(x, up, down) with its default Kaiser (beta 5) filter.  include/b200tts.h states the
// contract; tests/resample_oracle.py restates it in numpy.
//
// Packed ragged layout as wsola.cu: utterance b owns input samples [soff[b], soff[b+1]) and output samples [ooff[b], ooff[b+1]); its plan
// row names its ratio and where its polyphase table starts in the packed taps.  One thread per output sample reads its phase's taps, which
// are contiguous, through the read-only path: a table is up to 2048 x 21 doubles (336 KB at 2048/1), more than one CTA's shared memory,
// and a batch may mix ratios, while the tables in use stay resident in L2 and the ones of common ratios (50 to 75 KB) in L1.  Nothing
// uses atomics and every sum runs in a fixed order, so a batch computes exactly what its members compute one at a time.
#include <limits.h>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int RESAMPLE_THREADS = 256;        // one thread per output sample

// The index is formed in 64 bits, and so are n down and h_len + n down: a 35-minute recording at 16 kHz already has n down above 2^31
__global__ void __launch_bounds__(RESAMPLE_THREADS) resample_kernel(b200tts_resample_shape s, const float* __restrict__ wave,
                                                                    const int* __restrict__ soff, const int* __restrict__ ooff,
                                                                    const int4* __restrict__ plan, const double* __restrict__ taps,
                                                                    float* __restrict__ out) {
    const long long gl = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gl >= s.total_out_samples) return;
    const int g = (int)gl;
    const int b = utterance_of(ooff, s.B, g);
    const int4 p = plan[b];                      // up, down, h_len, table offset
    const int up = p.x, hl = p.z;
    const int s0 = soff[b], L = soff[b + 1] - s0;
    const long long t = hl + (long long)(g - ooff[b]) * p.y;
    const long long k0 = t / up;
    const int phase = (int)(t - k0 * up);
    const int T = (2 * hl + up) / up;            // ceil((2 h_len + 1) / up)
    // taps i of this phase with phase + i up <= 2 h_len, and inputs k0 - i inside [0, L)
    const long long i1 = min((long long)((2 * hl - phase) / up + 1), k0 + 1);
    const long long i0 = min(max(0LL, k0 - (L - 1)), i1);
    const double* h = taps + p.w + (long long)phase * T;
    const float* x = wave + s0 + k0;
    double y = 0.0;
#pragma unroll 4
    for (int i = (int)i0; i < (int)i1; ++i) y = fma((double)__ldg(x - i), __ldg(h + i), y);
    out[g] = (float)y;
}

}  // namespace

}  // namespace b200tts
using namespace b200tts;

extern "C" {

int b200tts_resample(const b200tts_resample_shape* shape, const float* wave, const int32_t* soff, const int32_t* ooff, const int32_t* plan,
                     const double* taps, float* out, void* stream) {
    B200_REQUIRE(shape && wave && soff && ooff && plan && taps && out, "resample: null argument");
    const b200tts_resample_shape& s = *shape;
    B200_REQUIRE(s.B >= 1 && s.total_samples >= s.B && s.total_out_samples >= s.B && s.total_taps >= 1,
                 "resample: need B >= 1, at least one input and one output sample per utterance and a table (B = %d, total_samples = %d, "
                 "total_out_samples = %d, total_taps = %d)", s.B, s.total_samples, s.total_out_samples, s.total_taps);
    B200_REQUIRE(s.max_factor >= 1 && s.max_factor <= B200TTS_RESAMPLE_MAX_FACTOR, "resample: max_factor %d must be in [1, %d]",
                 s.max_factor, B200TTS_RESAMPLE_MAX_FACTOR);
    B200_REQUIRE((const void*)out != (const void*)wave && (const void*)out != (const void*)taps,
                 "resample: out must not alias wave or taps");
    B200_REQUIRE(((uintptr_t)plan & 15) == 0, "resample: plan must be 16-byte aligned");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("resample", st);
    resample_kernel<<<cdiv(s.total_out_samples, RESAMPLE_THREADS), RESAMPLE_THREADS, 0, st>>>(
        s, wave, soff, ooff, reinterpret_cast<const int4*>(plan), taps, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
