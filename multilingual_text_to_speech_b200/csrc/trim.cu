// Silence trimming, librosa 0.7.0 effects.trim: frame powers of the reflect-padded signal, then the first and last frame within top_db of
// the loudest.  include/b200tts.h states the contract; tests/resample_oracle.py restates it in numpy.
//
// Packed ragged layout: utterance b owns samples [soff[b], soff[b+1]) and frames [foff[b], foff[b+1]).  One warp per frame sums its W
// squares (a lane takes every 32nd sample, then a fixed shuffle tree); one CTA per utterance reduces the maximum and the two bounds.
// Nothing uses atomics, so a batch computes exactly what its members compute one at a time.
#include <limits.h>
#include <math.h>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int POWER_WARPS = 8;               // frames per CTA of the power kernel
constexpr int BOUNDS_THREADS = 256;          // one CTA per utterance
constexpr double AMIN = 1e-10;               // power_to_db's amin

__global__ void __launch_bounds__(POWER_WARPS * 32) trim_power_kernel(b200tts_trim_shape s, const float* __restrict__ wave,
                                                                      const int* __restrict__ soff, const int* __restrict__ foff,
                                                                      double* __restrict__ power) {
    const int gf = blockIdx.x * POWER_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (gf >= s.total_frames) return;
    const int b = utterance_of(foff, s.B, gf);
    const int s0 = soff[b], L = soff[b + 1] - s0, W = s.frame_length;
    // padded index f hop as a signal index; the padded indices of the frames lie in [-W / 2, L - 1 + W / 2]
    const long long start = (long long)(gf - foff[b]) * s.hop - W / 2;
    const bool one_reflection = L - 1 >= W / 2;  // else L <= W / 2 + 1, and every index fits reflect_index's int arithmetic
    const float* x = wave + s0;
    double acc = 0.0;
    for (int j = lane; j < W; j += 32) {
        const long long v = start + j;
        const int k = v >= 0 && v < L ? (int)v
                      : one_reflection ? (int)(v < 0 ? -v : 2LL * (L - 1) - v)
                                       : reflect_index((int)v, L);
        const double xv = (double)x[k];
        acc = fma(xv, xv, acc);
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sh);
    if (lane == 0) power[gf] = acc / W;
}

template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* red) {
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, sh));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < BOUNDS_THREADS / 32; ++w) v = op(v, red[w]);
    __syncthreads();
    return v;
}

__global__ void __launch_bounds__(BOUNDS_THREADS) trim_bounds_kernel(b200tts_trim_shape s, const int* __restrict__ soff,
                                                                     const int* __restrict__ foff, const double* __restrict__ power,
                                                                     int* __restrict__ bounds) {
    __shared__ double red_p[BOUNDS_THREADS / 32];
    __shared__ int red_i[BOUNDS_THREADS / 32];
    const int b = blockIdx.x, f0 = foff[b], F = foff[b + 1] - f0, L = soff[b + 1] - soff[b];
    const double* p = power + f0;
    double mx = 0.0;                             // powers are >= 0
    for (int f = threadIdx.x; f < F; f += BOUNDS_THREADS) mx = fmax(mx, p[f]);
    mx = block_reduce(mx, [](double a, double c) { return fmax(a, c); }, red_p);
    const double ref_db = 10.0 * log10(fmax(AMIN, mx));
    int first = INT_MAX, last = -1;
    for (int f = threadIdx.x; f < F; f += BOUNDS_THREADS) {
        if (10.0 * log10(fmax(AMIN, p[f])) - ref_db > -s.top_db) {
            first = min(first, f);
            last = max(last, f);
        }
    }
    first = block_reduce(first, [](int a, int c) { return min(a, c); }, red_i);
    last = block_reduce(last, [](int a, int c) { return max(a, c); }, red_i);
    if (threadIdx.x == 0) {
        const bool any = last >= 0;
        bounds[2 * b] = any ? (int)min((long long)first * s.hop, (long long)L) : 0;
        bounds[2 * b + 1] = any ? (int)min((long long)(last + 1) * s.hop, (long long)L) : 0;
    }
}

}  // namespace

}  // namespace b200tts
using namespace b200tts;

extern "C" {

int b200tts_trim_silence(const b200tts_trim_shape* shape, const float* wave, const int32_t* soff, const int32_t* foff, double* power,
                         int32_t* bounds, void* stream) {
    B200_REQUIRE(shape && wave && soff && foff && power && bounds, "trim_silence: null argument");
    const b200tts_trim_shape& s = *shape;
    B200_REQUIRE(s.B >= 1 && s.total_samples >= s.B && s.total_frames >= s.B,
                 "trim_silence: need B >= 1 and at least one sample and one frame per utterance (B = %d, total_samples = %d, "
                 "total_frames = %d)", s.B, s.total_samples, s.total_frames);
    B200_REQUIRE(s.frame_length >= 1 && s.hop >= 1, "trim_silence: frame_length %d and hop %d must be at least 1", s.frame_length, s.hop);
    B200_REQUIRE(isfinite(s.top_db), "trim_silence: top_db must be finite");
    B200_REQUIRE((const void*)power != (const void*)wave && (const void*)bounds != (const void*)wave &&
                 (const void*)bounds != (const void*)power, "trim_silence: power and bounds must not alias wave or each other");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("trim_silence", st);
    trim_power_kernel<<<cdiv(s.total_frames, POWER_WARPS), POWER_WARPS * 32, 0, st>>>(s, wave, soff, foff, power);
    B200_LAUNCH_CHECK();
    trim_bounds_kernel<<<s.B, BOUNDS_THREADS, 0, st>>>(s, soff, foff, power, bounds);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
