// Pitch modification: TD-PSOLA pitch shifting in two stages -- the analysis and synthesis pitch marks of each utterance, then the
// overlap-add of the grains as a gather.  include/b200tts.h states the contract; tests/psola_oracle.py restates it in numpy.
//
// Packed ragged layout as pitch.cu: utterance b owns samples [soff[b], soff[b+1]) and frames [off[b], off[b+1]).  The mark walk is serial
// within an utterance: one warp per utterance, every lane following the same walk and the lanes sharing each argmax.  The overlap-add is
// one thread per output sample.  Nothing uses atomics and every sum runs in increasing grain order, so a batch computes exactly what its
// members compute one at a time.  Everything is fp64.
#include <limits.h>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int MARK_WARPS = 4;                // one warp per utterance
constexpr int OLA_THREADS = 256;             // one thread per output sample

struct PsolaWorkspace {
    int4* info;                              // [B]: analysis marks K, synthesis marks J, grain 0's left half-width, largest half-width W
    int* marks;                              // [total_samples], utterance b from soff[b]
    int* spacing;                            // d
    int* centre;                             // c
    int* nearest;                            // k
    uint8_t* voiced;
};

__host__ __device__ inline size_t psola_workspace_bytes(int B, int total_samples) {
    return (size_t)B * sizeof(int4) + (size_t)total_samples * (4 * sizeof(int) + sizeof(uint8_t));
}

__host__ __device__ inline PsolaWorkspace psola_workspace(void* ws, int B, int total_samples) {
    PsolaWorkspace w;
    w.info = static_cast<int4*>(ws);
    w.marks = reinterpret_cast<int*>(w.info + B);
    w.spacing = w.marks + total_samples;
    w.centre = w.spacing + total_samples;
    w.nearest = w.centre + total_samples;
    w.voiced = reinterpret_cast<uint8_t*>(w.nearest + total_samples);
    return w;
}

// one utterance's view of the tracks
struct Track {
    const float* f0;
    const float* ratio;
    int F, hop;
    double sr;
    __device__ int frame(int n) const { return min(F - 1, (n + hop / 2) / hop); }
    // rint(sr / f0) of sample n's frame, 0 when unvoiced; clamped to [2, B200TTS_PSOLA_MAX_PERIOD] (the host rejects anything outside)
    __device__ int period(int n) const {
        const float v = f0[frame(n)];
        if (isnan(v)) return 0;
        return (int)fmin(fmax(rint(sr / (double)v), 2.0), (double)B200TTS_PSOLA_MAX_PERIOD);
    }
    // the ratio of sample n's frame, clamped to [0.5, 2] (NaN -> 0.5; the host rejects anything outside)
    __device__ double rate(int n) const { return fmin(fmax((double)ratio[frame(n)], 0.5), 2.0); }
    // the first voiced sample in [a, bound], or -1: at most a few frames, since bound - a <= U and U <= hop in the library's use
    __device__ int first_voiced(int a, int bound) const {
        for (int f = frame(a), fe = frame(bound); f <= fe; ++f)
            if (!isnan(f0[f])) return max(a, max(0, f * hop - hop / 2));
        return -1;
    }
};

// first index of the maximum of x[lo .. hi] (inclusive, lo <= hi), every lane of the warp taking part and getting the result
__device__ int warp_argmax(const float* __restrict__ x, int lo, int hi, int lane) {
    float bv = 0.0f;
    int bi = INT_MAX;
    for (int i = lo + lane; i <= hi; i += 32) {
        const float v = x[i];
        if (bi == INT_MAX || v > bv) { bv = v; bi = i; }
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, sh);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, sh);
        if (oi != INT_MAX && (bi == INT_MAX || ov > bv || (ov == bv && oi < bi))) { bv = ov; bi = oi; }
    }
    return bi;
}

__global__ void __launch_bounds__(MARK_WARPS * 32) psola_marks_kernel(b200tts_psola_shape s, const float* __restrict__ wave,
                                                                      const int* __restrict__ soff, const float* __restrict__ f0,
                                                                      const float* __restrict__ ratio, const int* __restrict__ off,
                                                                      void* __restrict__ workspace) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * MARK_WARPS + (threadIdx.x >> 5);
    if (b >= s.B) return;
    const PsolaWorkspace w = psola_workspace(workspace, s.B, s.total_samples);
    const int s0 = soff[b], L = soff[b + 1] - s0, U = s.unvoiced_spacing;
    const float* x = wave + s0;
    const Track tr{f0 + off[b], ratio + off[b], off[b + 1] - off[b], s.hop, s.sr};
    int* marks = w.marks + s0;
    int* spacing = w.spacing + s0;
    uint8_t* voiced = w.voiced + s0;

    // analysis marks: every lane walks the same marks; lane 0 writes them
    int K = 0, wmax = U;
    int m = 0;
    {
        const int p0 = tr.period(0);
        if (p0) m = warp_argmax(x, 0, min(L, p0) - 1, lane);
    }
    const int p_first = tr.period(m);
    const int a0 = max(p_first ? p_first : U, m);
    wmax = max(wmax, a0);
    while (true) {
        const int p = tr.period(m);
        int next = -1;
        if (p) {
            const int c = m + p;
            if (c < L) next = tr.period(c) ? warp_argmax(x, c - p / 4, min(L - 1, c + p / 4), lane) : c;
        } else {
            const int o = tr.first_voiced(m + 1, min(m + U, L - 1));
            if (o >= 0) next = warp_argmax(x, o, min(L, o + tr.period(o)) - 1, lane);
            else if (m + U < L) next = m + U;
        }
        const int d = next >= 0 ? next - m : (p ? p : U);
        if (lane == 0) {
            marks[K] = m;
            spacing[K] = d;
            voiced[K] = p != 0;
        }
        ++K;
        wmax = max(wmax, d);
        if (next < 0) break;
        m = next;
    }
    if (lane != 0) return;

    // synthesis marks: t accumulates in fp64; the nearest-mark pointer only moves forward, as the centres never decrease
    int* centre = w.centre + s0;
    int* nearest = w.nearest + s0;
    double t = (double)marks[0];
    int J = 0, k = 0;
    while (true) {
        const int c = (int)rint(t);
        if (c >= L) break;
        while (k + 1 < K && marks[k] + marks[k + 1] < 2 * c) ++k;
        centre[J] = c;
        nearest[J] = k;
        ++J;
        const double d = (double)spacing[k];
        t += voiced[k] ? d / tr.rate(c) : d;
    }
    w.info[b] = make_int4(K, J, a0, wmax);
}

// one thread per output sample: the grains whose centre lies in [n - W, n + W] are found by binary search and summed in order
__global__ void __launch_bounds__(OLA_THREADS) psola_ola_kernel(b200tts_psola_shape s, const float* __restrict__ wave,
                                                                const int* __restrict__ soff, const void* __restrict__ workspace,
                                                                float* __restrict__ out) {
    const PsolaWorkspace w = psola_workspace(const_cast<void*>(workspace), s.B, s.total_samples);
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < s.total_samples; g += gridDim.x * blockDim.x) {
        const int b = utterance_of(soff, s.B, g);
        const int s0 = soff[b], L = soff[b + 1] - s0, n = g - s0;
        const int4 info = w.info[b];
        const int K = info.x, J = info.y, a0 = info.z, W = info.w;
        const int* marks = w.marks + s0;
        const int* spacing = w.spacing + s0;
        const int* centre = w.centre + s0;
        const int* nearest = w.nearest + s0;
        const float* x = wave + s0;
        int lo = 0, hi = J;                  // the first centre >= n - W
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (centre[mid] < n - W) lo = mid + 1; else hi = mid;
        }
        double num = 0.0, den = 0.0;
        for (int j = lo; j < J; ++j) {
            const int c = centre[j];
            if (c > n + W) break;
            const int k = nearest[j];
            const int a = k ? spacing[k - 1] : a0, bw = spacing[k], u = n - c, src = marks[k] + u;
            if (u < -a || u > bw || src < 0 || src >= L) continue;
            // cospi: the argument is within [-1, 1], and cos(pi v) would carry the stack frame of its large-argument reduction
            double wt;
            if (u <= 0) wt = k == 0 ? 1.0 : 0.5 * (1.0 + cospi((double)u / (a + 1)));
            else wt = k == K - 1 ? 1.0 : 0.5 * (1.0 + cospi((double)u / (bw + 1)));
            num += wt * (double)x[src];
            den += wt;
        }
        out[g] = (float)(num / fmax(den, 1.0));
    }
}

}  // namespace

static int psola_validate(const b200tts_psola_shape& s) {
    B200_REQUIRE(s.B >= 1 && s.total_samples >= s.B && s.total_frames >= s.B,
                 "psola: need B >= 1 and at least one sample and one frame per utterance (B = %d, total_samples = %d, total_frames = %d)",
                 s.B, s.total_samples, s.total_frames);
    B200_REQUIRE(s.hop >= 1, "psola: hop %d must be positive", s.hop);
    B200_REQUIRE(s.unvoiced_spacing >= 1 && s.unvoiced_spacing <= B200TTS_PSOLA_MAX_PERIOD, "psola: unvoiced_spacing %d must be in [1, %d]",
                 s.unvoiced_spacing, B200TTS_PSOLA_MAX_PERIOD);
    B200_REQUIRE(s.sr > 0 && s.sr < 1e30, "psola: sr must be positive and finite");
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_psola_workspace_bytes(const b200tts_psola_shape* shape) {
    if (!shape) { set_last_error("psola_workspace_bytes: null shape"); return 0; }
    if (psola_validate(*shape) != B200TTS_OK) return 0;
    return psola_workspace_bytes(shape->B, shape->total_samples);
}

int b200tts_psola_marks(const b200tts_psola_shape* shape, const float* wave, const int32_t* soff, const float* f0, const float* ratio,
                        const int32_t* off, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && wave && soff && f0 && ratio && off, "psola_marks: null argument");
    const b200tts_psola_shape& s = *shape;
    B200_TRY(psola_validate(s));
    const size_t need = psola_workspace_bytes(s.B, s.total_samples);
    B200_REQUIRE(workspace && workspace_bytes >= need, "psola_marks: workspace of %zu bytes is smaller than the %zu required",
                 workspace_bytes, need);
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("psola_marks", st);
    psola_marks_kernel<<<cdiv(s.B, MARK_WARPS), MARK_WARPS * 32, 0, st>>>(s, wave, soff, f0, ratio, off, workspace);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_psola_overlap_add(const b200tts_psola_shape* shape, const float* wave, const int32_t* soff, const void* workspace,
                              size_t workspace_bytes, float* out, void* stream) {
    B200_REQUIRE(shape && wave && soff && out, "psola_overlap_add: null argument");
    const b200tts_psola_shape& s = *shape;
    B200_TRY(psola_validate(s));
    const size_t need = psola_workspace_bytes(s.B, s.total_samples);
    B200_REQUIRE(workspace && workspace_bytes >= need, "psola_overlap_add: workspace of %zu bytes is smaller than the %zu required",
                 workspace_bytes, need);
    B200_REQUIRE(out != wave, "psola_overlap_add: out must not alias wave");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("psola_overlap_add", st);
    psola_ola_kernel<<<cdiv(s.total_samples, OLA_THREADS), OLA_THREADS, 0, st>>>(s, wave, soff, workspace, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
