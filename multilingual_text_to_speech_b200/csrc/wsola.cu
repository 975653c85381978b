// Time-scale modification: WSOLA in two stages -- the position of every synthesis frame, found by a serial search per utterance, then the
// overlap-add of the frames as a gather.  include/b200tts.h states the contract; tests/wsola_oracle.py restates it in numpy.
//
// Packed ragged layout as pitch.cu: utterance b owns input samples [soff[b], soff[b+1]), output samples [ooff[b], ooff[b+1]) and frames
// [foff[b], foff[b+1]).  The search is serial within an utterance: one CTA per utterance walks its frames, every thread scoring two
// neighbouring candidates per frame.  The overlap-add is one thread per output sample.  Nothing uses atomics and every sum runs in a fixed
// order, so a batch computes exactly what its members compute one at a time.  Everything is fp64.
#include <limits.h>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int SEARCH_THREADS = 1024;         // upper bound; a launch uses ceil((D + 1) / 32) warps, at most this many threads
constexpr int OLA_THREADS = 256;             // one thread per output sample

// dynamic shared memory of the search: the fp64 candidate span [2D + 2H + 1] and continuation [2H], then three fp32 staging buffers of
// 2D + 3H samples each (the frame being scored, the previous frame, and the next frame's prefetch)
__host__ __device__ inline int span_samples(int H, int D) { return 2 * D + 3 * H; }
__host__ __device__ inline int candidate_samples(int H, int D) { return 2 * D + 2 * H + 1; }
inline size_t search_smem_bytes(int H, int D) {
    return (size_t)(candidate_samples(H, D) + 2 * H) * sizeof(double) + 3 * (size_t)span_samples(H, D) * sizeof(float);
}
inline int search_threads(int D) { return min(SEARCH_THREADS, (D + 1 + 31) / 32 * 32); }

// x[start + i] for i in [0, S) into buf by cp.async, 0 outside [0, L) (zero-fill: no bytes are read); one commit group
__device__ __forceinline__ void stage_span(float* buf, const float* x, int L, long long start, int S) {
    for (int i = threadIdx.x; i < S; i += blockDim.x) {
        const long long j = start + i;
        const bool in = j >= 0 && j < L;
        const unsigned dst = (unsigned)__cvta_generic_to_shared(buf + i);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(in ? x + j : x), "r"(in ? 4 : 0) : "memory");
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
}

__device__ __forceinline__ void wait_staged() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// the search's order: larger score, then smaller |d|, then the negative d
__device__ __forceinline__ bool better(double s, int d, double bs, int bd) {
    if (s != bs) return s > bs;
    const int ad = abs(d), abd = abs(bd);
    return ad != abd ? ad < abd : d < bd;
}

__device__ __forceinline__ void warp_best(double& bs, int& bd) {
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, bs, sh);
        const int od = __shfl_xor_sync(0xffffffffu, bd, sh);
        if (better(os, od, bs, bd)) { bs = os; bd = od; }
    }
}

__global__ void __launch_bounds__(SEARCH_THREADS) wsola_search_kernel(b200tts_wsola_shape s, const float* __restrict__ wave,
                                                                      const int* __restrict__ soff, const double* __restrict__ warp,
                                                                      const int* __restrict__ foff, int* __restrict__ positions) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ double red_s[32];
    __shared__ int red_d[32];
    __shared__ int s_p;
    const int H = s.hop, D = s.tolerance, N = 2 * H, S = span_samples(H, D), V = candidate_samples(H, D);
    double* vd = reinterpret_cast<double*>(smem_raw);
    double* ud = vd + V;
    float* buf = reinterpret_cast<float*>(ud + N);
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int s0 = soff[b], L = soff[b + 1] - s0, f0 = foff[b], K = foff[b + 1] - f0;
    const float* x = wave + s0;
    const double* tau = warp + f0;
    int* pos = positions + f0;
    // a_k = rint(clamp(tau_k, 0, L)): fmax(NaN, 0) = 0, and the clamp keeps every index below within int
    auto nominal = [&](int k) { return (int)rint(fmin(fmax(tau[k], 0.0), (double)L)); };
    if (K <= 0) return;
    int a_prev = nominal(0), p_prev = a_prev;
    if (tid == 0) pos[0] = p_prev;
    if (K == 1) return;
    int a = nominal(1);
    stage_span(buf, x, L, (long long)a_prev - D - H, S);
    stage_span(buf + S, x, L, (long long)a - D - H, S);
    wait_staged();
    __syncthreads();
    for (int k = 1; k < K; ++k) {
        const float* cur = buf + (k % 3) * S;            // x[a_k - D - H ...]
        const float* prev = buf + ((k - 1) % 3) * S;     // x[a_{k-1} - D - H ...]
        // the next frame's span depends only on tau: fetch it while this frame is scored
        int a_next = 0;
        if (k + 1 < K) {
            a_next = nominal(k + 1);
            stage_span(buf + ((k + 1) % 3) * S, x, L, (long long)a_next - D - H, S);
        }
        // fp64 copies: vd[c + i] = v_{c - D, i - H} for candidate c, ud[i] = u_{i - H} = x[p_{k-1} + i]
        const int uoff = p_prev - a_prev + D + H;
        for (int i = tid; i < V; i += blockDim.x) vd[i] = (double)cur[i];
        for (int i = tid; i < N; i += blockDim.x) ud[i] = (double)prev[uoff + i];
        __syncthreads();
        // candidates 2q and 2q + 1 per thread: one new sample per step serves both, and each sum runs in increasing m
        double bs = -INFINITY;
        int bd = D + 1;                                  // no candidate yet: loses every comparison with a real one
        for (int q = tid; q <= D; q += blockDim.x) {
            const double* v = vd + 2 * q;
            double C0 = 0.0, E0 = 0.0, C1 = 0.0, E1 = 0.0;
            double v0 = v[0];
#pragma unroll 8
            for (int i = 0; i < N; ++i) {
                const double v1 = v[i + 1], uu = ud[i];
                C0 = fma(uu, v0, C0);
                E0 = fma(v0, v0, E0);
                C1 = fma(uu, v1, C1);
                E1 = fma(v1, v1, E1);
                v0 = v1;
            }
            const int d0 = 2 * q - D;
            const double sc0 = E0 > 0.0 ? C0 / sqrt(E0) : 0.0;
            if (better(sc0, d0, bs, bd)) { bs = sc0; bd = d0; }
            if (d0 + 1 <= D) {
                const double sc1 = E1 > 0.0 ? C1 / sqrt(E1) : 0.0;
                if (better(sc1, d0 + 1, bs, bd)) { bs = sc1; bd = d0 + 1; }
            }
        }
        warp_best(bs, bd);
        if (lane == 0) { red_s[wid] = bs; red_d[wid] = bd; }
        __syncthreads();
        if (wid == 0) {
            const int nw = blockDim.x >> 5;
            bs = lane < nw ? red_s[lane] : -INFINITY;
            bd = lane < nw ? red_d[lane] : D + 1;
            warp_best(bs, bd);
            if (lane == 0) {
                const int p = a + (bd <= D ? bd : 0);    // bd > D only when every score is NaN (non-finite input)
                s_p = p;
                pos[k] = p;
            }
        }
        wait_staged();
        __syncthreads();
        p_prev = s_p;
        a_prev = a;
        a = a_next;
    }
}

// one thread per output sample (the grid covers them all): frames n / H and n / H + 1, in that order.  The index is formed in 64 bits:
// with more than 2^30 output samples, blockIdx.x * blockDim.x + threadIdx.x or a grid stride added to it would overflow int
__global__ void __launch_bounds__(OLA_THREADS) wsola_ola_kernel(b200tts_wsola_shape s, const float* __restrict__ wave,
                                                                const int* __restrict__ soff, const int* __restrict__ positions,
                                                                const int* __restrict__ foff, const int* __restrict__ ooff,
                                                                float* __restrict__ out) {
    const long long gl = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gl >= s.total_out_samples) return;
    const int g = (int)gl, H = s.hop;
    const int b = utterance_of(ooff, s.B, g);
    const int n = g - ooff[b], s0 = soff[b], L = soff[b + 1] - s0, f0 = foff[b], K = foff[b + 1] - f0;
    const int k0 = n / H, r = n - k0 * H;
    double y = 0.0;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int k = k0 + j;
        if (k >= K) break;
        const int i = r + H - j * H;                     // n - kH + H, in [0, 2H)
        const long long src = (long long)positions[f0 + k] + i - H;
        const double xv = src >= 0 && src < L ? (double)wave[s0 + src] : 0.0;
        // cospi: the argument is within [0, 2), and cos(pi v) would carry the stack frame of its large-argument reduction
        y += (0.5 - 0.5 * cospi((double)i / H)) * xv;
    }
    out[g] = (float)y;
}

}  // namespace

static int wsola_validate(const b200tts_wsola_shape& s) {
    B200_REQUIRE(s.B >= 1 && s.total_samples >= s.B && s.total_out_samples >= s.B && s.total_frames >= 2 * s.B,
                 "wsola: need B >= 1, at least one input and one output sample and two frames per utterance (B = %d, total_samples = %d, "
                 "total_out_samples = %d, total_frames = %d)", s.B, s.total_samples, s.total_out_samples, s.total_frames);
    B200_REQUIRE(s.total_samples <= INT_MAX - B200TTS_WSOLA_MAX_TOLERANCE, "wsola: total_samples %d must be at most INT_MAX - %d",
                 s.total_samples, B200TTS_WSOLA_MAX_TOLERANCE);
    B200_REQUIRE(s.hop >= 1 && s.hop <= B200TTS_WSOLA_MAX_HOP, "wsola: hop %d must be in [1, %d]", s.hop, B200TTS_WSOLA_MAX_HOP);
    B200_REQUIRE(s.tolerance >= 0 && s.tolerance <= B200TTS_WSOLA_MAX_TOLERANCE, "wsola: tolerance %d must be in [0, %d]", s.tolerance,
                 B200TTS_WSOLA_MAX_TOLERANCE);
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

int b200tts_wsola_positions(const b200tts_wsola_shape* shape, const float* wave, const int32_t* soff, const double* warp,
                            const int32_t* foff, int32_t* positions, void* stream) {
    B200_REQUIRE(shape && wave && soff && warp && foff && positions, "wsola_positions: null argument");
    const b200tts_wsola_shape& s = *shape;
    B200_TRY(wsola_validate(s));
    B200_TRY(require_device());
    const size_t smem = search_smem_bytes(s.hop, s.tolerance);
    B200_CUDA(cudaFuncSetAttribute(wsola_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wsola_positions", st);
    wsola_search_kernel<<<s.B, search_threads(s.tolerance), smem, st>>>(s, wave, soff, warp, foff, positions);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wsola_overlap_add(const b200tts_wsola_shape* shape, const float* wave, const int32_t* soff, const int32_t* positions,
                              const int32_t* foff, const int32_t* ooff, float* out, void* stream) {
    B200_REQUIRE(shape && wave && soff && positions && foff && ooff && out, "wsola_overlap_add: null argument");
    const b200tts_wsola_shape& s = *shape;
    B200_TRY(wsola_validate(s));
    B200_REQUIRE((const void*)out != (const void*)wave, "wsola_overlap_add: out must not alias wave");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wsola_overlap_add", st);
    wsola_ola_kernel<<<cdiv(s.total_out_samples, OLA_THREADS), OLA_THREADS, 0, st>>>(s, wave, soff, positions, foff, ooff, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
