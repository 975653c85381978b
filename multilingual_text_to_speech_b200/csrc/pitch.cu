// Pitch analysis: probabilistic YIN (librosa 0.10 librosa.pyin) in three stages -- the cumulative mean normalised difference per frame,
// the observation probabilities of the pitch bins, and the Viterbi decode over voiced and unvoiced bins.
//
// Packed ragged layouts as analysis.cu: utterance b owns samples [soff[b], soff[b+1]) and frames [off[b], off[b+1]).  Stages A and B work
// on one frame at a time, stage C on one utterance per CTA; every sum runs in a fixed order with no atomics, so a batch computes exactly
// what its members compute one at a time.  Everything is fp64.
#include <float.h>
#include <algorithm>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int CMND_THREADS = 128;
constexpr int OBS_WARPS = 4;                 // one warp per frame
constexpr int VIT_THREADS = 1024;
constexpr int NT = B200TTS_PITCH_THRESHOLDS;
constexpr double NO_TROUGH_PROB = 0.01;
constexpr size_t VIT_SMEM_LIMIT = 227 * 1024;
// two rows of 2 n values, then prefix and suffix maxima (value, first index) of both halves
constexpr size_t vit_smem_bytes(int n) { return 2 * 2 * (size_t)n * sizeof(double) + 4 * (size_t)n * (sizeof(double) + sizeof(int)); }
static_assert(vit_smem_bytes(B200TTS_PITCH_MAX_BINS) <= VIT_SMEM_LIMIT, "the Viterbi rows fit in shared memory");
static_assert(2 * B200TTS_PITCH_MAX_BINS <= 65536, "uint16 back-pointers");

// Stage A, one CTA per frame.  The frame's samples go to shared memory in fp64; each thread takes lags tau = tid, tid + 128, ... <=
// max_period and sums acf and e over i in ascending order; thread 0 then accumulates the cumulative sums of d in lag order.
__global__ void __launch_bounds__(CMND_THREADS) pitch_cmnd_kernel(b200tts_pitch_shape s, const float* __restrict__ wave,
                                                                  const int* __restrict__ soff, const int* __restrict__ off,
                                                                  double* __restrict__ cmnd) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int N = s.frame_length, win = s.win_length, P = s.max_period;
    double* y = reinterpret_cast<double*>(smem_raw);            // [N]
    double* acf = y + N;                                         // [P + 1]
    double* en = acf + P + 1;                                    // [P + 1]
    double* cum = en + P + 1;                                    // [P + 1]: c(tau), the cumulative sums of d
    const int f = blockIdx.x, b = utterance_of(off, s.B, f);
    const int s0 = soff[b], L = soff[b + 1] - s0;
    const int start = (f - off[b]) * s.hop - N / 2;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int n = start + i;
        y[i] = (n >= 0 && n < L) ? (double)wave[s0 + n] : 0.0;
    }
    __syncthreads();
    for (int tau = threadIdx.x; tau <= P; tau += blockDim.x) {
        double a = 0.0, e = 0.0;
        for (int i = 1; i <= win; ++i) {
            a = fma(y[i], y[i + tau], a);
            const double v = y[i + tau];
            e = fma(v, v, e);
        }
        acf[tau] = fabs(a) < 1e-6 ? 0.0 : a;
        en[tau] = fabs(e) < 1e-6 ? 0.0 : e;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double c = 0.0;
        cum[0] = 0.0;
        for (int tau = 1; tau <= P; ++tau) {
            c += (en[0] + en[tau]) - 2.0 * acf[tau];
            cum[tau] = c;
        }
    }
    __syncthreads();
    const int K = P - s.min_period + 1;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const int tau = s.min_period + k;
        const double d = (en[0] + en[tau]) - 2.0 * acf[tau];
        cmnd[(size_t)f * K + k] = d / (cum[tau] / (double)tau + DBL_MIN);
    }
}

__device__ __forceinline__ bool is_trough(const double* __restrict__ x, int k, int K) {
    if (k == 0) return x[0] < x[1];
    if (k == K - 1) return x[K - 1] < x[K - 2];
    return x[k] < x[k - 1] && x[k] <= x[k + 1];
}

// pitch bin of the trough at lag index k: the parabolic shift, then rint(120 log2(sr / period / fmin)) clipped to [0, n]
__device__ __forceinline__ int trough_bin(const b200tts_pitch_shape& s, const double* __restrict__ x, int k, int K) {
    double shift = 0.0;
    if (k > 0 && k < K - 1) {
        const double a = x[k + 1] + x[k - 1] - 2.0 * x[k];
        const double b = (x[k + 1] - x[k - 1]) / 2.0;
        if (fabs(b) < fabs(a)) shift = -b / a;
    }
    const double period = (double)(s.min_period + k) + shift;
    const double r = rint(120.0 * log2(s.sr / period / s.fmin));
    return (int)fmin(fmax(r, 0.0), (double)s.n_bins);
}

// Stage B, one warp per frame.  The troughs are listed in lag order in shared memory (at most K / 2 + 1 of them: no two are adjacent).
// The probability of each trough sums over thresholds j in order; its position among the troughs below threshold j is the count below it
// in earlier 32-trough chunks (carry[j]) plus a ballot within the chunk.  Bins fall with the lag (the shift is below 1 in magnitude and
// troughs are at least 2 lags apart), so troughs sharing a bin are consecutive among those with nonzero probability, and the last wins.
__global__ void __launch_bounds__(OBS_WARPS * 32) pitch_obs_kernel(b200tts_pitch_shape s, const double* __restrict__ cmnd,
                                                                   double* __restrict__ obs, double* __restrict__ voiced_prob) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int K = s.max_period - s.min_period + 1, n = s.n_bins, TMAX = K / 2 + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * OBS_WARPS + warp;
    if (f >= s.total_frames) return;
    const size_t per_warp = (size_t)TMAX * (sizeof(double) + sizeof(int)) + 2 * NT * sizeof(int);
    unsigned char* base = smem_raw + warp * ((per_warp + 15) / 16 * 16);
    double* prob = reinterpret_cast<double*>(base);                     // [TMAX]
    int* tidx = reinterpret_cast<int*>(prob + TMAX);                    // [TMAX]
    int* nbelow = tidx + TMAX;                                          // [NT]: N_j
    int* carry = nbelow + NT;                                           // [NT]
    const double* x = cmnd + (size_t)f * K;
    double* o = obs + (size_t)f * n;
    for (int i = lane; i < n; i += 32) o[i] = 0.0;

    int T = 0;
    for (int k0 = 0; k0 < K; k0 += 32) {
        const int k = k0 + lane;
        const bool tr = k < K && is_trough(x, k, K);
        const unsigned m = __ballot_sync(0xffffffffu, tr);
        if (tr) tidx[T + __popc(m & ((1u << lane) - 1u))] = k;
        T += __popc(m);
    }
    __syncwarp();
    if (T == 0) {
        if (lane == 0) voiced_prob[f] = 0.0;
        return;
    }
    for (int j = lane; j < NT; j += 32) {
        int c = 0;
        for (int t = 0; t < T; ++t) c += x[tidx[t]] < s.thresholds[j];
        nbelow[j] = c;
        carry[j] = 0;
    }
    __syncwarp();
    for (int t0 = 0; t0 < T; t0 += 32) {
        const int t = t0 + lane;
        const double h = t < T ? x[tidx[t]] : INFINITY;
        double p = 0.0;
        for (int j = 0; j < NT; ++j) {
            const bool below = h < s.thresholds[j];
            const unsigned m = __ballot_sync(0xffffffffu, below);
            const int c = carry[j];
            if (below) {
                const int pos = c + __popc(m & ((1u << lane) - 1u));
                const double fact = (1.0 - exp(-2.0)) / (1.0 - exp(-2.0 * (double)nbelow[j]));
                p += fact * exp(-2.0 * (double)pos) * s.beta_probs[j];
            }
            __syncwarp();
            if (lane == 0) carry[j] = c + __popc(m);
            __syncwarp();
        }
        if (t < T) prob[t] = p;
    }
    // the first lowest trough
    double hm = INFINITY;
    int tm = T;
    for (int t = lane; t < T; t += 32) {
        const double h = x[tidx[t]];
        if (h < hm) { hm = h; tm = t; }
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) {
        const double oh = __shfl_xor_sync(0xffffffffu, hm, sh);
        const int ot = __shfl_xor_sync(0xffffffffu, tm, sh);
        if (oh < hm || (oh == hm && ot < tm)) { hm = oh; tm = ot; }
    }
    __syncwarp();
    if (lane == 0) {
        double mass = 0.0;
        for (int j = 0; j < NT && !(hm < s.thresholds[j]); ++j) mass += s.beta_probs[j];
        prob[tm] += NO_TROUGH_PROB * mass;
    }
    __syncwarp();
    // bins: lane-parallel over troughs; a trough wins its bin unless the next trough with nonzero probability has the same bin
    double vsum = 0.0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const int t = t0 + lane;
        int bin = -1;
        double p = 0.0;
        if (t < T && (p = prob[t]) != 0.0) bin = trough_bin(s, x, tidx[t], K);
        if (bin >= 0 && bin < n) {
            int next = -1;
            for (int u = t + 1; u < T; ++u) {
                if (prob[u] == 0.0) continue;
                next = trough_bin(s, x, tidx[u], K);
                break;
            }
            if (next != bin) {
                o[bin] = p;
                vsum += p;
            }
        }
    }
    // fixed-order warp sum of the winners
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) vsum += __shfl_xor_sync(0xffffffffu, vsum, sh);
    if (lane == 0) voiced_prob[f] = fmin(fmax(vsum, 0.0), 1.0);
}

struct Best { double v; int i; };

// inclusive scan of (value, index) maxima over one array of n values, one warp: each lane walks a contiguous block, the block maxima are
// combined across lanes by shuffles, and each lane walks its block again with the carry.  prefix: the first index of the maximum of
// w[0 .. m]; suffix: the first index of the maximum of w[m .. n).
template <bool SUFFIX>
__device__ void warp_max_scan(const double* __restrict__ w, int n, double* __restrict__ outv, int* __restrict__ outi, int lane) {
    const int per = (n + 31) / 32;
    const int lo = lane * per, hi = min(n, lo + per);
    Best acc{-INFINITY, -1};
    if (!SUFFIX) {
        for (int m = lo; m < hi; ++m) if (acc.i < 0 || w[m] > acc.v) acc = {w[m], m};
    } else {
        for (int m = hi - 1; m >= lo; --m) if (acc.i < 0 || w[m] >= acc.v) acc = {w[m], m};
    }
    // the carry from the blocks before (prefix) or after (suffix) this lane's, combined in index order
    Best carry{-INFINITY, -1};
    for (int l = 0; l < 32; ++l) {
        const int src = SUFFIX ? 31 - l : l;
        const double ov = __shfl_sync(0xffffffffu, acc.v, src);
        const int oi = __shfl_sync(0xffffffffu, acc.i, src);
        const bool before = SUFFIX ? src > lane : src < lane;
        if (before && oi >= 0) {
            if (carry.i < 0) carry = {ov, oi};
            else if (!SUFFIX ? ov > carry.v : ov >= carry.v) carry = {ov, oi};
        }
    }
    acc = carry;
    if (!SUFFIX) {
        for (int m = lo; m < hi; ++m) {
            if (acc.i < 0 || w[m] > acc.v) acc = {w[m], m};
            outv[m] = acc.v;
            outi[m] = acc.i;
        }
    } else {
        for (int m = hi - 1; m >= lo; --m) {
            if (acc.i < 0 || w[m] >= acc.v) acc = {w[m], m};
            outv[m] = acc.v;
            outi[m] = acc.i;
        }
    }
}

// Stage C, one CTA per utterance.  Destination bin i of either half takes the best of six groups of sources, in source-index order:
// voiced bins before the band, the voiced band, voiced bins after it, then the same for the unvoiced half.  Inside a band the candidate is
// value + log_trans exactly as the dense sum; outside it is value + log_tiny, whose maxima come from the prefix and suffix scans of those
// sums.  Strict comparisons in index order keep the lowest source on ties, as numpy's argmax.
__global__ void __launch_bounds__(VIT_THREADS) pitch_viterbi_kernel(b200tts_pitch_shape s, const double* __restrict__ obs,
                                                                    const double* __restrict__ vprob, const int* __restrict__ off,
                                                                    const double* __restrict__ log_trans, int* __restrict__ state,
                                                                    uint16_t* __restrict__ bp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int n = s.n_bins, W = s.transition_width, h = W / 2, S2 = 2 * n;
    double* rows = reinterpret_cast<double*>(smem_raw);                 // [2][2n]
    double* pv = rows + 2 * S2;                                          // [4][n]: prefix half 0, suffix half 0, prefix half 1, suffix half 1
    int* pi = reinterpret_cast<int*>(pv + 4 * n);                        // [4][n]
    const int b = blockIdx.x, f0 = off[b], F = off[b + 1] - f0;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const double LT = s.log_tiny;
    {
        const double lu = log((1.0 - vprob[f0]) / (double)n + DBL_MIN);
        for (int j = tid; j < S2; j += blockDim.x)
            rows[j] = j < n ? log(obs[(size_t)f0 * n + j] + DBL_MIN) + LT : lu + s.log_init;
    }
    __syncthreads();
    const double* stay = log_trans;
    const double* swch = log_trans + (size_t)W * n;
    for (int t = 1; t < F; ++t) {
        double* prev = rows + ((t - 1) & 1) * S2;
        double* cur = rows + (t & 1) * S2;
        // warps 0-3: the out-of-band sums prev + log_tiny of one half, staged in the scan's output array and scanned in place
        if (warp < 4) {
            double* wv = pv + warp * n;
            int* wi = pi + warp * n;
            const double* src = prev + (warp >> 1) * n;
            const int per = (n + 31) / 32;
            const int lo = lane * per, hi = min(n, lo + per);
            for (int m = lo; m < hi; ++m) wv[m] = src[m] + LT;
            __syncwarp();
            if (warp & 1) warp_max_scan<true>(wv, n, wv, wi, lane);
            else warp_max_scan<false>(wv, n, wv, wi, lane);
        }
        __syncthreads();
        const size_t fr = (size_t)(f0 + t);
        const double lu = log((1.0 - vprob[fr]) / (double)n + DBL_MIN);
        for (int i = tid; i < n; i += blockDim.x) {
            // bests of the two bands for destination (a, i) from source half c: bv[a][c]
            double bv[2][2];
            int bi[2][2];
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int c = 0; c < 2; ++c) { bv[a][c] = -INFINITY; bi[a][c] = -1; }
            const int q0 = max(0, h - i), q1 = min(W - 1, h + (n - 1 - i));
            for (int q = q0; q <= q1; ++q) {
                const int src = i - h + q;
                const double ls = stay[(size_t)q * n + i], lw = swch[(size_t)q * n + i];
                const double p0 = prev[src], p1 = prev[n + src];
                const double c00 = p0 + ls, c01 = p1 + lw, c10 = p0 + lw, c11 = p1 + ls;
                if (bi[0][0] < 0 || c00 > bv[0][0]) { bv[0][0] = c00; bi[0][0] = src; }
                if (bi[0][1] < 0 || c01 > bv[0][1]) { bv[0][1] = c01; bi[0][1] = n + src; }
                if (bi[1][0] < 0 || c10 > bv[1][0]) { bv[1][0] = c10; bi[1][0] = src; }
                if (bi[1][1] < 0 || c11 > bv[1][1]) { bv[1][1] = c11; bi[1][1] = n + src; }
            }
            const int pre = i - h - 1, suf = i + h + 1;
#pragma unroll
            for (int a = 0; a < 2; ++a) {
                double best = -INFINITY;
                int arg = -1;
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    if (pre >= 0) {
                        const double v = pv[(2 * c) * n + pre];
                        if (arg < 0 || v > best) { best = v; arg = c * n + pi[(2 * c) * n + pre]; }
                    }
                    if (arg < 0 || bv[a][c] > best) { best = bv[a][c]; arg = bi[a][c]; }
                    if (suf < n) {
                        const double v = pv[(2 * c + 1) * n + suf];
                        if (v > best) { best = v; arg = c * n + pi[(2 * c + 1) * n + suf]; }
                    }
                }
                const double lp = a == 0 ? log(obs[fr * n + i] + DBL_MIN) : lu;
                cur[a * n + i] = lp + best;
                bp[fr * S2 + a * n + i] = (uint16_t)arg;
            }
        }
        __syncthreads();
    }
    if (tid != 0) return;
    const double* last = rows + ((F - 1) & 1) * S2;
    int st = 0;
    for (int j = 1; j < S2; ++j) if (last[j] > last[st]) st = j;
    state[f0 + F - 1] = st;
    for (int t = F - 1; t > 0; --t) {
        st = bp[(size_t)(f0 + t) * S2 + st];
        state[f0 + t - 1] = st;
    }
}

}  // namespace

static int pitch_validate(const b200tts_pitch_shape& s) {
    B200_REQUIRE(s.B >= 1 && s.total_samples >= s.B && s.total_frames >= s.B,
                 "pitch: need B >= 1 and at least one sample and one frame per utterance (B = %d, total_samples = %d, total_frames = %d)",
                 s.B, s.total_samples, s.total_frames);
    B200_REQUIRE(s.frame_length >= 4 && s.frame_length % 2 == 0 && s.frame_length <= B200TTS_PITCH_MAX_FRAME_LENGTH,
                 "pitch: frame_length %d must be even and in [4, %d]", s.frame_length, B200TTS_PITCH_MAX_FRAME_LENGTH);
    B200_REQUIRE(s.win_length == s.frame_length / 2, "pitch: win_length %d must be frame_length / 2 = %d", s.win_length, s.frame_length / 2);
    B200_REQUIRE(s.hop >= 1, "pitch: hop %d must be positive", s.hop);
    B200_REQUIRE(s.min_period >= 1 && s.max_period > s.min_period && s.max_period <= s.frame_length - s.win_length - 1,
                 "pitch: need 1 <= min_period < max_period <= frame_length - win_length - 1 (min_period = %d, max_period = %d)",
                 s.min_period, s.max_period);
    B200_REQUIRE(s.n_bins >= 1 && s.n_bins <= B200TTS_PITCH_MAX_BINS, "pitch: n_bins %d must be in [1, %d]", s.n_bins, B200TTS_PITCH_MAX_BINS);
    B200_REQUIRE(s.transition_width >= 1 && s.transition_width % 2 == 1 && s.transition_width <= s.n_bins,
                 "pitch: transition_width %d must be odd and in [1, n_bins = %d]", s.transition_width, s.n_bins);
    B200_REQUIRE(s.sr > 0 && s.fmin > 0 && s.sr < 1e30 && s.fmin < 1e30, "pitch: sr and fmin must be positive and finite");
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_pitch_workspace_bytes(const b200tts_pitch_shape* shape) {
    if (!shape) { set_last_error("pitch_workspace_bytes: null shape"); return 0; }
    if (pitch_validate(*shape) != B200TTS_OK) return 0;
    return (size_t)shape->total_frames * 2 * shape->n_bins * sizeof(uint16_t);
}

int b200tts_pitch_cmnd(const b200tts_pitch_shape* shape, const float* wave, const int32_t* soff, const int32_t* off, double* cmnd_out,
                       void* stream) {
    B200_REQUIRE(shape && wave && soff && off && cmnd_out, "pitch_cmnd: null argument");
    const b200tts_pitch_shape& s = *shape;
    B200_TRY(pitch_validate(s));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = ((size_t)s.frame_length + 3 * (size_t)(s.max_period + 1)) * sizeof(double);
    B200_CUDA(cudaFuncSetAttribute(pitch_cmnd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("pitch_cmnd", st);
    pitch_cmnd_kernel<<<s.total_frames, CMND_THREADS, smem, st>>>(s, wave, soff, off, cmnd_out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_pitch_observations(const b200tts_pitch_shape* shape, const double* cmnd, double* obs_out, double* voiced_prob_out, void* stream) {
    B200_REQUIRE(shape && cmnd && obs_out && voiced_prob_out, "pitch_observations: null argument");
    const b200tts_pitch_shape& s = *shape;
    B200_TRY(pitch_validate(s));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const int K = s.max_period - s.min_period + 1, TMAX = K / 2 + 1;
    const size_t per_warp = ((size_t)TMAX * (sizeof(double) + sizeof(int)) + 2 * NT * sizeof(int) + 15) / 16 * 16;
    const size_t smem = OBS_WARPS * per_warp;
    B200_CUDA(cudaFuncSetAttribute(pitch_obs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("pitch_observations", st);
    pitch_obs_kernel<<<cdiv(s.total_frames, OBS_WARPS), OBS_WARPS * 32, smem, st>>>(s, cmnd, obs_out, voiced_prob_out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_pitch_viterbi(const b200tts_pitch_shape* shape, const double* obs, const double* voiced_prob, const int32_t* off,
                          const double* log_trans, int32_t* state_out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && obs && voiced_prob && off && log_trans && state_out, "pitch_viterbi: null argument");
    const b200tts_pitch_shape& s = *shape;
    B200_TRY(pitch_validate(s));
    const size_t need = (size_t)s.total_frames * 2 * s.n_bins * sizeof(uint16_t);
    B200_REQUIRE(workspace && workspace_bytes >= need, "pitch_viterbi: workspace of %zu bytes is smaller than the %zu required",
                 workspace_bytes, need);
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = vit_smem_bytes(s.n_bins);
    B200_CUDA(cudaFuncSetAttribute(pitch_viterbi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("pitch_viterbi", st);
    pitch_viterbi_kernel<<<s.B, VIT_THREADS, smem, st>>>(s, obs, voiced_prob, off, log_trans, state_out,
                                                         static_cast<uint16_t*>(workspace));
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
