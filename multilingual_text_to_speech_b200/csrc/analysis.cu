// Audio analysis: waveform -> log (mel) spectrogram -> cepstrum -> mel cepstral distortion, reference utils/audio.py:66-78, 117-161
// (librosa 0.7.0 stft, melspectrogram, amplitude_to_db, mfcc; the reference's mel_cepstral_distorision).
//
// Packed ragged layouts: utterance b owns samples [soff[b], soff[b+1]) and frames [off[b], off[b+1]), F_b = 1 + L_b // hop; spectra are
// frame-major [sum F, bins].  Every kernel reads only its own utterance's (or pair's) data in a fixed order with no atomics, so a batch
// computes exactly what its members compute one at a time.
//
// The transform runs in fp64 (the FFT of fft.cuh on double2): the reference computes an fp64 FFT of an fp64 signal and rounds it to
// complex64 afterwards, and an fp32 FFT would leave rounding noise about 80 dB below the frame energy, inside the range the dB scale keeps.
#include <float.h>
#include <algorithm>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int AN_FRAMES = 4;            // frames per CTA of the STFT kernel
constexpr int AN_THREADS = 256;
constexpr int DB_THREADS = 1024;
constexpr int CEP_FRAMES = 32;          // frames per CTA of the cepstrum kernel
constexpr int MCD_THREADS = 512;
// DTW: three rolling anti-diagonals of (fp64 cost, int32 path length) per pair, indexed along the shorter sequence (n + 1 entries each)
constexpr size_t DTW_SMEM_LIMIT = 227 * 1024;
constexpr int DTW_CELL_BYTES = 3 * (sizeof(double) + sizeof(int));
static_assert(B200TTS_DTW_MAX_FRAMES == (int)(DTW_SMEM_LIMIT / DTW_CELL_BYTES) - 1, "B200TTS_DTW_MAX_FRAMES follows from 227 KB");

// fp64 twiddles and window (fft.cuh), and the nonzero bin range [first, last] of each mel filter (first > last: an empty filter)
__global__ void analysis_tables_kernel(int N, int win, double2* __restrict__ twM, double2* __restrict__ twN, double* __restrict__ window,
                                       int n_mels, const float* __restrict__ basis, int2* __restrict__ ranges) {
    fill_fft_tables(N, win, twM, twN, window);
    const int K = N / 2 + 1;
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < n_mels; m += gridDim.x * blockDim.x) {
        int fk = K, lk = -1;
        for (int k = 0; k < K; ++k)
            if (basis[(size_t)m * K + k] != 0.f) { fk = min(fk, k); lk = k; }
        ranges[m] = make_int2(fk, lk);
    }
}

// Per frame: pre-emphasis y[n] - a y[n - 1] (y[-1] = 0) in fp64 on the fp32 samples -> reflect padding by N/2 -> fp64 window -> fp64 real
// FFT -> rounded to complex64 -> |.| by hypotf (numpy's abs of complex64).  n_mels > 0: out = basis . S, each filter summing its nonzero
// bins in ascending order in fp32.
__global__ void __launch_bounds__(AN_THREADS) analysis_stft_kernel(FftPlan p, int total, int B, int hop, const float* __restrict__ wave,
                                                                   const int* __restrict__ soff, const int* __restrict__ off, double pre,
                                                                   const double2* __restrict__ twM, const double2* __restrict__ twN,
                                                                   const double* __restrict__ window, int n_mels,
                                                                   const float* __restrict__ basis, const int2* __restrict__ ranges,
                                                                   float* __restrict__ out) {
    const FftSmem<double2> sm = load_tables<double2, AN_FRAMES>(p, twM, twN, window);
    const int M = p.M, N = p.N, K = M + 1, ld = M + 1, f0 = blockIdx.x * AN_FRAMES;
    const int nfr = min(AN_FRAMES, total - f0);
    double2* Z = sm.buf;
    double2* W = sm.buf + AN_FRAMES * ld;
    for (int i = threadIdx.x; i < nfr * N; i += blockDim.x) {
        const int f = i / N, n = i - f * N;
        const int gf = f0 + f, b = utterance_of(off, B, gf);
        const int s0 = soff[b], L = soff[b + 1] - s0;
        const int s = reflect_index((gf - off[b]) * hop + n - N / 2, L);
        const float* y = wave + s0;
        double v = (double)y[s];
        if (s > 0) v = __dadd_rn(v, -__dmul_rn(pre, (double)y[s - 1]));        // lfilter's roundings
        reinterpret_cast<double*>(Z + f * ld)[n] = v * sm.window[n];
    }
    __syncthreads();
    const double2* z = block_cfft(Z, W, ld, nfr, p, sm.twM, false);
    float* mag = reinterpret_cast<float*>(z == Z ? W : Z);          // the free buffer: [nfr][K] magnitudes for the mel sums
    for (int i = threadIdx.x; i < nfr * K; i += blockDim.x) {
        const int f = i / K, k = i - f * K;
        const double2 x = z[f * ld + (k == M ? 0 : k)], y = z[f * ld + (k == 0 ? 0 : M - k)];
        const double2 ev = make_double2(x.x + y.x, x.y - y.y);
        const double2 od = make_double2(x.x - y.x, x.y + y.y);
        const double2 t = cmul(od, sm.twN[k]);
        const float re = (float)(0.5 * (ev.x + t.y)), im = (float)(0.5 * (ev.y - t.x));     // (ev - i t) / 2, rounded to complex64
        const float a = hypotf(re, im);
        if (n_mels == 0) out[(size_t)(f0 + f) * K + k] = a;
        else mag[f * K + k] = a;
    }
    if (n_mels == 0) return;
    __syncthreads();
    for (int i = threadIdx.x; i < nfr * n_mels; i += blockDim.x) {
        const int f = i / n_mels, m = i - f * n_mels;
        const int2 r = ranges[m];
        float acc = 0.f;
        for (int k = r.x; k <= r.y; ++k) acc = fmaf(basis[(size_t)m * K + k], mag[f * K + k], acc);
        out[(size_t)(f0 + f) * n_mels + m] = acc;
    }
}

// librosa amplitude_to_db(S, ref=np.max, amin=1e-5, top_db=None) = power_to_db(S^2, ref=max(S)^2, amin=1e-10) in fp32, one CTA per
// utterance: the max over all its values (exact in any order), then 10 log10(max(1e-10, s^2)) - 10 log10(max(1e-10, ref^2)).
__global__ void __launch_bounds__(DB_THREADS) analysis_db_kernel(int bins, const int* __restrict__ off, const float* __restrict__ S,
                                                                 float* __restrict__ out) {
    __shared__ float red[64];
    const int b = blockIdx.x;
    const size_t e0 = (size_t)off[b] * bins, e1 = (size_t)off[b + 1] * bins;
    float mx = -INFINITY;
    for (size_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) mx = fmaxf(mx, fabsf(S[i]));
    mx = block_max(mx, red);
    const float ref_db = 10.f * log10f(fmaxf(1e-10f, __fmul_rn(mx, mx)));
    for (size_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) {
        const float a = fabsf(S[i]);
        out[i] = __fsub_rn(__fmul_rn(10.f, log10f(fmaxf(1e-10f, __fmul_rn(a, a)))), ref_db);
    }
}

// mfcc(S = mel_db / 10): DCT-II with norm='ortho' over the n_mels axis, first n_mfcc coefficients.  The matrix is built from fp64 cospi and
// rounded to fp32; each coefficient sums its n_mels products in ascending order with fmaf.
__global__ void analysis_cepstrum_kernel(int total, int n_mels, int n_mfcc, const float* __restrict__ mel_db, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* D = reinterpret_cast<float*>(smem_raw);                 // [n_mfcc, n_mels]
    float* x = D + n_mfcc * n_mels;                                // [CEP_FRAMES, n_mels]
    const int f0 = blockIdx.x * CEP_FRAMES, nfr = min(CEP_FRAMES, total - f0);
    for (int i = threadIdx.x; i < n_mfcc * n_mels; i += blockDim.x) {
        const int k = i / n_mels, n = i - k * n_mels;
        const double s = k == 0 ? sqrt(1.0 / n_mels) : sqrt(2.0 / n_mels);
        D[i] = (float)(s * cospi((double)k * (2 * n + 1) / (2.0 * n_mels)));
    }
    for (int i = threadIdx.x; i < nfr * n_mels; i += blockDim.x) x[i] = __fdiv_rn(mel_db[(size_t)f0 * n_mels + i], 10.f);
    __syncthreads();
    for (int i = threadIdx.x; i < nfr * n_mfcc; i += blockDim.x) {
        const int f = i / n_mfcc, k = i - f * n_mfcc;
        float acc = 0.f;
        for (int n = 0; n < n_mels; ++n) acc = fmaf(D[k * n_mels + n], x[f * n_mels + n], acc);
        out[(size_t)(f0 + f) * n_mfcc + k] = acc;
    }
}

// Euclidean distance of cepstral frames a and b over coefficients 1..n_mfcc-1 (c0 dropped, as the reference's [1:]): squares summed in
// index order with explicit roundings, then a correctly rounded sqrtf -- reproducible bit for bit by a numpy float32 mirror.
__device__ __forceinline__ float frame_distance(const float* __restrict__ a, const float* __restrict__ b, int n_mfcc) {
    float acc = 0.f;
    for (int c = 1; c < n_mfcc; ++c) {
        const float d = __fsub_rn(a[c], b[c]);
        acc = __fadd_rn(acc, __fmul_rn(d, d));
    }
    return sqrtf(acc);
}

// Fixed-order fp64 block sum: per-thread partials in shared memory, then a tree over them; the same order for any batch.
__device__ double block_sum_fixed(double v, double* red) {
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    return red[0];
}

// cut / stretch, one CTA per pair: the mean of the frame distances over the paired frames (reference utils/audio.py:143-153), summed in
// fp64.  stretch indexes the shorter sequence at i * n // m over the longer length m; at equal lengths the first sequence is the one
// indexed, as the reference's else branch does (an identity map).
__global__ void __launch_bounds__(MCD_THREADS) analysis_mcd_linear_kernel(int n_mfcc, int mode, const float* __restrict__ A,
                                                                          const int* __restrict__ off_a, const float* __restrict__ Bc,
                                                                          const int* __restrict__ off_b, double* __restrict__ mcd,
                                                                          int* __restrict__ path_len) {
    __shared__ double red[MCD_THREADS];
    const int p = blockIdx.x;
    const int oa = off_a[p], Fa = off_a[p + 1] - oa, ob = off_b[p], Fb = off_b[p + 1] - ob;
    const int m = mode == B200TTS_MCD_CUT ? min(Fa, Fb) : max(Fa, Fb);
    double acc = 0.0;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        int ia = i, ib = i;
        if (mode == B200TTS_MCD_STRETCH) {
            if (Fa > Fb) ib = (int)((long long)i * Fb / m);
            else ia = (int)((long long)i * Fa / m);
        }
        acc += (double)frame_distance(A + (size_t)(oa + ia) * n_mfcc, Bc + (size_t)(ob + ib) * n_mfcc, n_mfcc);
    }
    const double sum = block_sum_fixed(acc, red);
    if (threadIdx.x == 0) {
        mcd[p] = sum / m;
        if (path_len) path_len[p] = m;
    }
}

// Exact DTW, one CTA per pair (the recurrence of fastdtw.dtw): D[0,0] = 0, the borders infinite; cell (i, j), i, j >= 1, costs
// d(a[i-1], b[j-1]) plus its predecessor, the first minimum of the sums over (i-1, j), (i, j-1), (i-1, j-1) in that order; the path
// length follows the chosen predecessor.  Anti-diagonals s = i + j are swept in order, three of them kept in shared memory, indexed by the
// cell's position q along the shorter sequence (i when Fa <= Fb, else j), so nothing but the result reaches global memory.  A pair whose
// shorter side exceeds B200TTS_DTW_MAX_FRAMES gets NaN and path length -1 (the host rejects it before the launch).
__global__ void __launch_bounds__(MCD_THREADS) analysis_mcd_dtw_kernel(int n_mfcc, const float* __restrict__ A,
                                                                       const int* __restrict__ off_a, const float* __restrict__ Bc,
                                                                       const int* __restrict__ off_b, double* __restrict__ mcd,
                                                                       int* __restrict__ path_len) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int p = blockIdx.x;
    const int oa = off_a[p], Fa = off_a[p + 1] - oa, ob = off_b[p], Fb = off_b[p + 1] - ob;
    const bool by_i = Fa <= Fb;
    const int n = by_i ? Fa : Fb;
    if (n > B200TTS_DTW_MAX_FRAMES) {
        if (threadIdx.x == 0) {
            mcd[p] = __longlong_as_double(0x7ff8000000000000ll);
            if (path_len) path_len[p] = -1;
        }
        return;
    }
    const int W = n + 1;
    double* cost = reinterpret_cast<double*>(smem_raw);            // [3][W]: diagonals s - 2, s - 1, s in rotation
    int* len = reinterpret_cast<int*>(cost + 3 * W);
    for (int q = threadIdx.x; q < 3 * W; q += blockDim.x) { cost[q] = INFINITY; len[q] = 0; }
    __syncthreads();
    if (threadIdx.x == 0) cost[0] = 0.0;                            // D[0, 0] on diagonal 0 (slot 0, q = 0)
    __syncthreads();
    for (int s = 2; s <= Fa + Fb; ++s) {
        const int cur = s % 3, d1 = (s + 2) % 3, d2 = (s + 1) % 3;
        const int ilo = max(1, s - Fb), ihi = min(Fa, s - 1);
        const int qlo = by_i ? ilo : s - ihi, qhi = by_i ? ihi : s - ilo;
        for (int q = threadIdx.x; q < W; q += blockDim.x) {
            if (q < qlo || q > qhi) {
                // not a cell of this diagonal: the border value (the i = 0 and j = 0 cells read later are among these slots)
                cost[cur * W + q] = INFINITY;
                len[cur * W + q] = 0;
                continue;
            }
            const int i = by_i ? q : s - q, j = s - i;
            const double d = (double)frame_distance(A + (size_t)(oa + i - 1) * n_mfcc, Bc + (size_t)(ob + j - 1) * n_mfcc, n_mfcc);
            // slots of (i-1, j), (i, j-1), (i-1, j-1)
            const int qu = by_i ? q - 1 : q, ql = by_i ? q : q - 1, qd = q - 1;
            double best = cost[d1 * W + qu] + d;
            int bl = len[d1 * W + qu];
            const double cl = cost[d1 * W + ql] + d;
            if (cl < best) { best = cl; bl = len[d1 * W + ql]; }
            const double cd = cost[d2 * W + qd] + d;
            if (cd < best) { best = cd; bl = len[d2 * W + qd]; }
            cost[cur * W + q] = best;
            len[cur * W + q] = bl + 1;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int q = by_i ? Fa : Fb;
        const int slot = (Fa + Fb) % 3;
        const int L = len[slot * W + q];
        mcd[p] = cost[slot * W + q] / L;
        if (path_len) path_len[p] = L;
    }
}

}  // namespace

static int analysis_validate(const b200tts_analysis_shape& s, FftPlan* plan) {
    B200_REQUIRE(s.B >= 1 && s.total_samples >= s.B && s.total_frames >= s.B,
                 "analysis: need B >= 1 and at least one sample and one frame per utterance (B = %d, total_samples = %d, total_frames = %d)",
                 s.B, s.total_samples, s.total_frames);
    B200_REQUIRE(make_plan(s.N, plan), "analysis: unsupported FFT size N = %d (even, <= 2048, N/2 with prime factors <= 31 only)", s.N);
    B200_REQUIRE(s.win >= 1 && s.win <= s.N, "analysis: window length %d must be in [1, N = %d]", s.win, s.N);
    B200_REQUIRE(s.hop >= 1, "analysis: hop %d must be positive", s.hop);
    B200_REQUIRE(s.n_mels >= 0 && s.n_mels <= s.N / 2 + 1, "analysis: n_mels %d must be in [0, K = %d]", s.n_mels, s.N / 2 + 1);
    B200_REQUIRE(s.preemphasis == s.preemphasis && fabs(s.preemphasis) < 1e30, "analysis: preemphasis must be finite");
    B200_REQUIRE((long long)s.total_frames * (s.N / 2 + 1) < (1ll << 40), "analysis: batch too large");
    return B200TTS_OK;
}

// workspace: twiddles W_M [M] and W_N [M + 1] (double2), window [N] (double), mel filter ranges [n_mels] (int2); each region 256-byte aligned
struct AnalysisLayout { size_t twM, twN, window, ranges, bytes; };
static AnalysisLayout analysis_layout(const b200tts_analysis_shape& s) {
    const size_t M = s.N / 2;
    AnalysisLayout l;
    l.twM = 0;
    l.twN = align_up_sz(l.twM + M * sizeof(double2), 256);
    l.window = align_up_sz(l.twN + (M + 1) * sizeof(double2), 256);
    l.ranges = align_up_sz(l.window + (size_t)s.N * sizeof(double), 256);
    l.bytes = align_up_sz(l.ranges + (size_t)s.n_mels * sizeof(int2), 256);
    return l;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_analysis_workspace_bytes(const b200tts_analysis_shape* shape) {
    if (!shape) { set_last_error("analysis_workspace_bytes: null shape"); return 0; }
    FftPlan p;
    if (analysis_validate(*shape, &p) != B200TTS_OK) return 0;
    return analysis_layout(*shape).bytes;
}

int b200tts_stft_magnitude(const b200tts_analysis_shape* shape, const float* wave, const int32_t* soff, const int32_t* off,
                           const float* mel_basis, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && wave && soff && off && out, "stft_magnitude: null argument");
    B200_TRY(require_device());
    const b200tts_analysis_shape& s = *shape;
    FftPlan p;
    B200_TRY(analysis_validate(s, &p));
    B200_REQUIRE(s.n_mels == 0 || mel_basis, "stft_magnitude: n_mels = %d needs the mel basis", s.n_mels);
    const AnalysisLayout l = analysis_layout(s);
    B200_REQUIRE(workspace && workspace_bytes >= l.bytes, "stft_magnitude: workspace of %zu bytes is smaller than the %zu required",
                 workspace_bytes, l.bytes);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "stft_magnitude: workspace must be 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = static_cast<unsigned char*>(workspace);
    double2* twM = reinterpret_cast<double2*>(base + l.twM);
    double2* twN = reinterpret_cast<double2*>(base + l.twN);
    double* window = reinterpret_cast<double*>(base + l.window);
    int2* ranges = reinterpret_cast<int2*>(base + l.ranges);
    {
        KernelTimer kt("analysis_tables", st);
        analysis_tables_kernel<<<cdiv(s.N + s.N + 1, 256), 256, 0, st>>>(s.N, s.win, twM, twN, window, s.n_mels, mel_basis, ranges);
        B200_LAUNCH_CHECK();
    }
    const size_t smem = fft_smem_bytes<double2, AN_FRAMES>(p);
    B200_CUDA(cudaFuncSetAttribute(analysis_stft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("analysis_stft", st);
    analysis_stft_kernel<<<cdiv(s.total_frames, AN_FRAMES), AN_THREADS, smem, st>>>(p, s.total_frames, s.B, s.hop, wave, soff, off,
                                                                                    s.preemphasis, twM, twN, window, s.n_mels, mel_basis,
                                                                                    ranges, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_amplitude_to_db(const b200tts_analysis_shape* shape, const float* S, const int32_t* off, float* out, void* stream) {
    B200_REQUIRE(shape && S && off && out, "amplitude_to_db: null argument");
    B200_TRY(require_device());
    const b200tts_analysis_shape& s = *shape;
    FftPlan p;
    B200_TRY(analysis_validate(s, &p));
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("analysis_db", st);
    analysis_db_kernel<<<s.B, DB_THREADS, 0, st>>>(s.n_mels ? s.n_mels : p.M + 1, off, S, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_mel_cepstrum(int total_frames, int n_mels, int n_mfcc, const float* mel_db, float* out, void* stream) {
    B200_REQUIRE(mel_db && out, "mel_cepstrum: null argument");
    B200_REQUIRE(total_frames >= 1, "mel_cepstrum: total_frames %d must be positive", total_frames);
    B200_REQUIRE(n_mels >= 1 && n_mels <= 1024, "mel_cepstrum: n_mels %d must be in [1, 1024]", n_mels);
    B200_REQUIRE(n_mfcc >= 1 && n_mfcc <= n_mels, "mel_cepstrum: n_mfcc %d must be in [1, n_mels = %d]", n_mfcc, n_mels);
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)(n_mfcc + CEP_FRAMES) * n_mels * sizeof(float);      // at most 2 * 1024 * 32 * 4 bytes
    B200_CUDA(cudaFuncSetAttribute(analysis_cepstrum_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("analysis_cepstrum", st);
    analysis_cepstrum_kernel<<<cdiv(total_frames, CEP_FRAMES), 256, smem, st>>>(total_frames, n_mels, n_mfcc, mel_db, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_mel_cepstral_distortion(int B, int n_mfcc, int mode, const float* cep_a, const int32_t* off_a, const float* cep_b,
                                    const int32_t* off_b, double* mcd_out, int32_t* path_len_out, void* stream) {
    B200_REQUIRE(cep_a && off_a && cep_b && off_b && mcd_out, "mel_cepstral_distortion: null argument");
    B200_REQUIRE(B >= 1, "mel_cepstral_distortion: B %d must be positive", B);
    B200_REQUIRE(n_mfcc >= 2, "mel_cepstral_distortion: n_mfcc %d must be at least 2 (c0 is dropped)", n_mfcc);
    B200_REQUIRE(mode == B200TTS_MCD_CUT || mode == B200TTS_MCD_STRETCH || mode == B200TTS_MCD_DTW,
                 "mel_cepstral_distortion: unknown mode %d", mode);
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    if (mode != B200TTS_MCD_DTW) {
        KernelTimer kt("analysis_mcd", st);
        analysis_mcd_linear_kernel<<<B, MCD_THREADS, 0, st>>>(n_mfcc, mode, cep_a, off_a, cep_b, off_b, mcd_out, path_len_out);
        B200_LAUNCH_CHECK();
        return B200TTS_OK;
    }
    const size_t smem = (size_t)(B200TTS_DTW_MAX_FRAMES + 1) * DTW_CELL_BYTES;
    B200_CUDA(cudaFuncSetAttribute(analysis_mcd_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("analysis_dtw", st);
    analysis_mcd_dtw_kernel<<<B, MCD_THREADS, smem, st>>>(n_mfcc, cep_a, off_a, cep_b, off_b, mcd_out, path_len_out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
