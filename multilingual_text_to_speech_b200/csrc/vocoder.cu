// Griffin-Lim vocoder: log spectrogram -> waveform, reference utils/audio.py:88-97 (librosa 0.7.0 mel_to_stft, griffinlim, deemphasis).
//
// Packed ragged layout, frame-major: utterance b owns frames [off[b], off[b+1]); magnitudes are [sum F, K] fp32, angles and `rebuilt`
// [sum F, K] float2, K = N/2 + 1.  Waveforms are packed at hop * (off[b] - b) with hop * (F_b - 1) samples each.  Every kernel reads only
// its own utterance's data in a fixed order (no atomics), so a batch computes exactly what its utterances compute one at a time.
//
// Real FFT of length N = 2M: a complex Stockham FFT of length M in shared memory (mixed radix, plan built on the host, every twiddle one
// lookup in a table of M roots computed in fp64) plus the even / odd split.  fp32 throughout: Griffin-Lim is a phase-retrieval fixed point
// on inputs spanning 80 dB, so no reduced-precision tensor-core DFT.
#include <float.h>
#include <algorithm>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int FRAMES_PER_CTA = 4;
constexpr int FFT_THREADS = 256;
constexpr int NNLS_WARPS = 8;
constexpr int DEEMPH_THREADS = 1024;

// Sample q of the untrimmed overlap-add of utterance frames [0, F) (q in [0, N + hop * (F - 1))), divided by the window sum-square where
// that exceeds tiny(float32) (librosa istft).  The contributing frames are added in ascending order, as librosa's overlap-add does.
__device__ __forceinline__ float ola_sample(const float* __restrict__ frames, const float* __restrict__ window, int N, int hop, int F, int q) {
    int t0 = q - N + 1 <= 0 ? 0 : (q - N + 1 + hop - 1) / hop;
    int t1 = q / hop;
    if (t1 > F - 1) t1 = F - 1;
    float acc = 0.f, wss = 0.f;
    for (int t = t0; t <= t1; ++t) {
        const int n = q - t * hop;
        const float w = window[n];
        acc += frames[(size_t)t * N + n];
        wss = fmaf(w, w, wss);
    }
    return wss > FLT_MIN ? acc / wss : acc;
}

// Twiddles W_M^j, W_N^k (k <= M) and the periodic Hann window of length win centre-padded to N, all from fp64 and rounded to fp32.
__global__ void vocoder_tables_kernel(int N, int win, float2* __restrict__ twM, float2* __restrict__ twN, float* __restrict__ window) {
    fill_fft_tables(N, win, twM, twN, window);
}

// (a) per frame: X = S * angles -> inverse real FFT (numpy irfft: 1/N, imaginary parts of the DC and Nyquist bins ignored) -> times the
// window -> frames[f, 0:N]
__global__ void __launch_bounds__(FFT_THREADS) vocoder_istft_frames_kernel(FftPlan p, int total, const float* __restrict__ S,
                                                                           const float2* __restrict__ angles, const float2* __restrict__ twM,
                                                                           const float2* __restrict__ twN, const float* __restrict__ window,
                                                                           float* __restrict__ frames) {
    const FftSmem<float2> sm = load_tables<float2, FRAMES_PER_CTA>(p, twM, twN, window);
    const int M = p.M, K = M + 1, ld = M + 1, f0 = blockIdx.x * FRAMES_PER_CTA;
    const int nfr = min(FRAMES_PER_CTA, total - f0);
    float2* X = sm.buf;
    float2* Z = sm.buf + FRAMES_PER_CTA * ld;
    for (int i = threadIdx.x; i < nfr * K; i += blockDim.x) {
        const int f = i / K, k = i - f * K;
        const size_t g = (size_t)(f0 + f) * K + k;
        const float s = S[g];
        const float2 a = angles[g];
        X[f * ld + k] = make_float2(s * a.x, (k == 0 || k == M) ? 0.f : s * a.y);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nfr * M; i += blockDim.x) {
        const int f = i / M, k = i - f * M;
        const float2 x = X[f * ld + k], y = X[f * ld + M - k];
        const float2 ev = make_float2(x.x + y.x, x.y - y.y);          // X[k] + conj(X[M - k])
        const float2 od = make_float2(x.x - y.x, x.y + y.y);          // X[k] - conj(X[M - k])
        const float2 t = cmulc(od, sm.twN[k]);                        // * W_N^-k
        Z[f * ld + k] = make_float2(ev.x - t.y, ev.y + t.x);          // ev + i t
    }
    __syncthreads();
    const float2* z = block_cfft(Z, X, ld, nfr, p, sm.twM, true);
    const float scale = 1.f / (float)p.N;
    for (int i = threadIdx.x; i < nfr * p.N; i += blockDim.x) {
        const int f = i / p.N, n = i - f * p.N;
        const float2 v = z[f * ld + (n >> 1)];
        frames[(size_t)(f0 + f) * p.N + n] = ((n & 1) ? v.y : v.x) * scale * sm.window[n];
    }
}

// (b) per frame: the reflect-padded iSTFT signal around the frame (overlap-add gathered from `frames`) -> window -> forward real FFT ->
// rebuilt; then angles = rebuilt - momentum / (1 + momentum) * tprev, angles /= |angles| + 1e-16 (tprev = 0 when `first`).
// np.pad(mode='reflect') reflects again and again when the signal is shorter than the pad: the index map is periodic with period
// 2 (L - 1) (a single sample repeats).
__global__ void __launch_bounds__(FFT_THREADS) vocoder_stft_update_kernel(FftPlan p, int total, int B, int hop, const int* __restrict__ off,
                                                                          const float* __restrict__ frames, const float2* __restrict__ twM,
                                                                          const float2* __restrict__ twN, const float* __restrict__ window,
                                                                          float2* __restrict__ rebuilt, float2* __restrict__ angles,
                                                                          float mom, int first) {
    const FftSmem<float2> sm = load_tables<float2, FRAMES_PER_CTA>(p, twM, twN, window);
    const int M = p.M, N = p.N, K = M + 1, ld = M + 1, f0 = blockIdx.x * FRAMES_PER_CTA;
    const int nfr = min(FRAMES_PER_CTA, total - f0);
    float2* Z = sm.buf;
    float2* W = sm.buf + FRAMES_PER_CTA * ld;
    for (int i = threadIdx.x; i < nfr * N; i += blockDim.x) {
        const int f = i / N, n = i - f * N;
        const int gf = f0 + f, b = utterance_of(off, B, gf);
        const int ob = off[b], F = off[b + 1] - ob, L = hop * (F - 1);
        const int s = reflect_index((gf - ob) * hop + n - N / 2, L);  // sample of the trimmed signal
        const float y = ola_sample(frames + (size_t)ob * N, sm.window, N, hop, F, s + N / 2);
        reinterpret_cast<float*>(Z + f * ld)[n] = y * sm.window[n];
    }
    __syncthreads();
    const float2* z = block_cfft(Z, W, ld, nfr, p, sm.twM, false);
    for (int i = threadIdx.x; i < nfr * K; i += blockDim.x) {
        const int f = i / K, k = i - f * K;
        const float2 x = z[f * ld + (k == M ? 0 : k)], y = z[f * ld + (k == 0 ? 0 : M - k)];
        const float2 ev = make_float2(x.x + y.x, x.y - y.y);
        const float2 od = make_float2(x.x - y.x, x.y + y.y);
        const float2 t = cmul(od, sm.twN[k]);
        const float2 X = make_float2(0.5f * (ev.x + t.y), 0.5f * (ev.y - t.x));   // (ev - i t) / 2
        const size_t g = (size_t)(f0 + f) * K + k;
        float2 a = X;
        if (!first) {
            const float2 tp = rebuilt[g];
            a = make_float2(X.x - mom * tp.x, X.y - mom * tp.y);
        }
        rebuilt[g] = X;
        const float d = hypotf(a.x, a.y) + 1e-16f;
        angles[g] = make_float2(a.x / d, a.y / d);
    }
}

// final inverse: the trimmed overlap-add, one thread per output sample
__global__ void vocoder_waveform_kernel(int B, int N, int hop, long long total_samples, const int* __restrict__ off,
                                        const float* __restrict__ frames, const float* __restrict__ window, float* __restrict__ wave) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total_samples; i += (long long)gridDim.x * blockDim.x) {
        // utterance b starts at hop * (off[b] - b)
        int lo = 0, hi = B - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if ((long long)hop * (off[mid] - mid) <= i) lo = mid; else hi = mid - 1;
        }
        const int ob = off[lo], F = off[lo + 1] - ob;
        const int j = (int)(i - (long long)hop * (ob - lo));
        wave[i] = ola_sample(frames + (size_t)ob * N, window, N, hop, F, j + N / 2);
    }
}

// Steps 1-3 of the magnitude path.  Linear input: S = db_to_amplitude(s) ^ power elementwise.
__global__ void vocoder_linear_magnitude_kernel(long long n, const float* __restrict__ log_spec, float power, float* __restrict__ S) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        S[i] = powf(sqrtf(exp10f(0.1f * log_spec[i])), power);
}

// Mel input, one warp per frame: b = db_to_amplitude(s), x = nnls(A, b) by FISTA from clip(pinv(A) b, 0) with step 1 / ||A||^2, then
// x ^ power.  Every linear bin lies in at most two adjacent filters (the Slaney basis), so A x and A^T r cost about 2 K multiply-adds:
// bin k keeps (lo[k], A[lo, k], A[lo + 1, k]) and filter m the bin range [first[m], last[m]].
__global__ void __launch_bounds__(NNLS_WARPS * 32) vocoder_mel_nnls_kernel(int total, int K, int nm, const float* __restrict__ log_mel,
                                                                         const float* __restrict__ basis, const float* __restrict__ pinv_t,
                                                                         float step, int iters, float power, float* __restrict__ S) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int* lo = reinterpret_cast<int*>(smem_raw);
    int* first = lo + K;
    int* last = first + nm;
    float* a0 = reinterpret_cast<float*>(last + nm);
    float* a1 = a0 + K;
    float* per_warp = a1 + K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* xs = per_warp + warp * (2 * K + 2 * nm);
    float* ys = xs + K;
    float* bm = ys + K;
    float* r = bm + nm;

    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        int l = -1;
        for (int m = 0; m < nm && l < 0; ++m)
            if (basis[(size_t)m * K + k] != 0.f) l = m;
        lo[k] = l;
        a0[k] = l >= 0 ? basis[(size_t)l * K + k] : 0.f;
        a1[k] = (l >= 0 && l + 1 < nm) ? basis[(size_t)(l + 1) * K + k] : 0.f;
    }
    for (int m = threadIdx.x; m < nm; m += blockDim.x) {
        int fk = K, lk = -1;
        for (int k = 0; k < K; ++k)
            if (basis[(size_t)m * K + k] != 0.f) { fk = min(fk, k); lk = k; }
        first[m] = fk;
        last[m] = lk;
    }
    __syncthreads();

    const int f = blockIdx.x * NNLS_WARPS + warp;
    if (f >= total) return;
    for (int m = lane; m < nm; m += 32) bm[m] = sqrtf(exp10f(0.1f * log_mel[(size_t)f * nm + m]));
    __syncwarp();
    for (int k = lane; k < K; k += 32) {
        float acc = 0.f;
        for (int m = 0; m < nm; ++m) acc = fmaf(pinv_t[(size_t)m * K + k], bm[m], acc);
        acc = fmaxf(acc, 0.f);
        xs[k] = acc;
        ys[k] = acc;
    }
    __syncwarp();
    float t = 1.f;
    for (int it = 0; it < iters; ++it) {
        for (int m = lane; m < nm; m += 32) {
            float acc = -bm[m];
            for (int k = first[m]; k <= last[m]; ++k) acc = fmaf(lo[k] == m ? a0[k] : a1[k], ys[k], acc);
            r[m] = acc;
        }
        __syncwarp();
        const float tn = 0.5f * (1.f + sqrtf(fmaf(4.f * t, t, 1.f)));
        const float beta = (t - 1.f) / tn;
        for (int k = lane; k < K; k += 32) {
            const int l = lo[k];
            const float g = l < 0 ? 0.f : fmaf(a0[k], r[l], l + 1 < nm ? a1[k] * r[l + 1] : 0.f);
            const float xn = fmaxf(fmaf(-step, g, ys[k]), 0.f);
            ys[k] = fmaf(beta, xn - xs[k], xn);
            xs[k] = xn;
        }
        __syncwarp();
        t = tn;
    }
    for (int k = lane; k < K; k += 32) S[(size_t)f * K + k] = powf(xs[k], power);
}

// De-emphasis y[n] = x[n] + a y[n - 1] (scipy lfilter([1], [1, -a])) and y /= max(y), one CTA per utterance.  Two-level scan of the
// first-order recurrence: each thread runs its contiguous chunk from 0 and keeps (a^len, last value); the block scans those affine maps
// (warp shuffles, then across warps); each thread re-runs its chunk from its carry.  The division is by the largest sample, not the largest
// magnitude, as the reference's Python max(y) is.  Rows (the WaveRNN folds): CTA b filters the row wave[b hop, (b + 1) hop) and does not
// normalise; off is not read.
template <bool Rows>
__global__ void __launch_bounds__(DEEMPH_THREADS) vocoder_deemphasis_kernel(int hop, const int* __restrict__ off, float a,
                                                                           float* __restrict__ wave) {
    __shared__ float wa[32], wv[32], red[64];
    const int b = blockIdx.x;
    int L;
    float* y;
    if constexpr (Rows) {
        L = hop;
        y = wave + (size_t)hop * b;
    } else {
        const int ob = off[b];
        L = hop * (off[b + 1] - ob - 1);
        y = wave + (size_t)hop * (ob - b);
    }
    const int chunk = (L + blockDim.x - 1) / blockDim.x;
    const int s0 = min(L, (int)threadIdx.x * chunk), s1 = min(L, s0 + chunk);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float mx = -INFINITY;
    if (a != 0.f) {
        float A = 1.f, V = 0.f;
        for (int i = s0; i < s1; ++i) { V = fmaf(a, V, y[i]); A *= a; }
        // inclusive scan of (A, V) maps: (A1, V1) then (A2, V2) = (A1 A2, A2 V1 + V2)
        for (int o = 1; o < 32; o <<= 1) {
            const float pa = __shfl_up_sync(0xffffffffu, A, o), pv = __shfl_up_sync(0xffffffffu, V, o);
            if (lane >= o) { V = fmaf(A, pv, V); A *= pa; }
        }
        if (lane == 31) { wa[warp] = A; wv[warp] = V; }
        __syncthreads();
        if (warp == 0) {
            float A2 = lane < (int)(blockDim.x >> 5) ? wa[lane] : 1.f, V2 = lane < (int)(blockDim.x >> 5) ? wv[lane] : 0.f;
            for (int o = 1; o < 32; o <<= 1) {
                const float pa = __shfl_up_sync(0xffffffffu, A2, o), pv = __shfl_up_sync(0xffffffffu, V2, o);
                if (lane >= o) { V2 = fmaf(A2, pv, V2); A2 *= pa; }
            }
            wa[lane] = A2; wv[lane] = V2;
        }
        __syncthreads();
        // carry into this thread: the previous warps' total, then the previous lanes of this warp
        const float cw = warp > 0 ? wv[warp - 1] : 0.f;
        const float pA = __shfl_up_sync(0xffffffffu, A, 1), pV = __shfl_up_sync(0xffffffffu, V, 1);
        const float carry = lane > 0 ? fmaf(pA, cw, pV) : cw;
        float prev = carry;
        for (int i = s0; i < s1; ++i) { prev = fmaf(a, prev, y[i]); y[i] = prev; mx = fmaxf(mx, prev); }
    } else {
        for (int i = s0; i < s1; ++i) mx = fmaxf(mx, y[i]);
    }
    if constexpr (Rows) return;
    mx = block_max(mx, red);
    for (int i = s0; i < s1; ++i) y[i] = y[i] / mx;
}

}  // namespace

static int vocoder_validate(const b200tts_vocoder_shape& s, FftPlan* plan) {
    B200_REQUIRE(s.B >= 1 && s.total_frames >= 2 * s.B, "vocoder: need B >= 1 and at least 2 frames per utterance (B = %d, total_frames = %d)",
                 s.B, s.total_frames);
    B200_REQUIRE(make_plan(s.N, plan), "vocoder: unsupported FFT size N = %d (even, <= 2048, N/2 with prime factors <= 31 only)", s.N);
    B200_REQUIRE(s.win >= 1 && s.win <= s.N, "vocoder: window length %d must be in [1, N = %d]", s.win, s.N);
    B200_REQUIRE(s.hop >= 1 && s.hop <= s.win, "vocoder: hop %d must be in [1, win = %d]", s.hop, s.win);
    B200_REQUIRE(s.n_mels >= 0 && s.n_mels <= s.N / 2 + 1, "vocoder: n_mels %d must be in [0, K = %d]", s.n_mels, s.N / 2 + 1);
    B200_REQUIRE(s.nnls_iters >= 0, "vocoder: negative nnls_iters %d", s.nnls_iters);
    B200_REQUIRE(s.power > 0.f, "vocoder: power must be positive");
    B200_REQUIRE((long long)s.hop * (s.total_frames - s.B) < (1ll << 31) && (long long)s.total_frames * s.N < (1ll << 40),
                 "vocoder: batch too large");
    return B200TTS_OK;
}

// workspace: twiddles W_M [M], W_N [M + 1], window [N], frame buffer [total_frames, N]; each region 256-byte aligned
struct VocoderLayout { size_t twM, twN, window, frames, bytes; };
static VocoderLayout vocoder_layout(const b200tts_vocoder_shape& s) {
    const size_t M = s.N / 2;
    VocoderLayout l;
    l.twM = 0;
    l.twN = align_up_sz(l.twM + M * sizeof(float2), 256);
    l.window = align_up_sz(l.twN + (M + 1) * sizeof(float2), 256);
    l.frames = align_up_sz(l.window + (size_t)s.N * sizeof(float), 256);
    l.bytes = align_up_sz(l.frames + (size_t)s.total_frames * s.N * sizeof(float), 256);
    return l;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_vocoder_workspace_bytes(const b200tts_vocoder_shape* shape) {
    if (!shape) { set_last_error("vocoder_workspace_bytes: null shape"); return 0; }
    FftPlan p;
    if (vocoder_validate(*shape, &p) != B200TTS_OK) return 0;
    return vocoder_layout(*shape).bytes;
}

int b200tts_vocoder_fft_plan(int N, int* radices, int capacity) {
    B200_REQUIRE(radices || capacity == 0, "vocoder_fft_plan: null radices");
    FftPlan p;
    B200_REQUIRE(make_plan(N, &p), "vocoder: unsupported FFT size N = %d (even, <= 2048, N/2 with prime factors <= 31 only)", N);
    for (int i = 0; i < p.nst && i < capacity; ++i) radices[i] = p.radix[i];
    return p.nst;
}

int b200tts_spectrogram_magnitude(const b200tts_vocoder_shape* shape, const float* log_spec, const float* mel_basis, const float* mel_pinv_t,
                                  float nnls_step, float* S_out, void* stream) {
    B200_REQUIRE(shape && log_spec && S_out, "spectrogram_magnitude: null argument");
    B200_TRY(require_device());
    const b200tts_vocoder_shape& s = *shape;
    FftPlan p;
    B200_TRY(vocoder_validate(s, &p));
    cudaStream_t st = (cudaStream_t)stream;
    const int K = p.M + 1;
    if (s.n_mels == 0) {
        KernelTimer kt("vocoder_magnitude", st);
        const long long n = (long long)s.total_frames * K;
        vocoder_linear_magnitude_kernel<<<(int)std::min<long long>((n + 255) / 256, NUM_SMS * 16), 256, 0, st>>>(n, log_spec, s.power, S_out);
        B200_LAUNCH_CHECK();
        return B200TTS_OK;
    }
    B200_REQUIRE(mel_basis && mel_pinv_t, "spectrogram_magnitude: a mel input needs the mel basis and its transposed pseudo-inverse");
    B200_REQUIRE(nnls_step > 0.f, "spectrogram_magnitude: the NNLS step must be positive");
    const size_t smem = (size_t)(2 * K + 2 * s.n_mels) * sizeof(int) + (size_t)K * 2 * sizeof(float) +
                        (size_t)NNLS_WARPS * (2 * K + 2 * s.n_mels) * sizeof(float);
    B200_CUDA(cudaFuncSetAttribute(vocoder_mel_nnls_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("vocoder_magnitude", st);
    vocoder_mel_nnls_kernel<<<cdiv(s.total_frames, NNLS_WARPS), NNLS_WARPS * 32, smem, st>>>(s.total_frames, K, s.n_mels, log_spec, mel_basis,
                                                                                           mel_pinv_t, nnls_step, s.nnls_iters, s.power, S_out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_griffinlim(const b200tts_vocoder_shape* shape, const float* S, const int32_t* off, float* angles, float* rebuilt, int first,
                       int iters, float* wave, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && S && off && angles && rebuilt, "griffinlim: null argument");
    B200_TRY(require_device());
    const b200tts_vocoder_shape& s = *shape;
    FftPlan p;
    B200_TRY(vocoder_validate(s, &p));
    B200_REQUIRE(iters >= 0, "griffinlim: negative iteration count %d", iters);
    const VocoderLayout l = vocoder_layout(s);
    B200_REQUIRE(workspace && workspace_bytes >= l.bytes, "griffinlim: workspace of %zu bytes is smaller than the %zu required", workspace_bytes,
                 l.bytes);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "griffinlim: workspace must be 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = static_cast<unsigned char*>(workspace);
    float2* twM = reinterpret_cast<float2*>(base + l.twM);
    float2* twN = reinterpret_cast<float2*>(base + l.twN);
    float* window = reinterpret_cast<float*>(base + l.window);
    float* frames = reinterpret_cast<float*>(base + l.frames);
    float2* ang = reinterpret_cast<float2*>(angles);
    float2* reb = reinterpret_cast<float2*>(rebuilt);
    const float mom = s.momentum / (1.f + s.momentum);

    vocoder_tables_kernel<<<cdiv(s.N + s.N + 1, 256), 256, 0, st>>>(s.N, s.win, twM, twN, window);
    B200_LAUNCH_CHECK();
    const size_t smem = fft_smem_bytes<float2, FRAMES_PER_CTA>(p);
    B200_CUDA(cudaFuncSetAttribute(vocoder_istft_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B200_CUDA(cudaFuncSetAttribute(vocoder_stft_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = cdiv(s.total_frames, FRAMES_PER_CTA);
    for (int it = 0; it <= iters; ++it) {
        if (it == iters && !wave) break;
        {
            KernelTimer kt("vocoder_istft_frames", st);
            vocoder_istft_frames_kernel<<<grid, FFT_THREADS, smem, st>>>(p, s.total_frames, S, ang, twM, twN, window, frames);
            B200_LAUNCH_CHECK();
        }
        if (it < iters) {
            KernelTimer kt("vocoder_stft_update", st);
            vocoder_stft_update_kernel<<<grid, FFT_THREADS, smem, st>>>(p, s.total_frames, s.B, s.hop, off, frames, twM, twN, window, reb, ang,
                                                                        mom, first && it == 0);
            B200_LAUNCH_CHECK();
        }
    }
    if (wave) {
        KernelTimer kt("vocoder_waveform", st);
        const long long n = (long long)s.hop * (s.total_frames - s.B);
        vocoder_waveform_kernel<<<(int)std::min<long long>((n + 255) / 256, NUM_SMS * 16), 256, 0, st>>>(s.B, s.N, s.hop, n, off, frames,
                                                                                                       window, wave);
        B200_LAUNCH_CHECK();
    }
    return B200TTS_OK;
}

int b200tts_deemphasis_normalize(const b200tts_vocoder_shape* shape, float* wave, const int32_t* off, void* stream) {
    B200_REQUIRE(shape && wave && off, "deemphasis_normalize: null argument");
    B200_TRY(require_device());
    const b200tts_vocoder_shape& s = *shape;
    FftPlan p;
    B200_TRY(vocoder_validate(s, &p));
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("vocoder_deemphasis", st);
    vocoder_deemphasis_kernel<false><<<s.B, DEEMPH_THREADS, 0, st>>>(s.hop, off, s.preemphasis, wave);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"

int b200tts::deemphasis_rows(int rows, int len, float a, float* y, cudaStream_t st) {
    if (a == 0.f) return B200TTS_OK;
    vocoder_deemphasis_kernel<true><<<rows, DEEMPH_THREADS, 0, st>>>(len, nullptr, a, y);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}
