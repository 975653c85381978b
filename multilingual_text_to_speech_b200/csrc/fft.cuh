// Shared-memory real FFT pieces of the audio kernels (vocoder.cu: fp32 Griffin-Lim; analysis.cu: fp64 forward transform).
//
// Real FFT of length N = 2M: a complex Stockham FFT of length M in shared memory (mixed radix, plan built on the host, every twiddle one
// lookup in a table of M roots computed in fp64) plus the even / odd split.  The complex type C is float2 (real type float) or double2
// (double); the tables are rounded to C's precision.
#pragma once
#include "common.cuh"

namespace b200tts {

namespace {

constexpr int FFT_MAX_STAGES = 12;

struct FftPlan {
    int M, N, nst;
    int radix[FFT_MAX_STAGES];
};

// radix-4 stages first, then one radix 2, then the odd primes in ascending order: the cost of a stage is M * radix multiply-adds
int make_plan(int N, FftPlan* p) {
    if (N < 2 || N > 2048 || (N & 1)) return 0;
    p->N = N;
    p->M = N / 2;
    p->nst = 0;
    int m = p->M;
    while (m % 4 == 0) { p->radix[p->nst++] = 4; m /= 4; }
    if (m % 2 == 0) { p->radix[p->nst++] = 2; m /= 2; }
    for (int q = 3; q <= 31; q += 2)
        while (m % q == 0) { p->radix[p->nst++] = q; m /= q; }
    return m == 1;
}

template <class C> struct FftReal;
template <> struct FftReal<float2> { using T = float; };
template <> struct FftReal<double2> { using T = double; };

__device__ __forceinline__ float fft_fma(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ double fft_fma(double a, double b, double c) { return fma(a, b, c); }
__device__ __forceinline__ void fft_store(float2* p, double c, double s) { *p = make_float2((float)c, (float)s); }
__device__ __forceinline__ void fft_store(double2* p, double c, double s) { *p = make_double2(c, s); }

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cmulc(float2 a, float2 b) { return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y); }   // a * conj(b)

// Complex FFT of length M over `nfr` frames stored at a[f * ld ...], ping-ponging with b; returns the buffer holding the result.
// Stage s (radix R, Ns = product of the earlier radices): output o = blk * Ns * R + j * Ns + k reads inputs jj + r * M / R with
// jj = blk * Ns + k, weighted by W_M^(r * (k + j * Ns) * M / (Ns * R)) -- the stage twiddle and the radix-R DFT in one root (conjugated for
// the inverse).  Each output is computed by one thread in ascending r.
template <class C>
__device__ C* block_cfft(C* a, C* b, int ld, int nfr, const FftPlan& p, const C* __restrict__ tw, bool inverse) {
    const int M = p.M;
    int Ns = 1;
    for (int s = 0; s < p.nst; ++s) {
        const int R = p.radix[s], NsR = Ns * R, sc = M / NsR, st = M / R;
        for (int idx = threadIdx.x; idx < nfr * M; idx += blockDim.x) {
            const int f = idx / M, o = idx - f * M;
            const int k = o % Ns, j = (o / Ns) % R, blk = o / NsR;
            const C* in = a + f * ld + blk * Ns + k;
            const int e = (k + j * Ns) * sc;
            int ti = 0;
            C acc;
            acc.x = 0;
            acc.y = 0;
            for (int r = 0; r < R; ++r) {
                const C v = in[r * st];
                const C w = tw[ti];
                acc.x = fft_fma(v.x, w.x, acc.x);
                acc.y = fft_fma(v.y, w.x, acc.y);
                if (inverse) { acc.x = fft_fma(-v.y, -w.y, acc.x); acc.y = fft_fma(v.x, -w.y, acc.y); }
                else         { acc.x = fft_fma(-v.y, w.y, acc.x);  acc.y = fft_fma(v.x, w.y, acc.y); }
                ti += e;
                if (ti >= M) ti -= M;
            }
            b[f * ld + o] = acc;
        }
        __syncthreads();
        C* t = a; a = b; b = t;
        Ns = NsR;
    }
    return a;
}

// utterance of frame f: the b with off[b] <= f < off[b + 1]
__device__ __forceinline__ int utterance_of(const int* __restrict__ off, int B, int f) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= f) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// np.pad(mode='reflect') as an index map: sample s (any integer) of the padded signal reads sample reflect_index(s, L) of a signal of L
// samples.  numpy reflects again and again when the signal is shorter than the pad: the map is periodic with period 2 (L - 1), and a
// single sample repeats.
__device__ __forceinline__ int reflect_index(int s, int L) {
    if (L == 1) return 0;
    const int period = 2 * (L - 1);
    s %= period;
    if (s < 0) s += period;
    if (s >= L) s = period - s;
    return s;
}

// Twiddles W_M^j, W_N^k (k <= M) and the periodic Hann window of length win centre-padded to N, all from fp64 and rounded to C's precision.
// Grid-stride over N + 2M + 1 entries.
template <class C>
__device__ __forceinline__ void fill_fft_tables(int N, int win, C* __restrict__ twM, C* __restrict__ twN,
                                                typename FftReal<C>::T* __restrict__ window) {
    using T = typename FftReal<C>::T;
    const int M = N / 2, lpad = (N - win) / 2;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N + 2 * M + 1; i += gridDim.x * blockDim.x) {
        double s, c;
        if (i < M) {
            sincospi(-2.0 * i / M, &s, &c);
            fft_store(twM + i, c, s);
        } else if (i < 2 * M + 1) {
            const int k = i - M;
            sincospi(-2.0 * k / N, &s, &c);
            fft_store(twN + k, c, s);
        } else {
            const int n = i - 2 * M - 1;
            const int m = n - lpad;
            window[n] = (m >= 0 && m < win) ? (T)(0.5 - 0.5 * cospi(2.0 * m / win)) : (T)0;
        }
    }
}

template <class C>
struct FftSmem {
    C *twM, *twN;
    typename FftReal<C>::T* window;
    C* buf;      // 2 * FRAMES buffers of M + 1 entries
};

// Dynamic shared memory of an FFT kernel that keeps FRAMES frames: twiddles W_M [M], W_N [M + 1], 2 * FRAMES frame buffers of M + 1
// entries, the window [N].  The tables are copied in from global memory.
template <class C, int FRAMES>
__device__ __forceinline__ FftSmem<C> load_tables(const FftPlan& p, const C* twM, const C* twN, const typename FftReal<C>::T* window) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FftSmem<C> s;
    const int M = p.M;
    s.twM = reinterpret_cast<C*>(smem_raw);
    s.twN = s.twM + M;
    s.buf = s.twN + (M + 1);
    s.window = reinterpret_cast<typename FftReal<C>::T*>(s.buf + 2 * FRAMES * (M + 1));
    for (int i = threadIdx.x; i < M; i += blockDim.x) s.twM[i] = twM[i];
    for (int i = threadIdx.x; i <= M; i += blockDim.x) s.twN[i] = twN[i];
    for (int i = threadIdx.x; i < p.N; i += blockDim.x) s.window[i] = window[i];
    __syncthreads();
    return s;
}

template <class C, int FRAMES>
size_t fft_smem_bytes(const FftPlan& p) {
    return (size_t)(p.M + (p.M + 1) + 2 * FRAMES * (p.M + 1)) * sizeof(C) + (size_t)p.N * sizeof(typename FftReal<C>::T);
}

}  // namespace

}  // namespace b200tts
