// Streaming Griffin-Lim: Real-Time Iterative Spectrogram Inversion with Look-Ahead (RTISI-LA; Zhu, Beauregard and Wyse, IEEE TASLP 2007),
// the specification in DESIGN ("Griffin-Lim vocoder", "Streaming").  The magnitudes come from b200tts_spectrogram_magnitude (vocoder.cu);
// this file owns the per-stream state and the frame loop.
//
// One CTA per stream and call: it loads its slot (the committed overlap-add c as a ring of N samples indexed by z mod N, the windowed
// estimates w x_j of the look-ahead set as a ring of k + 1 frames indexed by j mod (k + 1), their magnitudes, the counters and the
// de-emphasis carry) into shared memory, processes every ready frame in order and stores the slot back.  The frames of the look-ahead set
// are projected together, one real FFT pair per frame, on fft.cuh's shared-memory transform.  The released samples are divided in parallel
// and de-emphasised by one thread from the carried state.  No atomics and no reads of another slot: a stream's bits depend on its own frames
// only, not on its company or on how its frames were cut into calls.
#include <float.h>
#include <limits.h>
#include <algorithm>
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int GL_THREADS = 256;
constexpr int GL_MAX_A = B200TTS_GL_STREAM_MAX_LOOKAHEAD + 1;   // frames of the look-ahead set: one FFT pass
constexpr int GL_MAX_ROWS = 64;
constexpr size_t GL_MAX_SMEM = 227 * 1024;                      // sm_90 opt-in dynamic shared memory per block

struct GlRows { b200tts_gl_stream_row r[GL_MAX_ROWS]; };
struct GlSlotHeader { int committed, admitted, frames; float carry; };

// byte offsets: the tables in the workspace, the regions within a slot, the slot state in shared memory after the FFT tables
struct GlLayout { size_t twM, twN, window, slots, slot_bytes, c, x, S, bytes, smem_state, smem; };

GlLayout gl_layout(const b200tts_gl_stream_shape& s, const FftPlan& p) {
    const size_t M = p.M, K = M + 1, A = s.lookahead + 1;
    GlLayout l;
    l.twM = 0;
    l.twN = align_up_sz(l.twM + M * sizeof(float2), 256);
    l.window = align_up_sz(l.twN + K * sizeof(float2), 256);
    l.slots = align_up_sz(l.window + (size_t)s.N * sizeof(float), 256);
    l.c = 256;                                                     // after the header
    l.x = align_up_sz(l.c + (size_t)s.N * sizeof(float), 256);
    l.S = align_up_sz(l.x + A * s.N * sizeof(float), 256);
    l.slot_bytes = align_up_sz(l.S + A * K * sizeof(float), 256);
    l.bytes = l.slots + (size_t)s.slots * l.slot_bytes;
    l.smem_state = align_up_sz(fft_smem_bytes<float2, GL_MAX_A>(p), 16);
    l.smem = l.smem_state + ((size_t)s.N + A * s.N + A * K) * sizeof(float);
    return l;
}

// sum of w^2(z - i hop) over the frames 0 <= i <= last that cover sample z of the untrimmed signal, in ascending i
__device__ __forceinline__ float window_sumsquare(const float* __restrict__ w, int N, int hop, int z, int last) {
    const int i0 = z - N + 1 <= 0 ? 0 : (z - N + 1 + hop - 1) / hop;
    const int i1 = min(z / hop, last);
    float s = 0.f;
    for (int i = i0; i <= i1; ++i) {
        const float v = w[z - i * hop];
        s = fmaf(v, v, s);
    }
    return s;
}

// Frame f of the FFT buffer (frame j = j0 + f, f < nfr) <- w * p_j: p_j = (c + the overlap-add of the estimates of frames [m, upto)) / e
// over the frame's span, 0 where the one-sided envelope e is 0.
__device__ __forceinline__ void gl_fill(const FftSmem<float2>& sm, const FftPlan& p, int hop, int A, int m, int j0, int nfr, int upto,
                                        const float* c, const float* x) {
    const int N = p.N, ld = p.M + 1;
    const int open_end = m * hop + N;                               // c is zero from here on
    for (int i = threadIdx.x; i < nfr * N; i += blockDim.x) {
        const int f = i / N, n = i - f * N;
        const int z = (j0 + f) * hop + n;
        float acc = z < open_end ? c[z % N] : 0.f;
        for (int q = m; q < upto; ++q) {
            const int d = z - q * hop;
            if (d >= 0 && d < N) acc += x[(q % A) * N + d];
        }
        const float e = window_sumsquare(sm.window, N, hop, z, INT_MAX);
        reinterpret_cast<float*>(sm.buf + f * ld)[n] = sm.window[n] * (e != 0.f ? acc / e : 0.f);
    }
    __syncthreads();
}

// The frames filled by gl_fill -> x_j = w * irfft(S_j X / |X|) with X = rfft(frame) (phase 1 where X = 0; numpy irfft: 1/N, the imaginary
// parts of the DC and Nyquist bins ignored), into the estimate ring.
__device__ __forceinline__ void gl_project(const FftSmem<float2>& sm, const FftPlan& p, int A, int j0, int nfr, const float* Sr, float* x) {
    const int M = p.M, N = p.N, K = M + 1, ld = M + 1;
    float2* Z = sm.buf;
    float2* W = sm.buf + GL_MAX_A * ld;
    float2* r = block_cfft(Z, W, ld, nfr, p, sm.twM, false);
    float2* o = r == Z ? W : Z;
    for (int i = threadIdx.x; i < nfr * K; i += blockDim.x) {
        const int f = i / K, k = i - f * K;
        const float2 u = r[f * ld + (k == M ? 0 : k)], v = r[f * ld + (k == 0 ? 0 : M - k)];
        const float2 ev = make_float2(u.x + v.x, u.y - v.y);
        const float2 od = make_float2(u.x - v.x, u.y + v.y);
        const float2 t = cmul(od, sm.twN[k]);
        const float2 X = make_float2(0.5f * (ev.x + t.y), 0.5f * (ev.y - t.x));   // (ev - i t) / 2
        const float mag = hypotf(X.x, X.y);
        const float2 ph = mag > 0.f ? make_float2(X.x / mag, X.y / mag) : make_float2(1.f, 0.f);
        const float s = Sr[((j0 + f) % A) * K + k];
        o[f * ld + k] = make_float2(s * ph.x, (k == 0 || k == M) ? 0.f : s * ph.y);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nfr * M; i += blockDim.x) {
        const int f = i / M, k = i - f * M;
        const float2 u = o[f * ld + k], v = o[f * ld + M - k];
        const float2 ev = make_float2(u.x + v.x, u.y - v.y);          // Y[k] + conj(Y[M - k])
        const float2 od = make_float2(u.x - v.x, u.y + v.y);          // Y[k] - conj(Y[M - k])
        const float2 t = cmulc(od, sm.twN[k]);                        // * W_N^-k
        r[f * ld + k] = make_float2(ev.x - t.y, ev.y + t.x);          // ev + i t
    }
    __syncthreads();
    const float2* z = block_cfft(r, o, ld, nfr, p, sm.twM, true);
    const float scale = 1.f / (float)N;
    for (int i = threadIdx.x; i < nfr * N; i += blockDim.x) {
        const int f = i / N, n = i - f * N;
        const float2 v = z[f * ld + (n >> 1)];
        x[((j0 + f) % A) * N + n] = ((n & 1) ? v.y : v.x) * scale * sm.window[n];
    }
    __syncthreads();
}

__global__ void gl_stream_reset_kernel(int N, int win, float2* __restrict__ twM, float2* __restrict__ twN, float* __restrict__ window,
                                       unsigned char* __restrict__ slots, size_t slot_bytes, GlRows list) {
    fill_fft_tables(N, win, twM, twN, window);
    float4* s = reinterpret_cast<float4*>(slots + (size_t)list.r[blockIdx.x].slot * slot_bytes);
    for (size_t i = threadIdx.x; i < slot_bytes / sizeof(float4); i += blockDim.x) s[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

__global__ void __launch_bounds__(GL_THREADS) gl_stream_run_kernel(FftPlan p, int hop, int A, int iters, float a, GlRows rows,
                                                                   const float* __restrict__ S_new, float* __restrict__ wave,
                                                                   const float2* __restrict__ twM, const float2* __restrict__ twN,
                                                                   const float* __restrict__ window, unsigned char* __restrict__ slots,
                                                                   GlLayout l) {
    const FftSmem<float2> sm = load_tables<float2, GL_MAX_A>(p, twM, twN, window);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int N = p.N, K = p.M + 1;
    float* c = reinterpret_cast<float*>(smem_raw + l.smem_state);
    float* x = c + N;
    float* Sr = x + A * N;
    float* scratch = reinterpret_cast<float*>(sm.buf);

    const b200tts_gl_stream_row row = rows.r[blockIdx.x];
    unsigned char* slot = slots + (size_t)row.slot * l.slot_bytes;
    GlSlotHeader* hdr = reinterpret_cast<GlSlotHeader*>(slot);
    float* gc = reinterpret_cast<float*>(slot + l.c);
    float* gx = reinterpret_cast<float*>(slot + l.x);
    float* gS = reinterpret_cast<float*>(slot + l.S);
    const GlSlotHeader h = *hdr;
    for (int i = threadIdx.x; i < N; i += blockDim.x) c[i] = gc[i];
    for (int i = threadIdx.x; i < A * N; i += blockDim.x) x[i] = gx[i];
    for (int i = threadIdx.x; i < A * K; i += blockDim.x) Sr[i] = gS[i];
    __syncthreads();

    const int F = row.frames, fr = h.frames;
    const float* Sn = S_new + row.s_off * K;                        // frame j >= fr at row j - fr (only read when F > fr)
    int m = h.committed, adm = h.admitted;
    float carry = h.carry;
    int rel = max(0, m * hop - N / 2);                               // output samples released so far
    int out = 0;                                                     // of them in this call
    for (;;) {
        const bool process = m < F && (m + A - 1 < F || row.ended);
        // with lookahead 0 the last frame can be committed before the end is known: the call that learns of the end releases the rest
        const bool tail = !process && row.ended && m == F && rel < hop * (F - 1);
        if (!process && !tail) break;
        const int lf = process ? m : F - 1;                          // the released samples lie under frames 0..lf only
        const int base = lf * hop;
        if (process) {
            const int last = std::min(m + A - 1, F - 1);
            // admit the frames up to `last` one at a time, then `iters` Jacobi iterations over the whole look-ahead set [m, adm)
            for (int it = 0; adm <= last || it < iters;) {
                const bool admit = adm <= last;
                if (admit && adm >= fr)
                    for (int k = threadIdx.x; k < K; k += blockDim.x) Sr[(adm % A) * K + k] = Sn[(size_t)(adm - fr) * K + k];
                const int j0 = admit ? adm : m, nfr = admit ? 1 : adm - m;
                gl_fill(sm, p, hop, A, m, j0, nfr, adm, c, x);
                gl_project(sm, p, A, j0, nfr, Sr, x);
                if (admit) ++adm; else ++it;
            }
            for (int n = threadIdx.x; n < N; n += blockDim.x) c[(base + n) % N] += x[(m % A) * N + n];   // commit
            __syncthreads();
        }
        const bool final = row.ended && lf == F - 1;                 // release
        const int rel_end = final ? hop * (F - 1) : max(0, base + hop - N / 2);
        // stride over the offset within the span: rel + q + blockDim.x would overflow int for a stream near the 2^31 sample limit
        for (int q = threadIdx.x; q < rel_end - rel; q += blockDim.x) {
            const int z = rel + q + N / 2;
            const float v = c[z % N];
            const float wss = window_sumsquare(sm.window, N, hop, z, lf);
            scratch[q] = wss > FLT_MIN ? v / wss : v;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            float* y = wave + row.wave_off + out;
            for (int q = 0; q < rel_end - rel; ++q) {
                float v = scratch[q];
                if (a != 0.f) v = fmaf(a, carry, v);
                carry = v;
                y[q] = v;
            }
        }
        if (process && !final)                                       // the released span's ring entries start the next frame's tail
            for (int n = threadIdx.x; n < hop; n += blockDim.x) c[(base + n) % N] = 0.f;
        out += rel_end - rel;
        rel = rel_end;
        __syncthreads();
        if (process) ++m;
    }
    for (int j = std::max(adm, fr); j < F; ++j)                      // frames received but not yet admitted
        for (int k = threadIdx.x; k < K; k += blockDim.x) Sr[(j % A) * K + k] = Sn[(size_t)(j - fr) * K + k];
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) gc[i] = c[i];
    for (int i = threadIdx.x; i < A * N; i += blockDim.x) gx[i] = x[i];
    for (int i = threadIdx.x; i < A * K; i += blockDim.x) gS[i] = Sr[i];
    if (threadIdx.x == 0) *hdr = GlSlotHeader{m, adm, F, carry};
}

}  // namespace

static int gl_stream_validate(const b200tts_gl_stream_shape& s, FftPlan* p) {
    B200_REQUIRE(make_plan(s.N, p), "gl_stream: unsupported FFT size N = %d (even, <= 2048, N/2 with prime factors <= 31 only)", s.N);
    B200_REQUIRE(s.win >= 1 && s.win <= s.N, "gl_stream: window length %d must be in [1, N = %d]", s.win, s.N);
    B200_REQUIRE(s.hop >= 1 && s.hop <= s.win, "gl_stream: hop %d must be in [1, win = %d]", s.hop, s.win);
    B200_REQUIRE(s.lookahead >= 0 && s.lookahead <= B200TTS_GL_STREAM_MAX_LOOKAHEAD, "gl_stream: lookahead %d must be in [0, %d]", s.lookahead,
                 B200TTS_GL_STREAM_MAX_LOOKAHEAD);
    // without look-ahead a frame's samples below (m + 1) hop are released before the length is known: they must lie in the output range
    B200_REQUIRE(s.lookahead >= 1 || 2 * s.hop <= s.N, "gl_stream: lookahead 0 needs hop %d <= N / 2 = %d", s.hop, s.N / 2);
    B200_REQUIRE(s.iters >= 1, "gl_stream: iters %d must be at least 1", s.iters);
    B200_REQUIRE(s.slots >= 1 && s.slots <= GL_MAX_ROWS, "gl_stream: slots %d must be in [1, %d]", s.slots, GL_MAX_ROWS);
    B200_REQUIRE(s.preemphasis > -1.f && s.preemphasis < 1.f, "gl_stream: preemphasis must lie in (-1, 1)");
    const GlLayout l = gl_layout(s, *p);
    B200_REQUIRE(l.smem <= GL_MAX_SMEM, "gl_stream: N = %d with lookahead %d needs %zu bytes of shared memory per stream, more than %zu", s.N,
                 s.lookahead, l.smem, GL_MAX_SMEM);
    return B200TTS_OK;
}

static int gl_check_workspace(const GlLayout& l, void* ws, size_t ws_bytes, const char* what) {
    B200_REQUIRE(ws && ws_bytes >= l.bytes, "%s: workspace of %zu bytes is smaller than the %zu required", what, ws_bytes, l.bytes);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "%s: workspace must be 256-byte aligned", what);
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_gl_stream_workspace_bytes(const b200tts_gl_stream_shape* shape) {
    if (!shape) { set_last_error("gl_stream_workspace_bytes: null shape"); return 0; }
    FftPlan p;
    if (gl_stream_validate(*shape, &p) != B200TTS_OK) return 0;
    return gl_layout(*shape, p).bytes;
}

int b200tts_gl_stream_reset(const b200tts_gl_stream_shape* shape, void* workspace, size_t workspace_bytes, const int32_t* slots, int count,
                            void* stream) {
    B200_REQUIRE(shape, "gl_stream_reset: null argument");
    const b200tts_gl_stream_shape& s = *shape;
    FftPlan p;
    B200_TRY(gl_stream_validate(s, &p));
    const GlLayout l = gl_layout(s, p);
    B200_TRY(gl_check_workspace(l, workspace, workspace_bytes, "gl_stream_reset"));
    B200_REQUIRE(slots && count >= 1 && count <= s.slots, "gl_stream_reset: need 1 to %d slots (got %d)", s.slots, count);
    unsigned long long seen = 0;
    for (int i = 0; i < count; ++i) {
        B200_REQUIRE(slots[i] >= 0 && slots[i] < s.slots, "gl_stream_reset: slot %d outside [0, %d)", slots[i], s.slots);
        B200_REQUIRE(!(seen >> slots[i] & 1), "gl_stream_reset: slot %d listed twice", slots[i]);
        seen |= 1ull << slots[i];
    }
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = static_cast<unsigned char*>(workspace);
    GlRows rows{};
    for (int i = 0; i < count; ++i) rows.r[i].slot = slots[i];
    KernelTimer kt("gl_stream_reset", st);
    gl_stream_reset_kernel<<<count, 256, 0, st>>>(s.N, s.win, reinterpret_cast<float2*>(base + l.twM), reinterpret_cast<float2*>(base + l.twN),
                                                  reinterpret_cast<float*>(base + l.window), base + l.slots, l.slot_bytes, rows);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_gl_stream_run(const b200tts_gl_stream_shape* shape, const b200tts_gl_stream_row* rows, int count, const float* S_new, float* wave,
                          void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && S_new && wave, "gl_stream_run: null argument");
    const b200tts_gl_stream_shape& s = *shape;
    FftPlan p;
    B200_TRY(gl_stream_validate(s, &p));
    const GlLayout l = gl_layout(s, p);
    B200_TRY(gl_check_workspace(l, workspace, workspace_bytes, "gl_stream_run"));
    B200_REQUIRE(rows && count >= 1 && count <= s.slots, "gl_stream_run: need 1 to %d rows (got %d)", s.slots, count);
    unsigned long long seen = 0;
    for (int i = 0; i < count; ++i) {
        const b200tts_gl_stream_row& r = rows[i];
        B200_REQUIRE(r.slot >= 0 && r.slot < s.slots, "gl_stream_run: row %d: slot %d outside [0, %d)", i, r.slot, s.slots);
        B200_REQUIRE(!(seen >> r.slot & 1), "gl_stream_run: slot %d listed twice", r.slot);
        seen |= 1ull << r.slot;
        B200_REQUIRE(r.frames >= 0 && r.s_off >= 0 && r.wave_off >= 0, "gl_stream_run: row %d: negative frames or offset", i);
        B200_REQUIRE(!r.ended || r.frames >= 2, "gl_stream_run: row %d: a stream ends with at least 2 frames (got %d)", i, r.frames);
        B200_REQUIRE((long long)s.hop * r.frames + 2ll * s.N < (1ll << 31), "gl_stream_run: row %d: stream too long (%d frames)", i, r.frames);
    }
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = static_cast<unsigned char*>(workspace);
    GlRows list{};
    for (int i = 0; i < count; ++i) list.r[i] = rows[i];
    B200_CUDA(cudaFuncSetAttribute(gl_stream_run_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l.smem));
    KernelTimer kt("gl_stream_run", st);
    gl_stream_run_kernel<<<count, GL_THREADS, l.smem, st>>>(p, s.hop, s.lookahead + 1, s.iters, s.preemphasis, list, S_new, wave,
                                                            reinterpret_cast<const float2*>(base + l.twM),
                                                            reinterpret_cast<const float2*>(base + l.twN),
                                                            reinterpret_cast<const float*>(base + l.window), base + l.slots, l);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
