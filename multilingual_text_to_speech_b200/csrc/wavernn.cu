// WaveRNN vocoder (fatchord architecture): mel -> waveform, one GRU step per audio sample.
//
//   * wavernn_upsample_layer_kernel: nearest stretch x s then the 1-channel FIR of 2s+1 taps with zero padding s (one up_layers pair of
//     the upsampling network), every layer but the last, per utterance;
//   * wavernn_fold_kernel: the last layer of the mel path evaluated at the positions a chunk of the sample loop needs, the `indent` cut, the
//     nearest stretch of the MelResNet output (aux) and fold_with_overlap, as the [steps, rows, n_mels + aux_dims] rows of the conditioning
//     GEMMs (the products that do not depend on the previous sample run in the library GEMM before the loop);
//   * wavernn_window_rows_kernel: the same rows for consecutive sample positions of unfolded rows, each read from its own windows of the
//     penultimate mel layer and of aux (streaming generation, where the mel arrives in chunks);
//   * wavernn_loop_kernel: the persistent sample loop, one cooperative launch per chunk of steps (below);
//   * wavernn_unfold_kernel: mu-law decode, the square-root cross-fades, overlap-add, the cut to (F - 1) hop samples and the linear fade-out.
//
// The sample loop.  128 CTAs of 256 threads; CTA c owns hidden units [c U, (c + 1) U) of both GRUs (U = rnn_dims / 128; the r, z and n rows
// of its units form one 16-row weight tile per GRU matrix), fc1 / fc2 outputs [c V, (c + 1) V) (V = fc_dims / 128) and fc3 outputs
// [c O, (c + 1) O) (O = ceil(n_out / 128)).  Its six bf16 tiles (W_hh1, the x part of W_ih2, W_hh2, the x parts of fc1 and fc2, fc3; 96 KB at
// rnn = fc = 512) stay in shared memory for the whole launch, fragment-major so that each lane fetches its mma.sync A fragment with one
// 16-byte load.  Activations travel between CTAs as bf16 rows in global memory (L2): every CTA multiplies its tiles by all fold rows, 8 rows
// per m16n8k16 N tile, N tiles spread over the 8 warps, fp32 accumulation.  The K dimension is permuted identically in both operands
// (lane t takes 8 consecutive elements per 32-element block), so a B fragment is one 16-byte load too.  One step of all rows:
//   1. h1 = GRU1(G1 + u1 prev, W_hh1 h1 + b_hh1);  x1 = c + w prev + h1
//   2. h2 = GRU2(W_ih2x x1 + C2, W_hh2 h2 + b_hh2);  x2 = x1 + h2
//   3. y1 = relu(fc1x x2 + P1)     4. y2 = relu(fc2x y1 + P2)     5. logits = fc3 y2 + b3
//   6. one warp per row samples from its logits (fixed-order reductions) and writes the row's next input
// with a grid barrier after each stage: six per sample.  h1 and h2 are double-buffered by step parity (stage 1 / 2 of step t reads the
// previous step's rows while owners write this step's).  fp32 state (h1, h2, x1, prev) is only read by its owner.
#include <cuda_bf16.h>
#include <climits>
#include <math.h>
#include "decoder_internal.cuh"
#include "tc_ptx.cuh"

namespace b200tts {

namespace {

using namespace tcx;

constexpr int WR_CTAS = 128;
constexpr int WR_THREADS = 256;
constexpr int WR_WARPS = WR_THREADS / 32;
constexpr int WR_MATS = 6;

__device__ __forceinline__ __nv_bfloat16 bf(float v) { return __float2bfloat16_rn(v); }

// ---- upsampling ----
// out[c, i] = sum_{k=-s..s} w[k + s] in[c, (i + k) / s] over 0 <= i + k < len s (zero padding), i in [0, len s)
__global__ void wavernn_upsample_layer_kernel(int C, int len, int s, const float* __restrict__ w, const float* __restrict__ in,
                                              float* __restrict__ out) {
    const long long n = (long long)C * len * s;
    const int lo = len * s;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx / lo), i = (int)(idx - (long long)c * lo);
        const float* x = in + (size_t)c * len;
        float acc = 0.f;
        for (int k = -s; k <= s; ++k) {
            const int j = i + k;
            if (j >= 0 && j < lo) acc = fmaf(w[k + s], x[j / s], acc);
        }
        out[idx] = acc;
    }
}

// wavernn_upsample_layer_kernel over packed segments: segment g is [C, len_g] at in + in_off[g] and [C, len_g s] at out + s in_off[g]
struct WrSegments { int n, C; long long in_off[B200TTS_WAVERNN_MAX_STREAMS + 1]; int len[B200TTS_WAVERNN_MAX_STREAMS]; };
__global__ void wavernn_upsample_segments_kernel(const __grid_constant__ WrSegments g, int s, const float* __restrict__ w,
                                                 const float* __restrict__ in, float* __restrict__ out) {
    const long long n = g.in_off[g.n] * s;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        int lo_g = 0, hi_g = g.n - 1;
        while (lo_g < hi_g) {
            const int mid = (lo_g + hi_g + 1) >> 1;
            if (g.in_off[mid] * s <= idx) lo_g = mid; else hi_g = mid - 1;
        }
        const int len = g.len[lo_g], lo = len * s;
        const long long e = idx - g.in_off[lo_g] * s;
        const int c = (int)(e / lo), i = (int)(e - (long long)c * lo);
        const float* x = in + g.in_off[lo_g] + (size_t)c * len;
        float acc = 0.f;
        for (int k = -s; k <= s; ++k) {
            const int j = i + k;
            if (j >= 0 && j < lo) acc = fmaf(w[k + s], x[j / s], acc);
        }
        out[idx] = acc;
    }
}

// feat[i, r, :] for loop steps t0 + i of fold row r: the row's utterance b and fold f give the sample position q = f (target + overlap) +
// t0 + i of the utterance's F hop positions (zero beyond them: the tail padding of fold_with_overlap).  Columns [0, n_mels): the last mel
// layer at the uncut position q + pad hop; columns [n_mels, n_mels + aux_dims): aux[b, q / hop, :].
__global__ void wavernn_fold_kernel(b200tts_wavernn_fold_shape s, const float* __restrict__ mel_up, const long long* __restrict__ mel_off,
                                    const int* __restrict__ frames, const int* __restrict__ row_utt, const int* __restrict__ row_fold,
                                    const float* __restrict__ fir, const float* __restrict__ aux, int t0, int nsteps, float* __restrict__ feat) {
    const int D = s.n_mels + s.aux_dims;
    const long long n = (long long)nsteps * s.rows * D;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(idx % D);
        const long long ir = idx / D;
        const int r = (int)(ir % s.rows), i = (int)(ir / s.rows);
        const int b = row_utt[r], F = frames[b];
        const long long q = (long long)row_fold[r] * (s.target + s.overlap) + t0 + i;
        float v = 0.f;
        if (q < (long long)F * s.hop) {
            if (col < s.n_mels) {
                const int len = (F + 2 * s.pad) * s.hop / s.scale;       // samples of the penultimate layer
                const int lo = len * s.scale;
                const float* x = mel_up + mel_off[b] + (size_t)col * len;
                const int p = (int)q + s.pad * s.hop;
                float acc = 0.f;
                for (int k = -s.scale; k <= s.scale; ++k) {
                    const int j = p + k;
                    if (j >= 0 && j < lo) acc = fmaf(fir[k + s.scale], x[j / s.scale], acc);
                }
                v = acc;
            } else {
                v = aux[((size_t)b * s.max_frames + q / s.hop) * s.aux_dims + (col - s.n_mels)];
            }
        }
        feat[idx] = v;
    }
}

// feat[i, r, :] for the sample positions q = s0 + i (i < n, zero past it) of unfolded row r (zero for q >= F hop once F is known):
// wavernn_fold_kernel's arithmetic, with the penultimate layer read from the row's window mel + mel_off [n_mels, mel_len] that holds its
// samples [m0, m0 + mel_len), and aux from its window aux + aux_off [aux_len, aux_dims] that holds frames [a0, a0 + aux_len).  lo bounds the
// whole last layer ((F + 2 pad) hop, or past every read while F is unknown); the host checks that every read falls inside the windows.
struct WrWinRow { long long s0, m0, lo, mel_off, aux_off; int n, frames, mel_len, a0; };
struct WrWinRows { WrWinRow r[B200TTS_WAVERNN_MAX_STREAMS]; };
__global__ void wavernn_window_rows_kernel(int n_mels, int aux_dims, int hop, int pad, int scale, int rows, const __grid_constant__ WrWinRows w,
                                           const float* __restrict__ mel, const float* __restrict__ fir, const float* __restrict__ aux,
                                           int nsteps, float* __restrict__ feat) {
    const int D = n_mels + aux_dims;
    const long long n = (long long)nsteps * rows * D;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(idx % D);
        const long long ir = idx / D;
        const int r = (int)(ir % rows), i = (int)(ir / rows);
        const WrWinRow& s = w.r[r];
        const long long q = s.s0 + i;
        float v = 0.f;
        if (i < s.n && (s.frames == 0 || q < (long long)s.frames * hop)) {
            if (col < n_mels) {
                const float* xc = mel + s.mel_off + (size_t)col * s.mel_len;
                const long long p = q + (long long)pad * hop;
                float acc = 0.f;
                for (int k = -scale; k <= scale; ++k) {
                    const long long j = p + k;
                    if (j >= 0 && j < s.lo) acc = fmaf(fir[k + scale], xc[j / scale - s.m0], acc);
                }
                v = acc;
            } else {
                v = aux[s.aux_off + (size_t)(q / hop - s.a0) * aux_dims + (col - n_mels)];
            }
        }
        feat[idx] = v;
    }
}

// ---- the sample loop ----
struct WrDims {
    int R, Fc, n_out, U, V, O;
    int K[WR_MATS];       // inner dimension of each tile
    int off[WR_MATS];     // uint4 offset of each tile inside one CTA's packed block
    int per_cta;          // uint4 per CTA
};
__host__ __device__ inline WrDims wr_dims(int R, int Fc, int n_out) {
    WrDims d;
    d.R = R; d.Fc = Fc; d.n_out = n_out;
    d.U = R / WR_CTAS; d.V = Fc / WR_CTAS; d.O = (n_out + WR_CTAS - 1) / WR_CTAS;
    const int K[WR_MATS] = {R, R, R, R, Fc, Fc};
    int o = 0;
    for (int m = 0; m < WR_MATS; ++m) { d.K[m] = K[m]; d.off[m] = o; o += 2 * K[m]; }    // 16 rows x K bf16 = 2 K uint4
    d.per_cta = o;
    return d;
}

// weight row of tile row i of matrix m in CTA c (-1: zero row)
__host__ __device__ inline int wr_tile_row(const WrDims& d, int m, int c, int i) {
    if (m <= 2) return i < 3 * d.U ? (i / d.U) * d.R + c * d.U + i % d.U : -1;
    if (m <= 4) return i < d.V ? c * d.V + i : -1;
    const int o = c * d.O + i;
    return (i < d.O && o < d.n_out) ? o : -1;
}

struct WrWeights { const float* w[WR_MATS]; };

// packed[c][tile m][kb][s][lane] = {W[g][kk..kk+1], W[g+8][kk..kk+1], W[g][kk+2..kk+3], W[g+8][kk+2..kk+3]}, kk = 32 kb + 8 t + 4 s
__global__ void wavernn_pack_kernel(WrDims d, WrWeights W, uint4* __restrict__ packed) {
    const long long n = (long long)WR_CTAS * d.per_cta;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx / d.per_cta), j = (int)(idx % d.per_cta);
        int m = WR_MATS - 1;
        while (d.off[m] > j) --m;
        const int e = j - d.off[m];
        const int lane = e & 31, s = (e >> 5) & 1, kb = e >> 6;
        const int g = lane >> 2, t = lane & 3, kk = kb * 32 + 8 * t + 4 * s, K = d.K[m];
        const int r0 = wr_tile_row(d, m, c, g), r1 = wr_tile_row(d, m, c, g + 8);
        auto at = [&](int r, int k) { return r < 0 ? 0.f : W.w[m][(size_t)r * K + k]; };
        uint4 v;
        v.x = pack2(at(r0, kk), at(r0, kk + 1));
        v.y = pack2(at(r1, kk), at(r1, kk + 1));
        v.z = pack2(at(r0, kk + 2), at(r0, kk + 3));
        v.w = pack2(at(r1, kk + 2), at(r1, kk + 3));
        packed[idx] = v;
    }
}

struct WrLoopArgs {
    WrDims d;
    int rows, mode, L, t0, nsteps;
    int io0;              // step of uniforms / out column 0: 0 for a fold, t0 for a stream call (whose columns are its own steps)
    const uint4* packed;
    const float *b_hh1, *u1, *w_prev, *b_hh2, *b_fc3;
    const float *cc, *g1, *c2, *p1, *p2;
    const float* uni;
    float* out;
    float* dbg;
    float *h1, *h2, *x1, *prev, *logits;
    __nv_bfloat16 *h1b, *h2b, *x1b, *x2b, *y1b, *y2b;     // h1b / h2b: two slots of [rows, R]
    unsigned* bar;
    int* abort_flag;
    // ragged instantiation only: row r runs its steps i < row_n[r] with h1 / h2 slot parity (row_t[r] + i) & 1; rows = the active rows,
    // slot = the elements of one h1b / h2b slot (the workspace's rows x R)
    const long long* row_t;
    const int* row_n;
    size_t slot;
};

// acc (16 x 8 tile: weight rows x fold rows row0..row0+7) = tile . act[row0 + n, 0:K]^T
__device__ __forceinline__ void wr_mma(float (&acc)[4], const uint4* __restrict__ tile, const __nv_bfloat16* act, int K, int row0, int rows,
                                       int lane) {
    acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
    const int r = row0 + (lane >> 2), t = lane & 3;
    const bool ok = r < rows;
    const uint4* ap = reinterpret_cast<const uint4*>(act + (size_t)(ok ? r : 0) * K) + t;
    const int nkb = K / 32;
#pragma unroll 4
    for (int kb = 0; kb < nkb; ++kb) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if (ok) v = __ldcg(ap + kb * 4);
        const uint4 a0 = tile[(kb * 2) * 32 + lane], a1 = tile[(kb * 2 + 1) * 32 + lane];
        const uint32_t f0[4] = {a0.x, a0.y, a0.z, a0.w}, f1[4] = {a1.x, a1.y, a1.z, a1.w};
        mma_bf16(acc, f0, v.x, v.y);
        mma_bf16(acc, f1, v.z, v.w);
    }
}
// the 16 x 8 accumulator tile into the warp's shared scratch [16][8]
__device__ __forceinline__ void wr_spill(float* ep, const float (&acc)[4], int lane) {
    const int g = lane >> 2, t = lane & 3;
    ep[g * 8 + 2 * t] = acc[0];
    ep[g * 8 + 2 * t + 1] = acc[1];
    ep[(g + 8) * 8 + 2 * t] = acc[2];
    ep[(g + 8) * 8 + 2 * t + 1] = acc[3];
    __syncwarp();
}

__device__ __forceinline__ float gru_cell(float gir, float giz, float gin, float ghr, float ghz, float ghn, float h) {
    const float r = sigmoidf_acc(gir + ghr), z = sigmoidf_acc(giz + ghz);
    const float nn = tanhf(fmaf(r, ghn, gin));
    return fmaf(z, h - nn, nn);       // (1 - z) n + z h
}

// RAGGED = false: every row runs steps [t0, t0 + nsteps) (wavernn_run / _run_stream).  RAGGED = true: each row runs its own budget of this
// call's nsteps from its own step count (wavernn_run_rows); a row past its budget writes nothing.
template <bool RAGGED>
__global__ void __launch_bounds__(WR_THREADS, 1) wavernn_loop_kernel(WrLoopArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ float s_ep[WR_WARPS][2][16 * 8];
    __shared__ int s_ok;
    const WrDims& d = a.d;
    uint4* wt = reinterpret_cast<uint4*>(smem_raw);
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    {
        const uint4* src = a.packed + (size_t)c * d.per_cta;
        for (int i = threadIdx.x; i < d.per_cta; i += WR_THREADS) wt[i] = src[i];
    }
    __syncthreads();
    const int R = d.R, Fc = d.Fc, rows = a.rows, ntiles = (rows + 7) / 8;
    const int Ddbg = 4 * R + 2 * Fc + d.n_out;
    const int U = d.U, V = d.V, O = d.O;
    float* ep0 = s_ep[warp][0];
    float* ep1 = s_ep[warp][1];
    unsigned target = 0;

    for (int i = 0; i < a.nsteps; ++i) {
        const int tg = a.t0 + i, ti = RAGGED ? i : tg - a.io0;
        const int cur = tg & 1, prv = cur ^ 1;
        // ragged: the previous step's h1b / h2b slot of this lane's operand row (wr_mma reads row nt * 8 + lane / 4), by the row's own parity
        auto prv_slot = [&](const __nv_bfloat16* base, int nt) {
            const int r = nt * 8 + (lane >> 2);
            return r < rows ? base + (size_t)(((a.row_t[r] + i) & 1) ^ 1) * a.slot : base;
        };
        float* dbg = a.dbg ? a.dbg + (size_t)i * rows * Ddbg : nullptr;
        // 1. GRU1
        for (int nt = warp; nt < ntiles; nt += WR_WARPS) {
            float acc[4];
            if constexpr (RAGGED) wr_mma(acc, wt + d.off[0], prv_slot(a.h1b, nt), R, nt * 8, rows, lane);
            else wr_mma(acc, wt + d.off[0], a.h1b + (size_t)prv * rows * R, R, nt * 8, rows, lane);
            wr_spill(ep0, acc, lane);
            for (int e = lane; e < U * 8; e += 32) {
                const int j = e >> 3, n = e & 7, row = nt * 8 + n, u = c * U + j;
                if (row < rows && (!RAGGED || i < a.row_n[row])) {
                    const float p = __ldcg(a.prev + row);
                    const float* g1 = a.g1 + ((size_t)i * rows + row) * 3 * R;
                    const float gir = fmaf(a.u1[u], p, g1[u]), giz = fmaf(a.u1[R + u], p, g1[R + u]), gin = fmaf(a.u1[2 * R + u], p, g1[2 * R + u]);
                    const float ghr = ep0[j * 8 + n] + a.b_hh1[u], ghz = ep0[(U + j) * 8 + n] + a.b_hh1[R + u],
                                ghn = ep0[(2 * U + j) * 8 + n] + a.b_hh1[2 * R + u];
                    const size_t o = (size_t)row * R + u;
                    const float h = gru_cell(gir, giz, gin, ghr, ghz, ghn, a.h1[o]);
                    const float x = fmaf(a.w_prev[u], p, a.cc[((size_t)i * rows + row) * R + u]) + h;
                    const __nv_bfloat16 xb = bf(x);
                    a.h1[o] = h;
                    if constexpr (RAGGED) a.h1b[(size_t)((a.row_t[row] + i) & 1) * a.slot + o] = bf(h);
                    else a.h1b[(size_t)cur * rows * R + o] = bf(h);
                    a.x1[o] = x;
                    a.x1b[o] = xb;
                    if (dbg) { float* q = dbg + (size_t)row * Ddbg; q[u] = h; q[R + u] = __bfloat162float(xb); }
                }
            }
            __syncwarp();
        }
        if (!grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
        // 2. GRU2
        for (int nt = warp; nt < ntiles; nt += WR_WARPS) {
            float acc[4];
            wr_mma(acc, wt + d.off[1], a.x1b, R, nt * 8, rows, lane);
            wr_spill(ep0, acc, lane);
            if constexpr (RAGGED) wr_mma(acc, wt + d.off[2], prv_slot(a.h2b, nt), R, nt * 8, rows, lane);
            else wr_mma(acc, wt + d.off[2], a.h2b + (size_t)prv * rows * R, R, nt * 8, rows, lane);
            wr_spill(ep1, acc, lane);
            for (int e = lane; e < U * 8; e += 32) {
                const int j = e >> 3, n = e & 7, row = nt * 8 + n, u = c * U + j;
                if (row < rows && (!RAGGED || i < a.row_n[row])) {
                    const float* c2 = a.c2 + ((size_t)i * rows + row) * 3 * R;
                    const float gir = ep0[j * 8 + n] + c2[u], giz = ep0[(U + j) * 8 + n] + c2[R + u], gin = ep0[(2 * U + j) * 8 + n] + c2[2 * R + u];
                    const float ghr = ep1[j * 8 + n] + a.b_hh2[u], ghz = ep1[(U + j) * 8 + n] + a.b_hh2[R + u],
                                ghn = ep1[(2 * U + j) * 8 + n] + a.b_hh2[2 * R + u];
                    const size_t o = (size_t)row * R + u;
                    const float h = gru_cell(gir, giz, gin, ghr, ghz, ghn, a.h2[o]);
                    const __nv_bfloat16 xb = bf(a.x1[o] + h);
                    a.h2[o] = h;
                    if constexpr (RAGGED) a.h2b[(size_t)((a.row_t[row] + i) & 1) * a.slot + o] = bf(h);
                    else a.h2b[(size_t)cur * rows * R + o] = bf(h);
                    a.x2b[o] = xb;
                    if (dbg) { float* q = dbg + (size_t)row * Ddbg; q[2 * R + u] = h; q[3 * R + u] = __bfloat162float(xb); }
                }
            }
            __syncwarp();
        }
        if (!grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
        // 3. / 4. fc1, fc2
        for (int st = 0; st < 2; ++st) {
            const __nv_bfloat16* in = st == 0 ? a.x2b : a.y1b;
            __nv_bfloat16* outb = st == 0 ? a.y1b : a.y2b;
            const float* P = st == 0 ? a.p1 : a.p2;
            const int K = st == 0 ? R : Fc;
            for (int nt = warp; nt < ntiles; nt += WR_WARPS) {
                float acc[4];
                wr_mma(acc, wt + d.off[3 + st], in, K, nt * 8, rows, lane);
                wr_spill(ep0, acc, lane);
                for (int e = lane; e < V * 8; e += 32) {
                    const int j = e >> 3, n = e & 7, row = nt * 8 + n, o = c * V + j;
                    if (row < rows && (!RAGGED || i < a.row_n[row])) {
                        const __nv_bfloat16 yb = bf(fmaxf(ep0[j * 8 + n] + P[((size_t)i * rows + row) * Fc + o], 0.f));
                        outb[(size_t)row * Fc + o] = yb;
                        if (dbg) dbg[(size_t)row * Ddbg + 4 * R + st * Fc + o] = __bfloat162float(yb);
                    }
                }
                __syncwarp();
            }
            if (!grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
        }
        // 5. fc3
        if (c * O < d.n_out) {
            for (int nt = warp; nt < ntiles; nt += WR_WARPS) {
                float acc[4];
                wr_mma(acc, wt + d.off[5], a.y2b, Fc, nt * 8, rows, lane);
                wr_spill(ep0, acc, lane);
                for (int e = lane; e < O * 8; e += 32) {
                    const int j = e >> 3, n = e & 7, row = nt * 8 + n, o = c * O + j;
                    if (row < rows && o < d.n_out && (!RAGGED || i < a.row_n[row])) {
                        const float l = ep0[j * 8 + n] + a.b_fc3[o];
                        a.logits[(size_t)row * d.n_out + o] = l;
                        if (dbg) dbg[(size_t)row * Ddbg + 4 * R + 2 * Fc + o] = l;
                    }
                }
                __syncwarp();
            }
        }
        if (!grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
        // 6. sample, one warp per row
        for (int row = c * WR_WARPS + warp; row < rows; row += WR_CTAS * WR_WARPS) {
            if (RAGGED && i >= a.row_n[row]) continue;
            const float* lg = a.logits + (size_t)row * d.n_out;
            float sample;
            if (a.mode == B200TTS_WAVERNN_RAW) {
                const int n = d.n_out, per = (n + 31) / 32, k0 = lane * per, k1 = min(n, k0 + per);
                const float u = a.uni[(size_t)row * a.L + ti];
                float mx = -INFINITY;
                for (int k = k0; k < k1; ++k) mx = fmaxf(mx, __ldcg(lg + k));
                mx = warp_max(mx);
                float part = 0.f;
                for (int k = k0; k < k1; ++k) part += expf(__ldcg(lg + k) - mx);
                float incl = part;                                // inclusive scan over lanes, fixed order
                for (int o = 1; o < 32; o <<= 1) {
                    const float v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                const float total = __shfl_sync(0xffffffffu, incl, 31);
                const float thr = u * total;
                const unsigned hit = __ballot_sync(0xffffffffu, incl > thr && k1 > k0);
                int k = n - 1;                                    // rounding put u S at or beyond the last partial sum: the last class
                if (hit) {
                    const int src = __ffs(hit) - 1;
                    int kk = k1 - 1;
                    if (lane == src) {
                        float cum = incl - part;
                        for (int q = k0; q < k1; ++q) {
                            cum += expf(__ldcg(lg + q) - mx);
                            if (cum > thr) { kk = q; break; }
                        }
                    }
                    k = __shfl_sync(0xffffffffu, kk, src);
                }
                sample = 2.f * (float)k / (float)(n - 1) - 1.f;
            } else {
                const int nr = d.n_out / 3, U1 = nr + 1;
                const float* uu = a.uni + ((size_t)row * a.L + ti) * U1;
                // bi starts as a valid component on every lane and only ever takes another lane's bi: it stays in [0, nr) even when
                // NaN scores make every comparison false, so the loads below stay inside the row's logits
                float best = -INFINITY;
                int bi = 0;
                if (lane < nr) {
                    const float u = fmaf(1.f - 2e-5f, uu[lane], 1e-5f);
                    best = __ldcg(lg + lane) - logf(-logf(u));
                    bi = lane;
                }
                for (int o = 16; o > 0; o >>= 1) {             // argmax, the lowest index among equal values
                    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
                }
                const float mean = __ldcg(lg + nr + bi);
                const float ls = fmaxf(__ldcg(lg + 2 * nr + bi), -32.23619130191664f);   // log(1e-14)
                const float u = fmaf(1.f - 2e-5f, uu[nr], 1e-5f);
                sample = fminf(fmaxf(mean + expf(ls) * (logf(u) - logf(1.f - u)), -1.f), 1.f);
            }
            if (lane == 0) {
                a.prev[row] = sample;
                a.out[(size_t)row * a.L + ti] = sample;
            }
        }
        if (!grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
    }
}

// zero the recurrent state of the listed rows: h1, h2, both slots of h1b / h2b, the previous sample
struct WrRowList { int n; int row[B200TTS_WAVERNN_MAX_STREAMS]; };
__global__ void wavernn_reset_rows_kernel(const __grid_constant__ WrRowList l, int rows, int R, float* __restrict__ h1, float* __restrict__ h2,
                                          float* __restrict__ prev, __nv_bfloat16* __restrict__ h1b, __nv_bfloat16* __restrict__ h2b) {
    const long long n = (long long)l.n * R;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(idx / R), u = (int)(idx % R);
        const size_t o = (size_t)l.row[k] * R + u, slot = (size_t)rows * R;
        h1[o] = 0.f;
        h2[o] = 0.f;
        h1b[o] = h1b[slot + o] = h2b[o] = h2b[slot + o] = __float2bfloat16_rn(0.f);
        if (u == 0) prev[l.row[k]] = 0.f;
    }
}

// element k of numpy.linspace(-1, 1, n): k * step + start, the last one exactly 1
__device__ __forceinline__ double linspace_pm1(long long k, int n) {
    if (n == 1) return -1.0;
    return k == n - 1 ? 1.0 : (double)k * (2.0 / (n - 1)) + -1.0;
}

// The per-sample arithmetic of the unfold, shared by wavernn_unfold_kernel and wavernn_unfold_streams_kernel: acc += fold sample v at fold
// position j in [0, L), mu-law decoded (mu > 0), times the square-root cross-fade (sil = overlap / 2, fl = overlap - sil).  The product and
// the sum are one expression, as the compiler contracts them.
__device__ __forceinline__ void unfold_add(double& acc, double v, long long j, int L, int overlap, int sil, int fl, int mu) {
    if (mu > 0) v = (v > 0 ? 1.0 : (v < 0 ? -1.0 : 0.0)) / mu * (pow(1.0 + mu, fabs(v)) - 1.0);
    double w = 1.0;
    if (j < overlap) w = j < sil ? 0.0 : sqrt(0.5 * (1.0 + linspace_pm1(j - sil, fl)));
    else if (j >= L - overlap) {
        const long long k = j - (L - overlap);
        w = k >= fl ? 0.0 : sqrt(0.5 * (1.0 - linspace_pm1(k, fl)));
    }
    acc += v * w;
}

// the linear fade-out over the fo = 20 hop samples before the cut: k = position - (cut - fo)
__device__ __forceinline__ double unfold_fade_out(double acc, long long k, int fo) {
    if (k >= 0) acc *= (k == fo - 1) ? 0.0 : 1.0 + k * (-1.0 / (fo - 1));
    return acc;
}

// wave of utterance b (packed at wave_off[b], (F_b - 1) hop samples): sample i sums, over the folds f of the utterance in ascending order,
// fade(j) y[f, j] with j = i - f (target + overlap) in [0, L); mu-law decoded first (RAW); times the final linear fade-out.  fp64, then fp32.
__global__ void wavernn_unfold_kernel(int B, int hop, int target, int overlap, int mu, const int* __restrict__ frames,
                                      const int* __restrict__ row_off, const long long* __restrict__ wave_off, const float* __restrict__ y,
                                      float* __restrict__ wave, long long total) {
    const int L = target + 2 * overlap, sil = overlap / 2, fl = overlap - sil, fo = 20 * hop;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = B - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (wave_off[mid] <= idx) lo = mid; else hi = mid - 1;
        }
        const int b = lo;
        const long long i = idx - wave_off[b];
        const long long len = (long long)(frames[b] - 1) * hop;
        const int r0 = row_off[b], nf = row_off[b + 1] - r0;
        double acc = 0.0;
        for (int f = 0; f < nf; ++f) {
            const long long j = i - (long long)f * (target + overlap);
            if (j < 0 || j >= L) continue;
            unfold_add(acc, y[(size_t)(r0 + f) * L + j], j, L, overlap, sil, fl, mu);
        }
        wave[idx] = (float)unfold_fade_out(acc, i - (len - fo), fo);
    }
}

struct WrUnfoldStreams {
    int n;
    b200tts_wavernn_unfold_stream s[B200TTS_WAVERNN_MAX_STREAMS];
};

// wave[s.wave_off + q - s.q0] for q in [s.q0, s.q1) of every stream s: wavernn_unfold_kernel's sum over the folds f covering q, in ascending
// order, of fold f's sample at j = q - f (target + overlap), read from y[base[e] + j mod period[e]] (e = s.src + f - s.fold0; an absent
// fold, base < 0, adds nothing); then the fade-out before (F - 1) hop when F = s.frames is known.  One thread per output sample.
__global__ void wavernn_unfold_streams_kernel(WrUnfoldStreams g, int hop, int target, int overlap, int mu, const long long* __restrict__ base,
                                              const int* __restrict__ period, const float* __restrict__ y, float* __restrict__ wave,
                                              long long total) {
    const int L = target + 2 * overlap, sil = overlap / 2, fl = overlap - sil, fo = 20 * hop, step = target + overlap;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = g.n - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (g.s[mid].wave_off <= idx) lo = mid; else hi = mid - 1;
        }
        const b200tts_wavernn_unfold_stream& s = g.s[lo];
        const long long q = s.q0 + (idx - s.wave_off);
        // folds covering q: f step <= q < f step + L
        const long long f_hi = q / step, f_lo = q >= L ? (q - L) / step + 1 : 0;
        double acc = 0.0;
        for (long long f = f_lo; f <= f_hi; ++f) {
            const int e = s.src + (int)(f - s.fold0);
            const long long b = base[e];
            if (b < 0) continue;
            const long long j = q - f * step;
            unfold_add(acc, y[b + j % period[e]], j, L, overlap, sil, fl, mu);
        }
        if (s.frames > 0) acc = unfold_fade_out(acc, q - ((long long)(s.frames - 1) * hop - fo), fo);
        wave[idx] = (float)acc;
    }
}

// in place: y = mu-law decode of y (fp64, then fp32), ahead of the de-emphasis scan
__global__ void wavernn_mulaw_kernel(long long n, int mu, float* __restrict__ y) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const double v = y[i];
        y[i] = (float)((v > 0 ? 1.0 : (v < 0 ? -1.0 : 0.0)) / mu * (pow(1.0 + mu, fabs(v)) - 1.0));
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int wavernn_validate(const b200tts_wavernn_shape& s) {
    B200_REQUIRE(s.rows >= 1, "wavernn: need at least one fold row (rows = %d)", s.rows);
    B200_REQUIRE(s.rnn_dims >= WR_CTAS && s.rnn_dims % WR_CTAS == 0 && s.rnn_dims <= 5 * WR_CTAS,
                 "wavernn: rnn_dims %d must be a multiple of %d, at most %d", s.rnn_dims, WR_CTAS, 5 * WR_CTAS);
    B200_REQUIRE(s.fc_dims >= WR_CTAS && s.fc_dims % WR_CTAS == 0 && s.fc_dims <= 16 * WR_CTAS,
                 "wavernn: fc_dims %d must be a multiple of %d, at most %d", s.fc_dims, WR_CTAS, 16 * WR_CTAS);
    if (s.mode == B200TTS_WAVERNN_RAW) {
        B200_REQUIRE(s.n_out >= 2 && s.n_out <= 16 * WR_CTAS, "wavernn: RAW needs 2 to %d classes (n_out = %d)", 16 * WR_CTAS, s.n_out);
    } else {
        B200_REQUIRE(s.mode == B200TTS_WAVERNN_MOL, "wavernn: unknown mode %d", s.mode);
        B200_REQUIRE(s.n_out % 3 == 0 && s.n_out >= 3 && s.n_out <= 96, "wavernn: MOL needs 3 x (1..32) outputs (n_out = %d)", s.n_out);
    }
    B200_REQUIRE(s.fold_len >= 1, "wavernn: fold length %d must be positive", s.fold_len);
    B200_REQUIRE((long long)s.rows * s.fold_len * (s.n_out / 3 + 1) < (1ll << 40), "wavernn: batch too large");
    return B200TTS_OK;
}

// workspace: packed weights, fp32 state and scratch, bf16 activation rows, barrier; each region 256-byte aligned
struct WrLayout { size_t packed, h1, h2, x1, prev, logits, h1b, h2b, x1b, x2b, y1b, y2b, bar, bytes; };
static WrLayout wr_layout(const b200tts_wavernn_shape& s) {
    const WrDims d = wr_dims(s.rnn_dims, s.fc_dims, s.n_out);
    const size_t rows = s.rows, R = s.rnn_dims, Fc = s.fc_dims;
    WrLayout l;
    size_t off = 0;
    auto take = [&](size_t n) { const size_t o = off; off = align_up_sz(off + n, 256); return o; };
    l.packed = take((size_t)WR_CTAS * d.per_cta * 16);
    l.h1 = take(rows * R * 4);
    l.h2 = take(rows * R * 4);
    l.x1 = take(rows * R * 4);
    l.prev = take(rows * 4);
    l.logits = take(rows * s.n_out * 4);
    l.h1b = take(2 * rows * R * 2);
    l.h2b = take(2 * rows * R * 2);
    l.x1b = take(rows * R * 2);
    l.x2b = take(rows * R * 2);
    l.y1b = take(rows * Fc * 2);
    l.y2b = take(rows * Fc * 2);
    l.bar = take(256);            // counter, then the abort flag at +128
    l.bytes = off;
    return l;
}

static int wavernn_check(const b200tts_wavernn_shape& s, const void* ws, size_t ws_bytes) {
    B200_TRY(wavernn_validate(s));
    const WrLayout l = wr_layout(s);
    B200_REQUIRE(ws && ws_bytes >= l.bytes, "wavernn: workspace of %zu bytes is smaller than the %zu required", ws_bytes, l.bytes);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "wavernn: workspace must be 256-byte aligned");
    return B200TTS_OK;
}

// steps [t0, t0 + nsteps) from the state in the workspace; uniforms / out rows of L columns, column 0 at step io0
// ragged (row_t / row_n non-null): `rows` active rows, each from its own step count
static int wavernn_launch(const b200tts_wavernn_shape& s, const b200tts_wavernn_params& p, const b200tts_wavernn_cond& cond, int t0, int io0,
                          int L, int nsteps, const float* uniforms, float* out, float* dbg, void* ws, cudaStream_t st,
                          const long long* row_t = nullptr, const int* row_n = nullptr, int rows = 0) {
    B200_REQUIRE(p.b_hh1 && p.u1 && p.w_prev && p.b_hh2 && p.b_fc3, "wavernn_run: null parameter");
    B200_REQUIRE(cond.c && cond.g1 && cond.c2 && cond.p1 && cond.p2, "wavernn_run: null conditioning");
    B200_REQUIRE(uniforms && out, "wavernn_run: null uniforms or output");
    const WrLayout l = wr_layout(s);
    unsigned char* base = static_cast<unsigned char*>(ws);
    WrLoopArgs a;
    a.d = wr_dims(s.rnn_dims, s.fc_dims, s.n_out);
    a.rows = row_t ? rows : s.rows; a.mode = s.mode; a.L = L; a.t0 = t0; a.io0 = io0; a.nsteps = nsteps;
    a.row_t = row_t; a.row_n = row_n; a.slot = (size_t)s.rows * s.rnn_dims;
    a.packed = reinterpret_cast<const uint4*>(base + l.packed);
    a.b_hh1 = p.b_hh1; a.u1 = p.u1; a.w_prev = p.w_prev; a.b_hh2 = p.b_hh2; a.b_fc3 = p.b_fc3;
    a.cc = cond.c; a.g1 = cond.g1; a.c2 = cond.c2; a.p1 = cond.p1; a.p2 = cond.p2;
    a.uni = uniforms; a.out = out; a.dbg = dbg;
    a.h1 = reinterpret_cast<float*>(base + l.h1);
    a.h2 = reinterpret_cast<float*>(base + l.h2);
    a.x1 = reinterpret_cast<float*>(base + l.x1);
    a.prev = reinterpret_cast<float*>(base + l.prev);
    a.logits = reinterpret_cast<float*>(base + l.logits);
    a.h1b = reinterpret_cast<__nv_bfloat16*>(base + l.h1b);
    a.h2b = reinterpret_cast<__nv_bfloat16*>(base + l.h2b);
    a.x1b = reinterpret_cast<__nv_bfloat16*>(base + l.x1b);
    a.x2b = reinterpret_cast<__nv_bfloat16*>(base + l.x2b);
    a.y1b = reinterpret_cast<__nv_bfloat16*>(base + l.y1b);
    a.y2b = reinterpret_cast<__nv_bfloat16*>(base + l.y2b);
    a.bar = reinterpret_cast<unsigned*>(base + l.bar);
    a.abort_flag = reinterpret_cast<int*>(base + l.bar + 128);
    B200_CUDA(cudaMemsetAsync(a.bar, 0, sizeof(unsigned), st));       // the abort flag persists until the next prepare
    void* params[] = {&a};
    const void* fn = row_t ? (const void*)wavernn_loop_kernel<true> : (const void*)wavernn_loop_kernel<false>;
    return launch_persistent("wavernn_loop", fn, WR_CTAS, WR_THREADS, (size_t)a.d.per_cta * 16, false, params, st);
}

static int wavernn_run_rows_check(const b200tts_wavernn_shape& s, int active_rows, int nsteps) {
    B200_REQUIRE(active_rows >= 1 && active_rows <= s.rows && nsteps >= 1 && nsteps <= s.fold_len,
                 "wavernn_run_rows: %d active rows of %d, %d steps (at most fold_len = %d per call)", active_rows, s.rows, nsteps, s.fold_len);
    return B200TTS_OK;
}

static int wavernn_reset_rows_check(const b200tts_wavernn_shape& s, const int* rows, int count) {
    B200_REQUIRE(rows && count >= 1 && count <= s.rows, "wavernn_reset_rows: %d rows of a loop of %d", count, s.rows);
    for (int k = 0; k < count; ++k)
        B200_REQUIRE(rows[k] >= 0 && rows[k] < s.rows, "wavernn_reset_rows: row %d outside [0, %d)", rows[k], s.rows);
    return B200TTS_OK;
}

int wavernn_upsample_layer_check(int C, int len, int scale) {
    B200_REQUIRE(C >= 1 && len >= 1 && scale >= 1 && (long long)C * len * scale < (1ll << 40) && (long long)len * scale < (1ll << 31),
                 "wavernn_upsample_layer: bad dimensions (C = %d, len = %d, scale = %d)", C, len, scale);
    return B200TTS_OK;
}

static int wavernn_upsample_segments_check(int C, int nseg, const int* lens, int scale) {
    B200_REQUIRE(lens && nseg >= 1 && nseg <= B200TTS_WAVERNN_MAX_STREAMS, "wavernn_upsample_segments: %d segments (1 to %d)", nseg,
                 B200TTS_WAVERNN_MAX_STREAMS);
    long long total = 0;
    for (int g = 0; g < nseg; ++g) {
        B200_TRY(wavernn_upsample_layer_check(C, lens[g], scale));
        total += lens[g];
    }
    B200_REQUIRE((long long)C * total * scale < (1ll << 40), "wavernn_upsample_segments: %lld samples in all", total);
    return B200TTS_OK;
}

static int wavernn_fold_check(const b200tts_wavernn_fold_shape& s, int t0, int nsteps) {
    B200_REQUIRE(s.B >= 1 && s.rows >= s.B && s.n_mels >= 1 && s.aux_dims >= 0 && s.max_frames >= 1,
                 "wavernn_fold: bad dimensions (B = %d, rows = %d, n_mels = %d, aux_dims = %d, max_frames = %d)", s.B, s.rows, s.n_mels,
                 s.aux_dims, s.max_frames);
    B200_REQUIRE(s.hop >= 1 && s.scale >= 1 && s.hop % s.scale == 0 && s.pad >= 0,
                 "wavernn_fold: the hop %d must be a multiple of the last upsampling factor %d (pad %d)", s.hop, s.scale, s.pad);
    B200_REQUIRE(s.target >= 1 && s.overlap >= 0, "wavernn_fold: bad target %d / overlap %d", s.target, s.overlap);
    B200_REQUIRE(t0 >= 0 && nsteps >= 1 && t0 + nsteps <= s.target + 2 * s.overlap, "wavernn_fold: steps [%d, %d) outside the fold length %d",
                 t0, t0 + nsteps, s.target + 2 * s.overlap);
    return B200TTS_OK;
}

// every read of the positions [s0, s0 + nsteps) must fall inside the windows
static int wavernn_window_check(const b200tts_wavernn_window_shape& s, long long s0, int nsteps) {
    B200_REQUIRE(s.n_mels >= 1 && s.aux_dims >= 0 && s.frames >= 0 && s.mel_len >= 1 && s.aux_len >= 0 && s.m0 >= 0 && s.a0 >= 0,
                 "wavernn_window_rows: bad dimensions (n_mels = %d, aux_dims = %d, frames = %d, mel_len = %d, aux_len = %d, m0 = %lld, a0 = %d)",
                 s.n_mels, s.aux_dims, s.frames, s.mel_len, s.aux_len, s.m0, s.a0);
    B200_REQUIRE(s.hop >= 1 && s.scale >= 1 && s.hop % s.scale == 0 && s.pad >= 0,
                 "wavernn_window_rows: the hop %d must be a multiple of the last upsampling factor %d (pad %d)", s.hop, s.scale, s.pad);
    B200_REQUIRE(s0 >= 0 && nsteps >= 1, "wavernn_window_rows: positions [%lld, %lld)", s0, s0 + nsteps);
    long long q1 = s0 + nsteps;                          // positions [s0, q1) read the windows
    if (s.frames > 0 && q1 > (long long)s.frames * s.hop) q1 = (long long)s.frames * s.hop;
    if (q1 <= s0) return B200TTS_OK;
    const long long lo = s.frames > 0 ? (long long)(s.frames + 2 * s.pad) * s.hop : LLONG_MAX;
    long long j0 = s0 + (long long)s.pad * s.hop - s.scale, j1 = q1 - 1 + (long long)s.pad * s.hop + s.scale;
    if (j0 < 0) j0 = 0;
    if (j1 > lo - 1) j1 = lo - 1;
    B200_REQUIRE(j0 / s.scale >= s.m0 && j1 / s.scale < s.m0 + s.mel_len,
                 "wavernn_window_rows: positions [%lld, %lld) read penultimate samples [%lld, %lld], outside the window [%lld, %lld)", s0, q1,
                 j0 / s.scale, j1 / s.scale, s.m0, s.m0 + s.mel_len);
    B200_REQUIRE(s.aux_dims == 0 || (s0 / s.hop >= s.a0 && (q1 - 1) / s.hop < (long long)s.a0 + s.aux_len),
                 "wavernn_window_rows: positions [%lld, %lld) read aux frames [%lld, %lld], outside the window [%d, %d)", s0, q1, s0 / s.hop,
                 (q1 - 1) / s.hop, s.a0, s.a0 + s.aux_len);
    return B200TTS_OK;
}

// every row: wavernn_window_check of its own window, and the shared columns and factors of row 0
static int wavernn_window_rows_check(const b200tts_wavernn_window_row* rows, int active_rows, int nsteps) {
    B200_REQUIRE(rows && active_rows >= 1 && active_rows <= B200TTS_WAVERNN_MAX_STREAMS && nsteps >= 1,
                 "wavernn_window_rows: %d rows (1 to %d), %d steps", active_rows, B200TTS_WAVERNN_MAX_STREAMS, nsteps);
    const b200tts_wavernn_window_shape& w0 = rows[0].w;
    for (int r = 0; r < active_rows; ++r) {
        const b200tts_wavernn_window_row& d = rows[r];
        B200_REQUIRE(d.w.n_mels == w0.n_mels && d.w.aux_dims == w0.aux_dims && d.w.hop == w0.hop && d.w.pad == w0.pad && d.w.scale == w0.scale,
                     "wavernn_window_rows: row %d's columns or factors differ from row 0's", r);
        B200_REQUIRE(d.n >= 0 && d.n <= nsteps && d.mel_off >= 0 && d.aux_off >= 0, "wavernn_window_rows: row %d runs %d of %d steps "
                     "(offsets %lld, %lld)", r, d.n, nsteps, d.mel_off, d.aux_off);
        if (d.n > 0) B200_TRY(wavernn_window_check(d.w, d.s0, d.n));
    }
    return B200TTS_OK;
}

static int wavernn_unfold_check(int B, int hop, int target, int overlap, int mu) {
    B200_REQUIRE(B >= 1 && hop >= 1 && target >= 1 && overlap >= 0 && mu >= 0, "wavernn_unfold: bad arguments (B = %d, hop = %d, target = %d, "
                 "overlap = %d, mu = %d)", B, hop, target, overlap, mu);
    return B200TTS_OK;
}

// every stream: a non-empty range, packed right after the previous one, whose covering folds all have entries inside [0, nsrc)
static int wavernn_unfold_streams_check(int nstreams, int hop, int target, int overlap, int mu, const b200tts_wavernn_unfold_stream* streams,
                                 int nsrc, long long total) {
    B200_TRY(wavernn_unfold_check(1, hop, target, overlap, mu));
    B200_REQUIRE(streams && nstreams >= 1 && nstreams <= B200TTS_WAVERNN_MAX_STREAMS && nsrc >= 1,
                 "wavernn_unfold_streams: %d streams (1 to %d), %d fold sources", nstreams, B200TTS_WAVERNN_MAX_STREAMS, nsrc);
    const long long step = (long long)target + overlap, L = step + overlap;
    long long off = 0;
    for (int b = 0; b < nstreams; ++b) {
        const b200tts_wavernn_unfold_stream& s = streams[b];
        B200_REQUIRE(s.q0 >= 0 && s.q1 > s.q0 && s.wave_off == off && s.frames >= 0,
                     "wavernn_unfold_streams: stream %d writes positions [%lld, %lld) at %lld (expected %lld; frames %d)", b, s.q0, s.q1,
                     s.wave_off, off, s.frames);
        B200_REQUIRE(s.frames == 0 || s.q1 <= (long long)(s.frames - 1) * hop, "wavernn_unfold_streams: stream %d writes up to %lld, past the "
                     "cut %lld of its %d frames", b, s.q1, (long long)(s.frames - 1) * hop, s.frames);
        const long long f_lo = s.q0 >= L ? (s.q0 - L) / step + 1 : 0, f_hi = (s.q1 - 1) / step;
        B200_REQUIRE(s.fold0 >= 0 && s.fold0 <= f_lo && (long long)s.fold0 + s.nfolds > f_hi && s.src >= 0 && (long long)s.src + s.nfolds <= nsrc,
                     "wavernn_unfold_streams: stream %d's positions [%lld, %lld) read folds %lld to %lld; it lists folds %d to %d at sources "
                     "[%d, %d) of %d", b, s.q0, s.q1, f_lo, f_hi, s.fold0, s.fold0 + s.nfolds - 1, s.src, s.src + s.nfolds, nsrc);
        off += s.q1 - s.q0;
    }
    B200_REQUIRE(total == off, "wavernn_unfold_streams: total %lld, the streams write %lld", total, off);
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

int b200tts_wavernn_deemphasis(int rows, int len, int mu, float a, float* y, void* stream) {
    B200_REQUIRE(y, "wavernn_deemphasis: null argument");
    B200_REQUIRE(rows >= 1 && len >= 1 && mu >= 0 && (long long)rows * len < (1ll << 40), "wavernn_deemphasis: bad arguments (rows = %d, "
                 "len = %d, mu = %d)", rows, len, mu);
    B200_REQUIRE(a == a && a > -1.f && a < 1.f, "wavernn_deemphasis: the coefficient must lie in (-1, 1)");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wavernn_deemphasis", st);
    if (mu > 0) {
        wavernn_mulaw_kernel<<<grid_for((size_t)rows * len), 256, 0, st>>>((long long)rows * len, mu, y);
        B200_LAUNCH_CHECK();
    }
    return deemphasis_rows(rows, len, a, y, st);
}

size_t b200tts_wavernn_workspace_bytes(const b200tts_wavernn_shape* shape) {
    if (!shape) { set_last_error("wavernn_workspace_bytes: null shape"); return 0; }
    if (wavernn_validate(*shape) != B200TTS_OK) return 0;
    return wr_layout(*shape).bytes;
}

int b200tts_wavernn_prepare(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, void* workspace, size_t workspace_bytes,
                            void* stream) {
    B200_REQUIRE(shape && params, "wavernn_prepare: null argument");
    const b200tts_wavernn_shape& s = *shape;
    const b200tts_wavernn_params& p = *params;
    B200_TRY(wavernn_check(s, workspace, workspace_bytes));
    B200_TRY(require_device());
    B200_REQUIRE(p.w_hh1 && p.w_ih2x && p.w_hh2 && p.w_fc1x && p.w_fc2x && p.w_fc3, "wavernn_prepare: null weight");
    cudaStream_t st = (cudaStream_t)stream;
    const WrLayout l = wr_layout(s);
    const WrDims d = wr_dims(s.rnn_dims, s.fc_dims, s.n_out);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    B200_CUDA(cudaMemsetAsync(base + l.h1, 0, l.bytes - l.h1, st));    // zero state, zero previous sample, barrier and abort flag
    WrWeights W{{p.w_hh1, p.w_ih2x, p.w_hh2, p.w_fc1x, p.w_fc2x, p.w_fc3}};
    wavernn_pack_kernel<<<grid_for((size_t)WR_CTAS * d.per_cta), 256, 0, st>>>(d, W, reinterpret_cast<uint4*>(base + l.packed));
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wavernn_run(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond, int t0,
                        int nsteps, const float* uniforms, float* out, float* dbg, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && cond, "wavernn_run: null argument");
    const b200tts_wavernn_shape& s = *shape;
    B200_TRY(wavernn_check(s, workspace, workspace_bytes));
    B200_TRY(require_device());
    B200_REQUIRE(t0 >= 0 && nsteps >= 1 && t0 + nsteps <= s.fold_len, "wavernn_run: steps [%d, %d) outside the fold length %d", t0, t0 + nsteps,
                 s.fold_len);
    return wavernn_launch(s, *params, *cond, t0, 0, s.fold_len, nsteps, uniforms, out, dbg, workspace, (cudaStream_t)stream);
}

int b200tts_wavernn_run_stream(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond,
                               long long t, int nsteps, const float* uniforms, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && cond, "wavernn_run_stream: null argument");
    const b200tts_wavernn_shape& s = *shape;
    B200_TRY(wavernn_check(s, workspace, workspace_bytes));
    B200_TRY(require_device());
    B200_REQUIRE(t >= 0 && nsteps >= 1 && nsteps <= s.fold_len, "wavernn_run_stream: %d steps after %lld (at most fold_len = %d per call)",
                 nsteps, t, s.fold_len);
    // the loop only needs the step's parity (which slot of the double-buffered h1 / h2 rows is the previous step's)
    const int t0 = (int)(t & 1);
    return wavernn_launch(s, *params, *cond, t0, t0, nsteps, nsteps, uniforms, out, nullptr, workspace, (cudaStream_t)stream);
}

int b200tts_wavernn_run_rows(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond,
                             const int64_t* row_t, const int32_t* row_n, int active_rows, int nsteps, const float* uniforms, float* out,
                             void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && cond, "wavernn_run_rows: null argument");
    B200_REQUIRE(row_t && row_n && uniforms && out, "wavernn_run_rows: null row_t, row_n, uniforms or output");
    const b200tts_wavernn_shape& s = *shape;
    B200_TRY(wavernn_check(s, workspace, workspace_bytes));
    B200_TRY(wavernn_run_rows_check(s, active_rows, nsteps));
    B200_TRY(require_device());
    return wavernn_launch(s, *params, *cond, 0, 0, nsteps, nsteps, uniforms, out, nullptr, workspace, (cudaStream_t)stream,
                          reinterpret_cast<const long long*>(row_t), row_n, active_rows);
}

int b200tts_wavernn_reset_rows(const b200tts_wavernn_shape* shape, void* workspace, size_t workspace_bytes, const int32_t* rows, int count,
                               void* stream) {
    B200_REQUIRE(shape, "wavernn_reset_rows: null argument");
    const b200tts_wavernn_shape& s = *shape;
    B200_TRY(wavernn_check(s, workspace, workspace_bytes));
    B200_TRY(wavernn_reset_rows_check(s, rows, count));
    B200_TRY(require_device());
    const WrLayout l = wr_layout(s);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    for (int k0 = 0; k0 < count; k0 += B200TTS_WAVERNN_MAX_STREAMS) {
        WrRowList list;
        list.n = count - k0 < B200TTS_WAVERNN_MAX_STREAMS ? count - k0 : B200TTS_WAVERNN_MAX_STREAMS;
        for (int k = 0; k < list.n; ++k) list.row[k] = rows[k0 + k];
        wavernn_reset_rows_kernel<<<grid_for((size_t)list.n * s.rnn_dims), 256, 0, (cudaStream_t)stream>>>(
            list, s.rows, s.rnn_dims, reinterpret_cast<float*>(base + l.h1), reinterpret_cast<float*>(base + l.h2),
            reinterpret_cast<float*>(base + l.prev), reinterpret_cast<__nv_bfloat16*>(base + l.h1b), reinterpret_cast<__nv_bfloat16*>(base + l.h2b));
        B200_LAUNCH_CHECK();
    }
    return B200TTS_OK;
}

int b200tts_wavernn_window_rows(const b200tts_wavernn_window_row* rows, int active_rows, int nsteps, const float* mel, const float* fir,
                                const float* aux, float* feat, void* stream) {
    B200_REQUIRE(mel && fir && feat, "wavernn_window_rows: null argument");
    B200_TRY(wavernn_window_rows_check(rows, active_rows, nsteps));
    B200_REQUIRE(aux || rows[0].w.aux_dims == 0, "wavernn_window_rows: null aux");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const b200tts_wavernn_window_shape& w0 = rows[0].w;
    WrWinRows w;
    for (int r = 0; r < active_rows; ++r) {
        const b200tts_wavernn_window_row& d = rows[r];
        w.r[r] = WrWinRow{d.s0, d.w.m0, d.w.frames > 0 ? (long long)(d.w.frames + 2 * d.w.pad) * d.w.hop : LLONG_MAX, d.mel_off, d.aux_off, d.n,
                          d.w.frames, d.w.mel_len, d.w.a0};
    }
    KernelTimer kt("wavernn_window_rows", st);
    wavernn_window_rows_kernel<<<grid_for((size_t)nsteps * active_rows * (w0.n_mels + w0.aux_dims)), 256, 0, st>>>(
        w0.n_mels, w0.aux_dims, w0.hop, w0.pad, w0.scale, active_rows, w, mel, fir, aux, nsteps, feat);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wavernn_aborted(const b200tts_wavernn_shape* shape, const void* workspace, size_t workspace_bytes, int* aborted, void* stream) {
    B200_REQUIRE(shape && aborted, "wavernn_aborted: null argument");
    B200_TRY(require_device());
    const b200tts_wavernn_shape& s = *shape;
    B200_TRY(wavernn_check(s, workspace, workspace_bytes));
    cudaStream_t st = (cudaStream_t)stream;
    const WrLayout l = wr_layout(s);
    B200_CUDA(cudaMemcpyAsync(aborted, static_cast<const unsigned char*>(workspace) + l.bar + 128, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200TTS_OK;
}

int b200tts_wavernn_upsample_layer(int C, int len, int scale, const float* fir, const float* in, float* out, void* stream) {
    B200_REQUIRE(fir && in && out, "wavernn_upsample_layer: null argument");
    B200_TRY(wavernn_upsample_layer_check(C, len, scale));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wavernn_upsample", st);
    wavernn_upsample_layer_kernel<<<grid_for((size_t)C * len * scale), 256, 0, st>>>(C, len, scale, fir, in, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wavernn_upsample_segments(int C, int nseg, const int32_t* lens, int scale, const float* fir, const float* in, float* out,
                                      void* stream) {
    B200_REQUIRE(fir && in && out, "wavernn_upsample_segments: null argument");
    B200_TRY(wavernn_upsample_segments_check(C, nseg, lens, scale));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    WrSegments g;
    g.n = nseg; g.C = C; g.in_off[0] = 0;
    for (int k = 0; k < nseg; ++k) { g.len[k] = lens[k]; g.in_off[k + 1] = g.in_off[k] + (long long)C * lens[k]; }
    KernelTimer kt("wavernn_upsample", st);
    wavernn_upsample_segments_kernel<<<grid_for((size_t)g.in_off[nseg] * scale), 256, 0, st>>>(g, scale, fir, in, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wavernn_fold(const b200tts_wavernn_fold_shape* shape, const float* mel_up, const int64_t* mel_off, const int32_t* frames,
                         const int32_t* row_utt, const int32_t* row_fold, const float* fir, const float* aux, int t0, int nsteps, float* feat,
                         void* stream) {
    B200_REQUIRE(shape && mel_up && mel_off && frames && row_utt && row_fold && fir && feat, "wavernn_fold: null argument");
    B200_REQUIRE(aux || shape->aux_dims == 0, "wavernn_fold: null aux");
    const b200tts_wavernn_fold_shape& s = *shape;
    B200_TRY(wavernn_fold_check(s, t0, nsteps));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wavernn_fold", st);
    wavernn_fold_kernel<<<grid_for((size_t)nsteps * s.rows * (s.n_mels + s.aux_dims)), 256, 0, st>>>(
        s, mel_up, reinterpret_cast<const long long*>(mel_off), frames, row_utt, row_fold, fir, aux, t0, nsteps, feat);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wavernn_unfold(int B, int hop, int target, int overlap, int mu, const int32_t* frames, const int32_t* row_off, const int64_t* wave_off,
                           long long total, const float* y, float* wave, void* stream) {
    B200_REQUIRE(frames && row_off && wave_off && y && wave, "wavernn_unfold: null argument");
    B200_TRY(wavernn_unfold_check(B, hop, target, overlap, mu));
    B200_TRY(require_device());
    if (total <= 0) return B200TTS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wavernn_unfold", st);
    wavernn_unfold_kernel<<<grid_for((size_t)total), 256, 0, st>>>(B, hop, target, overlap, mu, frames, row_off,
                                                                   reinterpret_cast<const long long*>(wave_off), y, wave, total);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_wavernn_unfold_streams(int nstreams, int hop, int target, int overlap, int mu, const b200tts_wavernn_unfold_stream* streams,
                                   const int64_t* base, const int32_t* period, int nsrc, long long total, const float* y, float* wave,
                                   void* stream) {
    B200_REQUIRE(base && period && y && wave, "wavernn_unfold_streams: null argument");
    B200_TRY(wavernn_unfold_streams_check(nstreams, hop, target, overlap, mu, streams, nsrc, total));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    WrUnfoldStreams g;
    g.n = nstreams;
    for (int b = 0; b < nstreams; ++b) g.s[b] = streams[b];
    KernelTimer kt("wavernn_unfold", st);
    wavernn_unfold_streams_kernel<<<grid_for((size_t)total), 256, 0, st>>>(g, hop, target, overlap, mu, reinterpret_cast<const long long*>(base),
                                                                           period, y, wave, total);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
