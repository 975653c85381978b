// Decoder backward (BPTT): the reverse of decoder_fwd.cu.
// Restates what torch autograd replays for Decoder._decode (reference modules/tacotron2.py:148-209,
// train.py:83): frame/stop projection grads -> generator LSTM reverse loop -> attention LSTM +
// location-sensitive attention reverse loop (energies recomputed, never stored) -> time-batched dW GEMMs.
// A decode with free-running steps (teacher forcing < 1) runs the two reverse loops as a segmented sweep
// instead, because each such step sends gradient back through the frame it was fed.
#include <cuda_bf16.h>
#include "decoder_internal.cuh"

namespace b200tts {

namespace {

// ---------------------------------------------------------------------------------------------
// utility kernels
// ---------------------------------------------------------------------------------------------
// The inverse of split_frames_kernel: dFS [S, B, R*(N+1)] from the per-frame gradients, frame k = i*R + j of step i, slot j:
// dFS[i, b, j*N + n] = d_spec[b, k, n], dFS[i, b, R*N + j] = d_stop[b, k]; 0 for the frames of the last step past T.
__global__ void gather_frame_grads_kernel(float* __restrict__ dfs, const float* __restrict__ dspec,
                                          const float* __restrict__ dstop, int B, int S, int T, int N, int R) {
    const int W = R * (N + 1), RN = R * N;
    const size_t total = (size_t)B * S * W;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int c = idx % W;
        const int b = (idx / W) % B;
        const int i = idx / ((size_t)W * B);
        const int j = c < RN ? c / N : c - RN, k = i * R + j;
        float v = 0.f;
        if (k < T) {
            if (c < RN) { if (dspec) v = dspec[((size_t)b * T + k) * N + c - j * N]; }
            else if (dstop) v = dstop[(size_t)b * T + k];
        }
        dfs[idx] = v;
    }
}

// Column sums (bias gradients), deterministic two-level tree: partial[s][c] = sum of row slice s, then dst[c] += sum_s partial[s][c].
constexpr int COLSUM_SLICES = 64;
__global__ void colsum_partial_kernel(float* __restrict__ partial, const float* __restrict__ src, size_t rows, int cols, int ld) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const size_t per = (rows + gridDim.y - 1) / gridDim.y;
    const size_t r0 = blockIdx.y * per, r1 = r0 + per < rows ? r0 + per : rows;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    if (c < cols) {
        size_t r = r0 + threadIdx.y;
        for (; r + 24 < r1; r += 32) {
            a0 += src[r * ld + c]; a1 += src[(r + 8) * ld + c]; a2 += src[(r + 16) * ld + c]; a3 += src[(r + 24) * ld + c];
        }
        for (; r < r1; r += 8) a0 += src[r * ld + c];
    }
    sm[threadIdx.y][threadIdx.x] = (a0 + a1) + (a2 + a3);
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) s += sm[j][threadIdx.x];
        partial[(size_t)blockIdx.y * cols + c] = s;
    }
}
__global__ void colsum_finish_kernel(float* __restrict__ dst, float* __restrict__ dst2, const float* __restrict__ partial, int slices, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float s = 0.f;
    for (int j = 0; j < slices; ++j) s += partial[(size_t)j * cols + c];
    dst[c] += s;
    if (dst2) dst2[c] += s;
}
// dst[c] (+ dst2[c]) += sum_r src[r*ld + c]; scratch holds COLSUM_SLICES * cols floats
int colsum_add(float* dst, float* dst2, const float* src, size_t rows, int cols, int ld, float* scratch, cudaStream_t st) {
    int slices = (int)(rows / 256);
    slices = slices < 1 ? 1 : (slices > COLSUM_SLICES ? COLSUM_SLICES : slices);
    colsum_partial_kernel<<<dim3(cdiv(cols, 32), slices), dim3(32, 8), 0, st>>>(scratch, src, rows, cols, ld);
    B200_LAUNCH_CHECK();
    colsum_finish_kernel<<<cdiv(cols, 128), 128, 0, st>>>(dst, dst2, scratch, slices, cols);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

// dst[j] += sum_b src[b*n + j]
__global__ void batchsum_add_kernel(float* __restrict__ dst, const float* __restrict__ src, int batch, size_t n) {
    for (size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x; j < n; j += (size_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int b = 0; b < batch; ++b) s += src[(size_t)b * n + j];
        dst[j] += s;
    }
}

// dst[r*ldd + c] += src[r*lds + c]
__global__ void add2d_kernel(float* __restrict__ dst, int ldd, const float* __restrict__ src, int lds, int rows, int cols) {
    const size_t total = (size_t)rows * cols;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int r = idx / cols, c = idx % cols;
        dst[(size_t)r * ldd + c] += src[(size_t)r * lds + c];
    }
}

// prenet layer backward through dropout + relu: dz = dy * scale * (y > 0)   (y is post relu+dropout)
__global__ void relu_dropout_bwd_kernel(float* __restrict__ dz, const float* __restrict__ dy, const float* __restrict__ y,
                                        float scale, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dz[i] = y[i] > 0.f ? dy[i] * scale : 0.f;
}

// Feedback of a free-running step f >= 1 into the frame it was fed, x_f = FS[f-1, :, 0:N] (tacotron2.py:171,181; not detached),
// one CTA per utterance.  dp1 = d p1_f (the product dga_f . W_ih_att[:, :P], taken by the GEMM before this kernel):
//   dz1 = dp1 * scale1 * (p1 > 0);  dp0 = dz1 . W1;  dz0 = dp0 * scale0 * (p0 > 0);  dx = dz0 . W0
//   dFS[f-1, b, (R-1)N : RN] += dx;  [d h_gen | d ctx]_{f-1} += dx . Wfs[(R-1)N : RN, :]   (the fed-back frame is the last of step f-1's R;
//   direct / static parts, consumed by the reverse steps f-1)
// Every sum runs in a fixed order (no atomics).
struct FeedbackArgs {
    const float* dp1;                  // [B, P]
    const float* p0; const float* p1;  // [B, P] step f's prenet activations (after relu + dropout)
    const float* W0; const float* W1;  // prenet_w0 [P, N], prenet_w1 [P, P]
    const float* wfs;                  // [N, D+M]   rows of the fed-back frame in [frame_w ; stop_w]
    float* dfs;                        // [B, ld_fs] the fed-back frame's columns of dFS row f-1
    int ld_fs;
    float* dhgd;                       // [B, D]   row f-1
    float* dctxs;                      // [B, M]   row f-1
    float scale0, scale1;
    int B, P, N, D, M;
};
constexpr int FEEDBACK_THREADS = 256;
__host__ __device__ inline int feedback_slices(int N) { const int s = FEEDBACK_THREADS / N; return s < 1 ? 1 : s; }
inline size_t feedback_smem_floats(int P, int N) { return (size_t)2 * P + (size_t)(feedback_slices(N) + 1) * N; }

__global__ void __launch_bounds__(FEEDBACK_THREADS) frame_feedback_bwd_kernel(const FeedbackArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int b = blockIdx.x, tid = threadIdx.x, P = p.P, N = p.N, DM = p.D + p.M;
    const int ns = feedback_slices(N), per = (P + ns - 1) / ns;
    float* dz1 = sm; float* dz0 = dz1 + P; float* xpart = dz0 + P; float* dx = xpart + (size_t)ns * N;
    const size_t row = (size_t)b * P;
    for (int j = tid; j < P; j += FEEDBACK_THREADS) dz1[j] = p.p1[row + j] > 0.f ? p.dp1[row + j] * p.scale1 : 0.f;
    __syncthreads();
    // dp0[j] = sum_k dz1[k] W1[k, j]  (W1 rows are the layer's outputs)
    for (int j = tid; j < P; j += FEEDBACK_THREADS) {
        float acc = 0.f;
        for (int k = 0; k < P; ++k) acc = fmaf(dz1[k], p.W1[(size_t)k * P + j], acc);
        dz0[j] = p.p0[row + j] > 0.f ? acc * p.scale0 : 0.f;
    }
    __syncthreads();
    // dx[n] = sum_j dz0[j] W0[j, n]: `ns` slices of j per column, then the slices in order
    for (int t = tid; t < ns * N; t += FEEDBACK_THREADS) {
        const int n = t % N, sl = t / N, j1 = min(P, (sl + 1) * per);
        float acc = 0.f;
        for (int j = sl * per; j < j1; ++j) acc = fmaf(dz0[j], p.W0[(size_t)j * N + n], acc);
        xpart[(size_t)sl * N + n] = acc;
    }
    __syncthreads();
    for (int n = tid; n < N; n += FEEDBACK_THREADS) {
        float acc = 0.f;
        for (int sl = 0; sl < ns; ++sl) acc += xpart[(size_t)sl * N + n];
        dx[n] = acc;
        p.dfs[(size_t)b * p.ld_fs + n] += acc;
    }
    __syncthreads();
    for (int c = tid; c < DM; c += FEEDBACK_THREADS) {
        float acc = 0.f;
        for (int n = 0; n < N; ++n) acc = fmaf(dx[n], p.wfs[(size_t)n * DM + c], acc);
        if (c < p.D) p.dhgd[(size_t)b * p.D + c] += acc;
        else p.dctxs[(size_t)b * p.M + c - p.D] += acc;
    }
}

// ---------------------------------------------------------------------------------------------
// LSTM cell backward (pointwise) -- one thread owns 8 utterances of one hidden unit
// ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) lstm_cell_bwd_kernel(const CellBwdArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int Bp = (p.B + 7) & ~7;
    float* dqT = sm;                                   // [A][Bp]
    float* wq = sm + (size_t)p.A * Bp;                 // [A][CELL_UNITS + 1]
    const int u0 = blockIdx.x * CELL_UNITS, D = p.D, A = p.A;
    if (p.dq) {
        for (int idx = threadIdx.x; idx < A * Bp; idx += blockDim.x) {
            const int b = idx / A, a = idx % A;
            dqT[a * Bp + b] = b < p.B ? p.dq[(size_t)b * A + a] : 0.f;
        }
        for (int idx = threadIdx.x; idx < A * CELL_UNITS; idx += blockDim.x) {
            const int a = idx / CELL_UNITS, uu = idx % CELL_UNITS;
            wq[a * (CELL_UNITS + 1) + uu] = (u0 + uu < D) ? p.Wq[(size_t)a * D + u0 + uu] : 0.f;
        }
        __syncthreads();
    }
    const float inv_h = 1.f / (1.f - p.rate_h), inv_c = 1.f / (1.f - p.rate_c);
    const int nbg = Bp / 8;
    for (int item = threadIdx.x; item < CELL_UNITS * nbg; item += blockDim.x) {
        const int uu = item % CELL_UNITS, bg = item / CELL_UNITS, u = u0 + uu;
        float dhq[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) dhq[j] = 0.f;
        if (p.dq) {
            for (int a = 0; a < A; ++a) {
                const float w = wq[a * (CELL_UNITS + 1) + uu];
                const float4 d0 = *reinterpret_cast<const float4*>(&dqT[a * Bp + bg * 8]);
                const float4 d1 = *reinterpret_cast<const float4*>(&dqT[a * Bp + bg * 8 + 4]);
                dhq[0] = fmaf(w, d0.x, dhq[0]); dhq[1] = fmaf(w, d0.y, dhq[1]); dhq[2] = fmaf(w, d0.z, dhq[2]); dhq[3] = fmaf(w, d0.w, dhq[3]);
                dhq[4] = fmaf(w, d1.x, dhq[4]); dhq[5] = fmaf(w, d1.y, dhq[5]); dhq[6] = fmaf(w, d1.z, dhq[6]); dhq[7] = fmaf(w, d1.w, dhq[7]);
            }
        }
        if (u >= D) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int b = bg * 8 + j;
            if (b >= p.B) continue;
            const size_t bu = (size_t)b * D + u, g0 = (size_t)b * 4 * D + u;
            float dh = dhq[j];
            if (p.dh_static) dh += p.dh_static[(size_t)b * p.ld_dhs + u];
            float dc_in = 0.f, dh_rec = 0.f;
            if (!p.last) {
                for (int s = 0; s < p.nsplit; ++s) dh_rec += p.part[s * p.part_stride + (size_t)b * p.ld_part + p.part_col0 + u];
                dc_in = p.dc_state[bu];
                if (p.dhz_state) dh_rec += p.dhz_state[bu];
            }
            if (p.lengths && p.step >= p.lengths[b]) {    // frozen step: gradients of the state pass straight through
                p.dgates[g0] = 0.f; p.dgates[g0 + D] = 0.f; p.dgates[g0 + 2 * D] = 0.f; p.dgates[g0 + 3 * D] = 0.f;
                p.dc_state[bu] = dc_in;
                p.dhz_state[bu] = dh_rec;
                continue;
            }
            dh += dh_rec;
            const float gi = p.gates[g0], gf = p.gates[g0 + D], gg = p.gates[g0 + 2 * D], go = p.gates[g0 + 3 * D];
            const float cp = p.c_prev[bu];
            const float tc = tanhf(gf * cp + gi * gg);
            float dhn, dcn, dc_prev_direct = 0.f, dh_prev_direct = 0.f;     // grads wrt raw h', c'
            if (p.kind == B200TTS_CELL_ZONEOUT) {
                float kh, kc;    // d out / d raw
                if (p.training) {
                    kh = (1.f - p.rate_h) * (p.mask_h ? (float)p.mask_h[bu] * inv_h : 1.f);
                    kc = (1.f - p.rate_c) * (p.mask_c ? (float)p.mask_c[bu] * inv_c : 1.f);
                } else {
                    kh = 1.f - p.rate_h; kc = 1.f - p.rate_c;
                }
                dhn = dh * kh; dh_prev_direct = dh - dhn;
                dcn = dc_in * kc + dhn * go * (1.f - tc * tc);
                dc_prev_direct = dc_in - dc_in * kc;
            } else {
                dhn = (p.training && p.mask_h) ? dh * (float)p.mask_h[bu] * inv_h : dh;
                dcn = dc_in + dhn * go * (1.f - tc * tc);
            }
            p.dgates[g0] = dcn * gg * gi * (1.f - gi);
            p.dgates[g0 + D] = dcn * cp * gf * (1.f - gf);
            p.dgates[g0 + 2 * D] = dcn * gi * (1.f - gg * gg);
            p.dgates[g0 + 3 * D] = dhn * tc * go * (1.f - go);
            p.dc_state[bu] = dcn * gf + dc_prev_direct;
            if (p.dhz_state) p.dhz_state[bu] = dh_prev_direct;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Attention step backward, one CTA per utterance.  Recomputes location features and tanh
// arguments from the saved query and cumulative weights (SURVEY 7.3 "Backward memory").
// ---------------------------------------------------------------------------------------------
struct AttnBwdArgs {
    const float* q;            // [B, A] saved query of this step
    const float* memT;         // [B, L, A]
    const float* memory;       // [B, L, M]
    const int* lengths;
    const float* Wc; const float* Wloc; const float* bias; const float* v;
    const float* cum_prev;     // [B, L] cumulative weights the step consumed
    const float* w;  long long w_bstride;        // &align[0, i, 0]
    const float* dalign; long long dalign_bstride;   // &d_align[0, i, 0] or null
    const float* dctx_static;  // [B, M]
    const float* part; int nsplit; size_t part_stride; int ld_part;   // recurrent d ctx partials (cols [0, M)); null on last step
    float* dcum;               // [B, L] in: d cum_i, out: d cum_{i-1}
    float* dctx_tot;           // [B, M] out
    float* dq;                 // [B, A] out
    float* dmemT;              // [B, L, A] +=
    float* dWloc_acc;          // [B, A, C] +=
    float* dWc_acc;            // [B, C, K] +=
    float* dv_acc;             // [B, A] +=
    int B, L, M, A, C, K, LC, last;
};

struct AttnBwdSmem {
    int Lp, cumn, off_qb, off_vv, off_cump, off_Wl, off_WlT, off_Wcs, off_f, off_dF, off_w, off_de, off_ds, off_red, off_dctx,
        off_cred, total;
};
__host__ __device__ inline AttnBwdSmem attn_bwd_smem(int L, int M, int A, int C, int K, int LC) {
    AttnBwdSmem s;
    s.Lp = (L + 3) & ~3;
    s.cumn = (L + K - 1 + 3) & ~3;
    int o = 0;
    s.off_qb = o; o += A;
    s.off_vv = o; o += A;
    s.off_cump = o; o += s.cumn;
    s.off_Wl = o; o += A * C;
    s.off_WlT = o; o += C * A;
    s.off_Wcs = o; o += (C * K + 3) & ~3;
    s.off_f = o; o += C * s.Lp;
    s.off_dF = o; o += C * (s.Lp + 2 * K);        // K zeros either side so the transposed conv needs no bounds checks
    s.off_w = o; o += s.Lp;
    s.off_de = o; o += s.Lp;
    s.off_ds = o; o += LC * (A + 4);
    s.off_red = o; o += 64;
    s.off_dctx = o; o += (M + 3) & ~3;
    s.off_cred = o; o += (8 * A > 4 * s.Lp ? 8 * A : 4 * s.Lp);   // [8][A] query partials, later [4][Lp] conv partials
    s.total = o;
    return s;
}

__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_kernel(const AttnBwdArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = ATT_THREADS / 32;
    const int L = p.L, A = p.A, C = p.C, K = p.K, M = p.M, LC = p.LC;
    const int half = (K - 1) / 2;
    const AttnBwdSmem so = attn_bwd_smem(L, M, A, C, K, LC);
    const int Lp = so.Lp, dFld = Lp + 2 * K, AS = A + 4;
    float* qb = sm + so.off_qb; float* vv = sm + so.off_vv; float* cump = sm + so.off_cump;
    float* Wl = sm + so.off_Wl; float* WlT = sm + so.off_WlT; float* Wcs = sm + so.off_Wcs;
    float* f = sm + so.off_f; float* dF = sm + so.off_dF; float* wS = sm + so.off_w; float* de = sm + so.off_de;
    float* dsS = sm + so.off_ds; float* red = sm + so.off_red; float* dctx = sm + so.off_dctx; float* cred = sm + so.off_cred;
    int len = p.lengths[b];
    len = len < 0 ? 0 : (len > L ? L : len);

    // ---- phase 1: stage small operands ----
    for (int a = tid; a < A; a += ATT_THREADS) { qb[a] = p.q[(size_t)b * A + a] + p.bias[a]; vv[a] = p.v[a]; }
    for (int j = tid; j < L + K - 1; j += ATT_THREADS) {
        const int l = j - half;
        cump[j] = (l >= 0 && l < L) ? p.cum_prev[(size_t)b * L + l] : 0.f;
    }
    for (int idx = tid; idx < A * C; idx += ATT_THREADS) {
        const float wv = p.Wloc[idx];
        Wl[idx] = wv;
        WlT[(idx % C) * A + idx / C] = wv;
    }
    for (int idx = tid; idx < C * K; idx += ATT_THREADS) Wcs[idx] = p.Wc[idx];
    for (int idx = tid; idx < C * dFld; idx += ATT_THREADS) dF[idx] = 0.f;
    for (int l = tid; l < Lp; l += ATT_THREADS) wS[l] = l < L ? p.w[(size_t)b * p.w_bstride + l] : 0.f;
    for (int m = tid; m < M; m += ATT_THREADS) {
        float g = p.dctx_static[(size_t)b * M + m];
        if (!p.last)
            for (int s = 0; s < p.nsplit; ++s) g += p.part[s * p.part_stride + (size_t)b * p.ld_part + m];
        dctx[m] = g;
        p.dctx_tot[(size_t)b * M + m] = g;
    }
    __syncthreads();

    // ---- phase 2: location features; dw[l] = dalign + dcum + <dctx, memory[l]> ----
    for (int idx = tid; idx < C * Lp; idx += ATT_THREADS) {
        const int c = idx / Lp, l = idx % Lp;
        float acc = 0.f;
        if (l < L)
            for (int k = 0; k < K; ++k) acc = fmaf(Wcs[c * K + k], cump[l + k], acc);
        f[idx] = acc;
    }
    for (int l = warp; l < Lp; l += NW) {
        float acc = 0.f;
        if (l < len) {
            const float* row = p.memory + ((size_t)b * L + l) * M;
            for (int m = lane; m < M; m += 32) acc = fmaf(dctx[m], row[m], acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) {
            float g = 0.f;
            if (l < len) {
                g = acc + (p.last ? 0.f : p.dcum[(size_t)b * L + l]);
                if (p.dalign) g += p.dalign[(size_t)b * p.dalign_bstride + l];
            }
            de[l] = g;        // holds dw for now
        }
    }
    __syncthreads();

    // ---- phase 3: softmax backward ----
    float dot = 0.f;
    for (int l = tid; l < len; l += ATT_THREADS) dot = fmaf(wS[l], de[l], dot);
    dot = block_sum(dot, red);
    for (int l = tid; l < Lp; l += ATT_THREADS) de[l] = l < len ? wS[l] * (de[l] - dot) : 0.f;
    __syncthreads();

    // ---- phase 4: energy backward, chunked over positions ----
    float dq_reg[4] = {0.f, 0.f, 0.f, 0.f}, dv_reg[4] = {0.f, 0.f, 0.f, 0.f};
    const int ntile = ((A / 4) * (C / 4));                 // 4a x 4c tiles of dWloc (<= 256 by validation)
    const int t_a0 = (tid % (A / 4)) * 4, t_c0 = (tid / (A / 4)) * 4;
    float accW[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) accW[i][j] = 0.f;

    for (int lc0 = 0; lc0 < len; lc0 += LC) {
        const int rows = min(LC, ((len - lc0) + 3) & ~3);   // multiple of 4, rows beyond len are written as zeros
        // 4a: recompute s, ds
        for (int r0 = warp * 4; r0 < rows; r0 += NW * 4) {
            const int l0 = lc0 + r0;
            float s[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
            for (int c = 0; c < C; ++c) {
                const float4 fv = *reinterpret_cast<const float4*>(&f[c * Lp + l0]);
                float wv[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) wv[j] = (lane + 32 * j < A) ? WlT[c * A + lane + 32 * j] : 0.f;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    s[0][j] = fmaf(fv.x, wv[j], s[0][j]); s[1][j] = fmaf(fv.y, wv[j], s[1][j]);
                    s[2][j] = fmaf(fv.z, wv[j], s[2][j]); s[3][j] = fmaf(fv.w, wv[j], s[3][j]);
                }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int l = l0 + i;
                const float del = l < len ? de[l] : 0.f;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int a = lane + 32 * j;
                    if (a < A) {
                        float dsv = 0.f;
                        if (l < len) {
                            const size_t mi = ((size_t)b * L + l) * A + a;
                            const float th = tanhf(s[i][j] + qb[a] + p.memT[mi]);
                            dsv = del * vv[a] * (1.f - th * th);
                            dv_reg[j] = fmaf(del, th, dv_reg[j]);
                            dq_reg[j] += dsv;
                            p.dmemT[mi] += dsv;
                        }
                        dsS[(r0 + i) * AS + a] = dsv;
                    }
                }
            }
        }
        __syncthreads();
        // 4b: dF[c, l] = sum_a ds[l, a] * Wloc[a, c]      (4c x 4l register tiles)
        {
            const int ncg = C / 4;
            for (int t = tid; t < ncg * (rows / 4); t += ATT_THREADS) {
                const int c0 = (t % ncg) * 4, r0 = (t / ncg) * 4;
                float acc[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
                for (int a = 0; a < A; ++a) {
                    const float4 w4 = *reinterpret_cast<const float4*>(&Wl[a * C + c0]);
                    const float d0 = dsS[(r0 + 0) * AS + a], d1 = dsS[(r0 + 1) * AS + a];
                    const float d2 = dsS[(r0 + 2) * AS + a], d3 = dsS[(r0 + 3) * AS + a];
                    acc[0][0] = fmaf(w4.x, d0, acc[0][0]); acc[0][1] = fmaf(w4.x, d1, acc[0][1]); acc[0][2] = fmaf(w4.x, d2, acc[0][2]); acc[0][3] = fmaf(w4.x, d3, acc[0][3]);
                    acc[1][0] = fmaf(w4.y, d0, acc[1][0]); acc[1][1] = fmaf(w4.y, d1, acc[1][1]); acc[1][2] = fmaf(w4.y, d2, acc[1][2]); acc[1][3] = fmaf(w4.y, d3, acc[1][3]);
                    acc[2][0] = fmaf(w4.z, d0, acc[2][0]); acc[2][1] = fmaf(w4.z, d1, acc[2][1]); acc[2][2] = fmaf(w4.z, d2, acc[2][2]); acc[2][3] = fmaf(w4.z, d3, acc[2][3]);
                    acc[3][0] = fmaf(w4.w, d0, acc[3][0]); acc[3][1] = fmaf(w4.w, d1, acc[3][1]); acc[3][2] = fmaf(w4.w, d2, acc[3][2]); acc[3][3] = fmaf(w4.w, d3, acc[3][3]);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) dF[(c0 + i) * dFld + K + lc0 + r0 + j] = acc[i][j];
            }
        }
        // 4c: dWloc[a, c] += sum_l ds[l, a] * f[c, l]       (4a x 4c register tile per thread, kept across chunks)
        if (tid < ntile) {
            for (int r = 0; r < rows; ++r) {
                const float4 d4 = *reinterpret_cast<const float4*>(&dsS[r * AS + t_a0]);
                const float f0 = f[(t_c0 + 0) * Lp + lc0 + r], f1 = f[(t_c0 + 1) * Lp + lc0 + r];
                const float f2 = f[(t_c0 + 2) * Lp + lc0 + r], f3 = f[(t_c0 + 3) * Lp + lc0 + r];
                accW[0][0] = fmaf(d4.x, f0, accW[0][0]); accW[0][1] = fmaf(d4.x, f1, accW[0][1]); accW[0][2] = fmaf(d4.x, f2, accW[0][2]); accW[0][3] = fmaf(d4.x, f3, accW[0][3]);
                accW[1][0] = fmaf(d4.y, f0, accW[1][0]); accW[1][1] = fmaf(d4.y, f1, accW[1][1]); accW[1][2] = fmaf(d4.y, f2, accW[1][2]); accW[1][3] = fmaf(d4.y, f3, accW[1][3]);
                accW[2][0] = fmaf(d4.z, f0, accW[2][0]); accW[2][1] = fmaf(d4.z, f1, accW[2][1]); accW[2][2] = fmaf(d4.z, f2, accW[2][2]); accW[2][3] = fmaf(d4.z, f3, accW[2][3]);
                accW[3][0] = fmaf(d4.w, f0, accW[3][0]); accW[3][1] = fmaf(d4.w, f1, accW[3][1]); accW[3][2] = fmaf(d4.w, f2, accW[3][2]); accW[3][3] = fmaf(d4.w, f3, accW[3][3]);
            }
        }
        __syncthreads();
    }
    if (tid < ntile) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) p.dWloc_acc[((size_t)b * A + t_a0 + i) * C + t_c0 + j] += accW[i][j];
    }
    // query / energy-vector gradients: reduce the per-warp partials
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int a = lane + 32 * j;
        if (a < A) { cred[warp * A + a] = dq_reg[j]; }
    }
    __syncthreads();
    for (int a = tid; a < A; a += ATT_THREADS) {
        float s = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < NW; ++w8) s += cred[w8 * A + a];
        p.dq[(size_t)b * A + a] = s;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int a = lane + 32 * j;
        if (a < A) { cred[warp * A + a] = dv_reg[j]; }
    }
    __syncthreads();
    for (int a = tid; a < A; a += ATT_THREADS) {
        float s = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < NW; ++w8) s += cred[w8 * A + a];
        p.dv_acc[(size_t)b * A + a] += s;
    }
    __syncthreads();

    // ---- phase 5: location conv backward ----
    // dWc[c, k] += sum_l dF[c, l] * cum[l + k - half]     (thread = one c, 4 consecutive k, sliding window)
    {
        const int nkg = (K + 3) / 4;
        for (int t = tid; t < C * nkg; t += ATT_THREADS) {
            const int c = t / nkg, k0 = (t % nkg) * 4;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            // cump index l + k; entries beyond the padded array are only reached for k >= K (discarded)
            float w0 = cump[min(k0, so.cumn - 1)], w1 = cump[min(k0 + 1, so.cumn - 1)], w2 = cump[min(k0 + 2, so.cumn - 1)];
            for (int l = 0; l < len; ++l) {
                const float w3 = cump[min(l + k0 + 3, so.cumn - 1)];
                const float d = dF[c * dFld + K + l];
                a0 = fmaf(d, w0, a0); a1 = fmaf(d, w1, a1); a2 = fmaf(d, w2, a2); a3 = fmaf(d, w3, a3);
                w0 = w1; w1 = w2; w2 = w3;
            }
            float* dst = p.dWc_acc + ((size_t)b * C + c) * K + k0;
            if (k0 < K) dst[0] += a0;
            if (k0 + 1 < K) dst[1] += a1;
            if (k0 + 2 < K) dst[2] += a2;
            if (k0 + 3 < K) dst[3] += a3;
        }
    }
    // d cum_{i-1}[j] = d cum_i[j] + sum_{c,k} dF[c, j + half - k] * Wc[c, k]   (thread = 4 consecutive j, a quarter of c)
    {
        const int njg = Lp / 4;
        for (int t = tid; t < njg * 4; t += ATT_THREADS) {
            const int jg = t % njg, cq = t / njg, j0 = jg * 4;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            for (int c = cq; c < C; c += 4) {
                const float* row = dF + c * dFld + K + half;     // row[j - k] = dF[c, j + half - k]; zero padding covers out-of-range
                float d1 = row[j0 + 1], d2 = row[j0 + 2], d3 = row[j0 + 3];
                for (int k = 0; k < K; ++k) {
                    const float d0 = row[j0 - k];
                    const float wv = Wcs[c * K + k];
                    a0 = fmaf(d0, wv, a0); a1 = fmaf(d1, wv, a1); a2 = fmaf(d2, wv, a2); a3 = fmaf(d3, wv, a3);
                    d3 = d2; d2 = d1; d1 = d0;
                }
            }
            cred[cq * Lp + j0] = a0; cred[cq * Lp + j0 + 1] = a1; cred[cq * Lp + j0 + 2] = a2; cred[cq * Lp + j0 + 3] = a3;
        }
    }
    __syncthreads();
    for (int j = tid; j < L; j += ATT_THREADS) {
        const float conv = cred[j] + cred[Lp + j] + cred[2 * Lp + j] + cred[3 * Lp + j];
        const float prev = p.last ? 0.f : p.dcum[(size_t)b * L + j];
        p.dcum[(size_t)b * L + j] = prev + conv;
    }
}

// ---------------------------------------------------------------------------------------------
// Forward-attention step backward (modules/attention.py:89-124), one CTA per utterance.  Recomputes the transition
// probabilities from the saved query and alpha (no energy storage) with the forward's own code (fwd_att_transition), so
// the clamp decisions match the forward bit for bit.  Chain: w = c / S  ->  c = clamp(a, 1e-6) (gradient where a >= 1e-6)
// -> a = 0 beyond the length (in-place mask: no gradient) -> a = (alpha + alpha shifted) * s -> softmax -> tanh energies.
// ---------------------------------------------------------------------------------------------
struct FwdAttnBwdArgs {
    const float* q;            // [B, A] saved query of this step
    const float* memT;         // [B, L, A]
    const float* memory;       // [B, L, M]
    const int* lengths;
    const float* bias; const float* v;
    const float* alpha_prev;   // [B, L] alpha the step consumed
    const float* w;  long long w_bstride;            // &align[0, i, 0] (= the alpha the step produced)
    const float* dalign; long long dalign_bstride;   // &d_align[0, i, 0] or null
    const float* dctx_static;  // [B, M]
    const float* part; int nsplit; size_t part_stride; int ld_part;   // recurrent d ctx partials (cols [0, M)); null on last step
    float* dalpha;             // [B, L] in: d alpha_{i+1}, out: d alpha_i
    float* dctx_tot;           // [B, M] out
    float* dq;                 // [B, A] out
    float* dmemT;              // [B, L, A] +=
    float* dv_acc;             // [B, A] +=  (per-utterance partials, reduced over the batch in a fixed order afterwards)
    int B, L, M, A, last;
};

static inline size_t fwd_attn_bwd_smem_floats(int L, int M, int A) {
    const size_t Lp = (L + 3) & ~3;
    return (size_t)2 * A + 3 * Lp + 64 + ((M + 3) & ~3) + (size_t)(ATT_THREADS / 32) * A;
}

__global__ void __launch_bounds__(ATT_THREADS) fwd_attn_bwd_kernel(const FwdAttnBwdArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = ATT_THREADS / 32;
    const int L = p.L, A = p.A, M = p.M, Lp = (L + 3) & ~3;
    float* qb = sm; float* vv = qb + A;
    float* s = vv + A; float* g = s + Lp; float* da = g + Lp;
    float* red = da + Lp; float* dctx = red + 64; float* cred = dctx + ((M + 3) & ~3);
    int len = p.lengths[b];
    len = len < 0 ? 0 : (len > L ? L : len);
    const float* alpha = p.alpha_prev + (size_t)b * L;
    const float* w = p.w + (size_t)b * p.w_bstride;

    // ---- phase 1: stage q + bias, v, d context ----
    for (int a = tid; a < A; a += ATT_THREADS) { qb[a] = p.q[(size_t)b * A + a] + p.bias[a]; vv[a] = p.v[a]; }
    for (int m = tid; m < M; m += ATT_THREADS) {
        float gm = p.dctx_static[(size_t)b * M + m];
        if (!p.last)
            for (int k = 0; k < p.nsplit; ++k) gm += p.part[k * p.part_stride + (size_t)b * p.ld_part + m];
        dctx[m] = gm;
        p.dctx_tot[(size_t)b * M + m] = gm;
    }
    __syncthreads();

    // ---- phase 2: transition probabilities s (recomputed); d w[l] = d align + d alpha_{i+1} + <d ctx, memory[l]> over all L ----
    fwd_att_transition(qb, vv, p.memT + (size_t)b * L * A, L, A, s, red);
    for (int l = warp; l < L; l += NW) {
        const float* row = p.memory + ((size_t)b * L + l) * M;
        float acc = 0.f;
        for (int m = lane; m < M; m += 32) acc = fmaf(dctx[m], row[m], acc);
        acc = warp_sum(acc);
        if (lane == 0) {
            float gl = acc + (p.last ? 0.f : p.dalpha[(size_t)b * L + l]);
            if (p.dalign) gl += p.dalign[(size_t)b * p.dalign_bstride + l];
            g[l] = gl;
        }
    }
    __syncthreads();

    // ---- phase 3: L1 normalisation and clamp: d c = (d w - <d w, w>) / S;  d a = d c where l < len and a >= 1e-6 ----
    float dot = 0.f, csum = 0.f;
    for (int l = tid; l < L; l += ATT_THREADS) {
        dot = fmaf(g[l], w[l], dot);
        csum += fmaxf(fwd_att_product(alpha, s, l, len), FWD_ATT_FLOOR);
    }
    dot = block_sum(dot, red);
    const float denom = fmaxf(block_sum(csum, red), FWD_ATT_NORM_EPS);
    for (int l = tid; l < L; l += ATT_THREADS) {
        const float a = fwd_att_product(alpha, s, l, len);
        da[l] = (l < len && a >= FWD_ATT_FLOOR) ? (g[l] - dot) / denom : 0.f;
    }
    __syncthreads();

    // ---- phase 4: the product: d alpha[l] = d a[l] s[l] + d a[l+1] s[l+1];  d s[l] = d a[l] (alpha[l] + alpha[l-1]) ----
    float sds = 0.f;
    for (int l = tid; l < L; l += ATT_THREADS) {
        const float dnext = l + 1 < L ? da[l + 1] * s[l + 1] : 0.f;
        p.dalpha[(size_t)b * L + l] = fmaf(da[l], s[l], dnext);
        const float ds = da[l] * (alpha[l] + (l > 0 ? alpha[l - 1] : 0.f));
        g[l] = ds;
        sds = fmaf(s[l], ds, sds);
    }
    // softmax backward: d e[l] = s[l] (d s[l] - <s, d s>)
    sds = block_sum(sds, red);
    for (int l = tid; l < L; l += ATT_THREADS) g[l] = s[l] * (g[l] - sds);
    __syncthreads();

    // ---- phase 5: energy backward over every position: d pre = d e v (1 - tanh^2) -> d q, d memT; d v += d e tanh ----
    float dq_reg[4] = {0.f, 0.f, 0.f, 0.f}, dv_reg[4] = {0.f, 0.f, 0.f, 0.f};
    for (int l = warp; l < L; l += NW) {
        const float del = g[l];
        const size_t row = ((size_t)b * L + l) * A;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int a = lane + 32 * j;
            if (a < A) {
                const float th = tanhf(qb[a] + p.memT[row + a]);
                const float dpre = del * vv[a] * (1.f - th * th);
                dv_reg[j] = fmaf(del, th, dv_reg[j]);
                dq_reg[j] += dpre;
                p.dmemT[row + a] += dpre;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int a = lane + 32 * j;
        if (a < A) cred[warp * A + a] = dq_reg[j];
    }
    __syncthreads();
    for (int a = tid; a < A; a += ATT_THREADS) {
        float acc = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < NW; ++w8) acc += cred[w8 * A + a];
        p.dq[(size_t)b * A + a] = acc;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int a = lane + 32 * j;
        if (a < A) cred[warp * A + a] = dv_reg[j];
    }
    __syncthreads();
    for (int a = tid; a < A; a += ATT_THREADS) {
        float acc = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < NW; ++w8) acc += cred[w8 * A + a];
        p.dv_acc[(size_t)b * A + a] += acc;
    }
}

}  // namespace
int launch_cell_bwd(const CellBwdArgs& a, cudaStream_t st) {
    const int Bp = (a.B + 7) & ~7;
    const size_t smem = a.dq ? ((size_t)a.A * Bp + (size_t)a.A * (CELL_UNITS + 1)) * sizeof(float) : 0;
    static size_t configured = 48 * 1024;
    if (smem > configured) {
        B200_CUDA(cudaFuncSetAttribute(lstm_cell_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    lstm_cell_bwd_kernel<<<cdiv(a.D, CELL_UNITS), 256, smem, st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}
namespace {

int pick_attn_bwd_chunk(int L, int M, int A, int C, int K) {
    const int Lp = (L + 3) & ~3;
    int LC = Lp;
    while (LC > 4 && (size_t)attn_bwd_smem(L, M, A, C, K, LC).total * sizeof(float) > 220 * 1024) LC -= 4;
    return LC;
}

int launch_attn_bwd(AttnBwdArgs a, cudaStream_t st) {
    a.LC = pick_attn_bwd_chunk(a.L, a.M, a.A, a.C, a.K);
    const size_t smem = (size_t)attn_bwd_smem(a.L, a.M, a.A, a.C, a.K, a.LC).total * sizeof(float);
    B200_REQUIRE(smem <= 227 * 1024, "attention backward: shared memory %zu B exceeds 227 KB (L=%d)", smem, a.L);
    static size_t configured = 48 * 1024;
    if (smem > configured) {
        B200_CUDA(cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    attn_bwd_kernel<<<a.B, ATT_THREADS, smem, st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int launch_fwd_attn_bwd(const FwdAttnBwdArgs& a, cudaStream_t st) {
    const size_t smem = fwd_attn_bwd_smem_floats(a.L, a.M, a.A) * sizeof(float);
    B200_REQUIRE(smem <= 227 * 1024, "forward attention backward: shared memory %zu B exceeds 227 KB (L=%d)", smem, a.L);
    static size_t configured = 48 * 1024;
    if (smem > configured) {
        B200_CUDA(cudaFuncSetAttribute(fwd_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    fwd_attn_bwd_kernel<<<a.B, ATT_THREADS, smem, st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

// ---------------------------------------------------------------------------------------------
// backward workspace
// ---------------------------------------------------------------------------------------------
struct BwdLayout {
    size_t dfs, dhgd, dctxs, dgg, dhas, dga, dq, dctxt, dcum, dc, dhz, dmemT, dWloc_acc, dWc_acc, dv_acc, dp1, dp0, dwfs,
        part, gpart, pextra, pextra2, dggb, dgab,     // dggb / dgab: bf16 [T, B, 4D] histories of the gate gradients (wgmma loops)
        part_gen, dc_gen, dhz_gen,      // generator-recurrence state of the segmented sweep (inside the dgab region)
        total;
    int split_gen, split_att;
    size_t gpart_elems;
};

BwdLayout bwd_layout(const b200tts_decoder_shape& s) {
    BwdLayout l;
    size_t off = 0;
    auto take = [&](size_t n) { size_t o = off; off = align_up(off + n, 64); return o; };
    const size_t T = s.T, B = s.B, D = s.D, M = s.M, P = s.P, A = s.A, L = s.L, W = fs_width(s);
    const size_t C = forward_attention(s) ? 0 : s.C, K = forward_attention(s) ? 0 : s.K;     // ignored for forward attention
    l.dfs = take(T * B * W);
    l.dhgd = take(T * B * D);
    l.dctxs = take(T * B * M);
    l.dgg = take(T * B * 4 * D);
    l.dhas = take(T * B * D);
    l.dga = take(T * B * 4 * D);
    l.dq = take(T * B * A);
    l.dctxt = take(T * B * M);
    l.dcum = take(B * L);
    l.dc = take(B * D);
    l.dhz = take(B * D);
    l.dmemT = take(B * L * A);
    l.dWloc_acc = take(B * A * C);
    l.dWc_acc = take(B * C * K);
    l.dv_acc = take(B * A);
    l.dp1 = take(T * B * P);
    l.dp0 = take(T * B * P);
    l.dwfs = take(W * (D + M));
    l.split_gen = pick_splitk(s.B, s.D, 4 * s.D);
    l.split_att = pick_splitk(s.B, s.M + s.D, 4 * s.D);
    const size_t pg = (size_t)l.split_gen * B * D, pa = (size_t)l.split_att * B * (M + D);
    l.part = take(pg > pa ? pg : pa);
    // scratch for the split-K partials of the long-K weight-gradient GEMMs (only small outputs are split)
    l.gpart_elems = (size_t)6 * 1024 * 1024;
    l.gpart = take(l.gpart_elems);
    l.pextra = take(persist_bwd_gen_extra_bytes(s) / sizeof(float) + 64);
    l.pextra2 = take(att_bwd_extra(s).total / sizeof(float) + 64);
    l.dggb = take(T * B * 4 * D / 2 + 64);
    // The segmented sweep (decodes with free-running steps) runs both recurrences in turn with state carried across segments: the
    // attention recurrence keeps part / dc / dhz, the generator gets its own.  That sweep never runs the persistent attention reverse
    // loop, the only writer of dgab, so its generator state lives in the dgab region (grown only where T < 5 leaves it too small).
    const size_t seg_gen = align_up(pg, 64) + 2 * align_up(B * D, 64);
    const size_t ngab = T * B * 4 * D / 2 + 64;
    l.dgab = take(ngab > seg_gen ? ngab : seg_gen);
    l.part_gen = l.dgab;
    l.dc_gen = l.part_gen + align_up(pg, 64);
    l.dhz_gen = l.dc_gen + align_up(B * D, 64);
    l.total = off;
    return l;
}

// C (+)= op(A) . op(B), split-K chosen from the tile count; partial scratch shared by all calls
struct PackScope {
    PackScope() { tc_pack_cache_begin(); }
    ~PackScope() { tc_pack_cache_end(); }
};

int wgemm(cudaStream_t st, const BwdLayout& l, float* ws, int transA, int transB, int M, int N, int K, const float* A, int lda,
          const float* B, int ldb, float* C, int ldc, float beta, int batch = 1, long long sA = 0, long long sB = 0,
          long long sC = 0) {
    GemmDesc d;
    d.A = A; d.B = B; d.C = C; d.M = M; d.N = N; d.K = K; d.lda = lda; d.ldb = ldb; d.ldc = ldc; d.transA = transA;
    d.transB = transB; d.beta = beta; d.batch = batch; d.strideA = sA; d.strideB = sB; d.strideC = sC;
    return gemm_run_auto(d, ws + l.gpart, l.gpart_elems, st);
}
// weight gradient dW (+)= A^T . B with A [K, M] fp32 and B [K, N] fp32; B16 (optional) = the same B as bf16 rows (row stride ldb16) that
// the persistent forward loops left behind: read in place by the wgmma path (MN-major TMA operand), no conversion pass
int wgemm16(cudaStream_t st, const BwdLayout& l, float* ws, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
            const void* B16, int ldb16, float* C, int ldc, float beta, const void* A16 = nullptr, int lda16 = 0) {
    GemmDesc d;
    d.A = A; d.B = B; d.C = C; d.M = M; d.N = N; d.K = K; d.lda = lda; d.ldb = ldb; d.ldc = ldc; d.transA = 1; d.transB = 0; d.beta = beta;
    d.B16 = B16; d.ldb16 = ldb16; d.A16 = A16; d.lda16 = lda16;
    return gemm_run_auto(d, ws + l.gpart, l.gpart_elems, st);
}
// input gradient dX = A . B with A [M, K] fp32 (A16: the same matrix as bf16 rows, read in place) and B [K, N] fp32
int xgemm16(cudaStream_t st, const BwdLayout& l, float* ws, int M, int N, int K, const float* A, int lda, const void* A16, int lda16,
            const float* B, int ldb, float* C, int ldc, float beta) {
    GemmDesc d;
    d.A = A; d.B = B; d.C = C; d.M = M; d.N = N; d.K = K; d.lda = lda; d.ldb = ldb; d.ldc = ldc; d.transA = 0; d.transB = 0; d.beta = beta;
    d.A16 = A16; d.lda16 = lda16;
    return gemm_run_auto(d, ws + l.gpart, l.gpart_elems, st);
}

// ---------------------------------------------------------------------------------------------
// pieces of one decoder backward call, shared by the teacher-forced path and the segmented sweep
// ---------------------------------------------------------------------------------------------
struct BwdCtx {
    const b200tts_decoder_shape& s;
    const b200tts_decoder_params& w;
    const b200tts_decoder_inputs& in;
    const b200tts_decoder_outputs& fwd_out;
    const b200tts_decoder_output_grads& dout;
    const DecoderLayout& fl;
    const BwdLayout& l;
    const float* fws;
    float* bws;
    cudaStream_t st;
    const float* F(size_t off) const { return fws + off; }
    float* W(size_t off) const { return bws + off; }
    bool free_running(int i) const { return in.teacher && !in.teacher[i]; }
};

// d [frame_w ; stop_w] = dFS^T . [h_gen | ctx];  d frame_b, d stop_b = column sums of dFS
int frame_weight_grads(const BwdCtx& c, const b200tts_decoder_params& dw, const __nv_bfloat16* hgb1, int ldhb,
                       const __nv_bfloat16* aib1, int ldab) {
    const auto& s = c.s; const auto& l = c.l;
    const int D = s.D, M = s.M, RN = s.R * s.N, N1 = fs_width(s), MD = M + D;
    const size_t TB = (size_t)s.T * s.B;
    const float* ai1 = c.F(c.fl.ai) + (size_t)s.B * MD;
    B200_TRY(wgemm16(c.st, l, c.bws, N1, D, (int)TB, c.W(l.dfs), N1, c.F(c.fl.hg) + (size_t)s.B * D, D, hgb1, ldhb, c.W(l.dwfs), D + M, 0.f));
    B200_TRY(wgemm16(c.st, l, c.bws, N1, M, (int)TB, c.W(l.dfs), N1, ai1, MD, aib1 ? aib1 + D : nullptr, ldab, c.W(l.dwfs) + D, D + M, 0.f));
    add2d_kernel<<<grid_for((size_t)RN * (D + M)), 256, 0, c.st>>>(dw.frame_w, D + M, c.W(l.dwfs), D + M, RN, D + M);
    B200_LAUNCH_CHECK();
    add2d_kernel<<<grid_for((size_t)s.R * (D + M)), 256, 0, c.st>>>(dw.stop_w, D + M, c.W(l.dwfs) + (size_t)RN * (D + M), D + M, s.R, D + M);
    B200_LAUNCH_CHECK();
    B200_TRY(colsum_add(dw.frame_b, nullptr, c.W(l.dfs), TB, RN, N1, c.W(l.gpart), c.st));
    B200_TRY(colsum_add(dw.stop_b, nullptr, c.W(l.dfs) + RN, TB, s.R, N1, c.W(l.gpart), c.st));
    return B200TTS_OK;
}

// generator-LSTM reverse step i on the per-step chain: cell backward (carried d c / zoneout d h in dc / dhz), then the recurrent
// d h_gen_{i-1} = dgates_i . W_hh as split-K partials into `part`, which step i-1 consumes
int gen_bwd_step(const BwdCtx& c, int i, float* part, float* dc, float* dhz) {
    const auto& s = c.s; const auto& l = c.l;
    const int B = s.B, D = s.D;
    const size_t BD = (size_t)B * D, B4D = 4 * BD;
    CellBwdArgs ca{};
    ca.gates = c.F(c.fl.gg) + (size_t)i * B4D;
    ca.c_prev = c.F(c.fl.cg) + (size_t)i * BD;
    ca.dh_static = c.W(l.dhgd) + (size_t)i * BD; ca.ld_dhs = D;
    ca.part = part; ca.nsplit = l.split_gen; ca.part_stride = BD; ca.ld_part = D; ca.part_col0 = 0;
    ca.dq = nullptr; ca.Wq = nullptr; ca.A = 0;
    ca.dc_state = dc; ca.dhz_state = s.cell_kind == B200TTS_CELL_ZONEOUT ? dhz : nullptr;
    ca.mask_h = c.in.mask_gen_h ? c.in.mask_gen_h + (size_t)i * BD : nullptr;
    ca.mask_c = c.in.mask_gen_c ? c.in.mask_gen_c + (size_t)i * BD : nullptr;
    ca.kind = s.cell_kind; ca.training = s.training; ca.rate_h = s.rate_h; ca.rate_c = s.rate_c;
    ca.dgates = c.W(l.dgg) + (size_t)i * B4D; ca.B = B; ca.D = D; ca.last = (i == s.T - 1);
    B200_TRY(launch_cell_bwd(ca, c.st));
    if (i > 0) {
        GemmDesc d;      // d h_gen_{i-1} (recurrent) = dgates_i . W_hh
        d.A = ca.dgates; d.lda = 4 * D; d.B = c.w.gen_w_hh; d.ldb = D; d.transB = 0; d.M = B; d.N = D; d.K = 4 * D;
        d.splitk = l.split_gen; d.partial = part; d.keep_partials = 1;
        if (d.splitk == 1) { d.C = part; d.ldc = D; d.keep_partials = 0; d.partial = nullptr; }
        B200_TRY(gemm_run(d, c.st));
    }
    return B200TTS_OK;
}

// time-batched generator-LSTM weight gradients from the final gate gradients (dggb: their bf16 history, or null)
int gen_weight_grads(const BwdCtx& c, const b200tts_decoder_params& dw, const __nv_bfloat16* hgb, int ldhb, const __nv_bfloat16* aib1,
                     int ldab, const void* dggb) {
    const auto& s = c.s; const auto& l = c.l;
    const int D = s.D, M = s.M, MD = M + D;
    const size_t TB = (size_t)s.T * s.B;
    const float* ai1 = c.F(c.fl.ai) + (size_t)s.B * MD;
    B200_TRY(wgemm16(c.st, l, c.bws, 4 * D, D, (int)TB, c.W(l.dgg), 4 * D, c.F(c.fl.hg), D, hgb, ldhb, dw.gen_w_hh, D, 1.f, dggb, 4 * D));
    B200_TRY(wgemm16(c.st, l, c.bws, 4 * D, D, (int)TB, c.W(l.dgg), 4 * D, ai1 + M, MD, aib1, ldab, dw.gen_w_ih, D + M, 1.f, dggb, 4 * D));
    B200_TRY(wgemm16(c.st, l, c.bws, 4 * D, M, (int)TB, c.W(l.dgg), 4 * D, ai1, MD, aib1 ? aib1 + D : nullptr, ldab, dw.gen_w_ih + D, D + M, 1.f,
                     dggb, 4 * D));
    B200_TRY(colsum_add(dw.gen_b_ih, dw.gen_b_hh, c.W(l.dgg), TB, 4 * D, 4 * D, c.W(l.gpart), c.st));
    return B200TTS_OK;
}

// d h_att (static part) and d ctx (generator-input part, accumulated onto what is there) of steps [i0, i1)
int gen_input_grads(const BwdCtx& c, int i0, int i1, const void* dggb) {
    const auto& s = c.s; const auto& l = c.l;
    const int B = s.B, D = s.D, M = s.M;
    const int rows = (i1 - i0) * B;
    const float* dgg = c.W(l.dgg) + (size_t)i0 * B * 4 * D;
    const void* dgg16 = dggb ? static_cast<const void*>(static_cast<const __nv_bfloat16*>(dggb) + (size_t)i0 * B * 4 * D) : nullptr;
    B200_TRY(xgemm16(c.st, l, c.bws, rows, D, 4 * D, dgg, 4 * D, dgg16, 4 * D, c.w.gen_w_ih, D + M, c.W(l.dhas) + (size_t)i0 * B * D, D, 0.f));
    B200_TRY(xgemm16(c.st, l, c.bws, rows, M, 4 * D, dgg, 4 * D, dgg16, 4 * D, c.w.gen_w_ih + D, D + M, c.W(l.dctxs) + (size_t)i0 * B * M, M, 1.f));
    return B200TTS_OK;
}

// zero the accumulators of the attention reverse steps on the per-step chains
int att_chain_init(const BwdCtx& c) {
    const auto& s = c.s; const auto& l = c.l;
    B200_TRY(launch_fill(c.W(l.dmemT), 0.f, (size_t)s.B * s.L * s.A, c.st));
    if (!forward_attention(s)) {
        B200_TRY(launch_fill(c.W(l.dWloc_acc), 0.f, (size_t)s.B * s.A * s.C, c.st));
        B200_TRY(launch_fill(c.W(l.dWc_acc), 0.f, (size_t)s.B * s.C * s.K, c.st));
    }
    B200_TRY(launch_fill(c.W(l.dv_acc), 0.f, (size_t)s.B * s.A, c.st));
    return B200TTS_OK;
}

// attention reverse step i on the per-step chain: attention backward (d cum / d alpha carried in dcum), attention-LSTM cell backward
// (carried state in dc / dhz), then the recurrent [d ctx_{i-1} | d h_att_{i-1}] = dgates_i . [W_ih[:, P:] | W_hh] as split-K partials
// into `part`, which step i-1 consumes
int att_bwd_step(const BwdCtx& c, int i, float* part, float* dc, float* dhz) {
    const auto& s = c.s; const auto& l = c.l; const auto& fl = c.fl; const auto& w = c.w;
    const int B = s.B, T = s.T, D = s.D, M = s.M, A = s.A, L = s.L, MD = M + D;
    const size_t BD = (size_t)B * D, B4D = 4 * BD;
    const int last = (i == T - 1);
    if (forward_attention(s)) {
        FwdAttnBwdArgs fa{};
        fa.q = c.F(fl.q) + (size_t)i * B * A; fa.memT = c.F(fl.memT); fa.memory = c.in.memory; fa.lengths = c.in.text_lengths;
        fa.bias = w.attn_bias; fa.v = w.attn_energy;
        fa.alpha_prev = c.F(fl.cum) + (size_t)i * B * L;
        fa.w = c.fwd_out.alignments + (size_t)i * L; fa.w_bstride = (long long)T * L;
        fa.dalign = c.dout.d_alignments ? c.dout.d_alignments + (size_t)i * L : nullptr; fa.dalign_bstride = (long long)T * L;
        fa.dctx_static = c.W(l.dctxs) + (size_t)i * B * M;
        fa.part = part; fa.nsplit = l.split_att; fa.part_stride = (size_t)B * MD; fa.ld_part = MD;
        fa.dalpha = c.W(l.dcum); fa.dctx_tot = c.W(l.dctxt) + (size_t)i * B * M; fa.dq = c.W(l.dq) + (size_t)i * B * A;
        fa.dmemT = c.W(l.dmemT); fa.dv_acc = c.W(l.dv_acc);
        fa.B = B; fa.L = L; fa.M = M; fa.A = A; fa.last = last;
        B200_TRY(launch_fwd_attn_bwd(fa, c.st));
    } else {
        AttnBwdArgs aa{};
        aa.q = c.F(fl.q) + (size_t)i * B * A; aa.memT = c.F(fl.memT); aa.memory = c.in.memory; aa.lengths = c.in.text_lengths;
        aa.Wc = w.attn_loc_features; aa.Wloc = w.attn_location; aa.bias = w.attn_bias; aa.v = w.attn_energy;
        aa.cum_prev = c.F(fl.cum) + (size_t)i * B * L;
        aa.w = c.fwd_out.alignments + (size_t)i * L; aa.w_bstride = (long long)T * L;
        aa.dalign = c.dout.d_alignments ? c.dout.d_alignments + (size_t)i * L : nullptr; aa.dalign_bstride = (long long)T * L;
        aa.dctx_static = c.W(l.dctxs) + (size_t)i * B * M;
        aa.part = part; aa.nsplit = l.split_att; aa.part_stride = (size_t)B * MD; aa.ld_part = MD;
        aa.dcum = c.W(l.dcum); aa.dctx_tot = c.W(l.dctxt) + (size_t)i * B * M; aa.dq = c.W(l.dq) + (size_t)i * B * A;
        aa.dmemT = c.W(l.dmemT); aa.dWloc_acc = c.W(l.dWloc_acc); aa.dWc_acc = c.W(l.dWc_acc); aa.dv_acc = c.W(l.dv_acc);
        aa.B = B; aa.L = L; aa.M = M; aa.A = A; aa.C = s.C; aa.K = s.K; aa.last = last;
        B200_TRY(launch_attn_bwd(aa, c.st));
    }

    CellBwdArgs ca{};
    ca.gates = c.F(fl.ga) + (size_t)i * B4D;
    ca.c_prev = c.F(fl.ca) + (size_t)i * BD;
    ca.dh_static = c.W(l.dhas) + (size_t)i * BD; ca.ld_dhs = D;
    ca.part = part; ca.nsplit = l.split_att; ca.part_stride = (size_t)B * MD; ca.ld_part = MD; ca.part_col0 = M;
    ca.dq = c.W(l.dq) + (size_t)i * B * A; ca.Wq = w.attn_query; ca.A = A;
    ca.dc_state = dc; ca.dhz_state = s.cell_kind == B200TTS_CELL_ZONEOUT ? dhz : nullptr;
    ca.mask_h = c.in.mask_att_h ? c.in.mask_att_h + (size_t)i * BD : nullptr;
    ca.mask_c = c.in.mask_att_c ? c.in.mask_att_c + (size_t)i * BD : nullptr;
    ca.kind = s.cell_kind; ca.training = s.training; ca.rate_h = s.rate_h; ca.rate_c = s.rate_c;
    ca.dgates = c.W(l.dga) + (size_t)i * B4D; ca.B = B; ca.D = D; ca.last = last;
    B200_TRY(launch_cell_bwd(ca, c.st));
    if (i > 0) {
        GemmDesc d;      // [d ctx_{i-1} | d h_att_{i-1}] (recurrent) = dgates_i . [W_ih[:, P:] | W_hh]
        d.A = ca.dgates; d.lda = 4 * D; d.B = c.F(fl.wcat_att); d.ldb = MD; d.transB = 0; d.M = B; d.N = MD; d.K = 4 * D;
        d.splitk = l.split_att; d.partial = part; d.keep_partials = 1;
        if (d.splitk == 1) { d.C = part; d.ldc = MD; d.keep_partials = 0; d.partial = nullptr; }
        B200_TRY(gemm_run(d, c.st));
    }
    return B200TTS_OK;
}

// dropout scale of the prenet layer whose keep masks are `mask` (NULL: no dropout there)
inline float prenet_scale(const b200tts_decoder_shape& s, const uint8_t* mask) { return mask ? 1.f / (1.f - s.prenet_rate) : 1.f; }

// relu + dropout backward of one prenet layer over all T steps, in place on dz [T, B, P].  Teacher-forced steps were dropped with the
// time-batched masks (mask_tf), free-running steps with the per-step masks (mask_fr); a caller may pass either set without the other,
// so each maximal run of steps with one scale gets one launch (a teacher-forced decode: a single launch over every row).
int prenet_relu_bwd(const BwdCtx& c, float* dz, const float* y, const uint8_t* mask_tf, const uint8_t* mask_fr) {
    const auto& s = c.s;
    const size_t BP = (size_t)s.B * s.P;
    const float scale_tf = prenet_scale(s, mask_tf), scale_fr = prenet_scale(s, mask_fr);
    auto scale_of = [&](int i) { return c.free_running(i) ? scale_fr : scale_tf; };
    for (int i0 = 0; i0 < s.T;) {
        const float scale = scale_of(i0);
        int i1 = i0 + 1;
        while (i1 < s.T && scale_of(i1) == scale) ++i1;
        const size_t n = (size_t)(i1 - i0) * BP;
        relu_dropout_bwd_kernel<<<grid_for(n), 256, 0, c.st>>>(dz + (size_t)i0 * BP, dz + (size_t)i0 * BP, y + (size_t)i0 * BP, scale, n);
        B200_LAUNCH_CHECK();
        i0 = i1;
    }
    return B200TTS_OK;
}

// feedback of free-running step f >= 1 into row f-1: d p1_f = dga_f . W_ih_att[:, :P] (long K = 4D: the GEMM, into row f of dp1, which
// the time-batched prenet pass rewrites later), then the rest of the chain in frame_feedback_bwd_kernel
int frame_feedback(const BwdCtx& c, int f) {
    const auto& s = c.s; const auto& l = c.l;
    const int B = s.B, D = s.D, M = s.M, P = s.P, N = s.N, W = fs_width(s), last = (s.R - 1) * N;
    float* dp1 = c.W(l.dp1) + (size_t)f * B * P;
    B200_TRY(xgemm16(c.st, l, c.bws, B, P, 4 * D, c.W(l.dga) + (size_t)f * B * 4 * D, 4 * D, nullptr, 0, c.w.att_w_ih, P + M, dp1, P, 0.f));
    FeedbackArgs a{};
    a.dp1 = dp1;
    a.p0 = c.F(c.fl.p0) + (size_t)f * B * P; a.p1 = c.F(c.fl.p1) + (size_t)f * B * P;
    a.W0 = c.w.prenet_w0; a.W1 = c.w.prenet_w1; a.wfs = c.F(c.fl.wfs) + (size_t)last * (D + M);
    a.dfs = c.W(l.dfs) + (size_t)(f - 1) * B * W + last; a.ld_fs = W;
    a.dhgd = c.W(l.dhgd) + (size_t)(f - 1) * B * D;
    a.dctxs = c.W(l.dctxs) + (size_t)(f - 1) * B * M;
    a.scale0 = prenet_scale(s, c.in.mask_step_prenet0); a.scale1 = prenet_scale(s, c.in.mask_step_prenet1);
    a.B = B; a.P = P; a.N = N; a.D = D; a.M = M;
    const size_t smem = feedback_smem_floats(P, N) * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "decoder_backward: frame feedback needs %zu B of shared memory (P=%d N=%d)", smem, P, N);
    frame_feedback_bwd_kernel<<<B, FEEDBACK_THREADS, smem, c.st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // namespace

static int attention_step_backward_validate(int B, int L, int M, int A, int C, int K) {
    B200_REQUIRE(B > 0 && L > 0 && M > 0 && A > 0 && C > 0 && K > 0, "attention_step_backward: non-positive dimension (B=%d L=%d M=%d A=%d C=%d K=%d)",
                 B, L, M, A, C, K);
    B200_REQUIRE(A <= 128 && A % 4 == 0 && C % 4 == 0 && (A / 4) * (C / 4) <= ATT_THREADS && M <= 512 && (K % 2) == 1,
                 "attention_step_backward: unsupported dims A=%d C=%d M=%d K=%d", A, C, M, K);
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

// The three decoder queries below answer for the step shape (T -> ceil(T / R) steps) that the forward and backward calls run on.
size_t b200tts_decoder_bwd_workspace_bytes(const b200tts_decoder_shape* shape) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    return bwd_layout(step_shape(*shape)).total * sizeof(float);
}

// byte offset of the phase counters of the persistent backward kernels inside the backward workspace (0: generator, 1: attention)
size_t b200tts_debug_persist_bwd_profile_offset(const b200tts_decoder_shape* shape, int which) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    const b200tts_decoder_shape s = step_shape(*shape);
    const BwdLayout l = bwd_layout(s);
    if (which == 0) return l.pextra * sizeof(float) + persist_bwd_gen_extra_bytes(s) - NUM_SMS * 8 * 8;
    return l.pextra2 * sizeof(float) + att_bwd_extra(s).barrier + 256;
}

int b200tts_debug_decoder_views(const b200tts_decoder_shape* shape, size_t* out, int n) {
    if (!shape || !out || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    const b200tts_decoder_shape s = step_shape(*shape);
    const DecoderLayout l = decoder_layout(s);
    const PersistLayout pl = persist_layout(s);
    const TcPersistGeom g = tc_persist_geom(s);
    const BwdLayout bl = bwd_layout(s);
    const size_t pbase = l.persist * sizeof(float);
    size_t v[30];
    const size_t fwd[11] = {l.ai, l.ca, l.hg, l.cg, l.ga, l.gg, l.q, l.cum, l.memT, l.fs, l.p1};
    for (int k = 0; k < 11; ++k) v[k] = fwd[k] * sizeof(float);
    v[11] = pbase + pl.aib;
    v[12] = pbase + pl.hgb;
    // the per-step histories of the backward workspace: dfs, dhgd, dctxs, dgg, dhas, dga, dq, dctxt, dmemT, dggb, dgab
    const size_t bwd[11] = {bl.dfs, bl.dhgd, bl.dctxs, bl.dgg, bl.dhas, bl.dga, bl.dq, bl.dctxt, bl.dmemT, bl.dggb, bl.dgab};
    for (int k = 0; k < 11; ++k) v[13 + k] = bwd[k] * sizeof(float);
    v[24] = (size_t)g.Kp_att;
    v[25] = (size_t)g.Kp_gen;
    // the prenet's rows, appended so that the indices above keep their meaning: its input and first layer (forward), and the
    // gradients of both layers after the relu / dropout backward, which works in place (backward)
    v[26] = l.xtm * sizeof(float);
    v[27] = l.p0 * sizeof(float);
    v[28] = bl.dp1 * sizeof(float);
    v[29] = bl.dp0 * sizeof(float);
    const int m = n < 30 ? n : 30;
    for (int k = 0; k < m; ++k) out[k] = v[k];
    return m;
}

// standalone backward of one attention step (module-level API): per-utterance accumulators in the workspace, reduced over the batch here
size_t b200tts_attention_step_backward_workspace_elems(int B, int M, int A, int C, int K) {
    return (size_t)B * ((size_t)A * C + (size_t)C * K + A + M);
}
// the per-chunk position count LC launch_attn_bwd runs these dims with, or 0 when not even 4-row chunks fit in shared memory
int b200tts_debug_attention_backward_chunk(int L, int M, int A, int C, int K) {
    if (attention_step_backward_validate(1, L, M, A, C, K) != B200TTS_OK) return 0;
    const int LC = pick_attn_bwd_chunk(L, M, A, C, K);
    if ((size_t)attn_bwd_smem(L, M, A, C, K, LC).total * sizeof(float) > 227 * 1024) {
        set_last_error("attention backward: L=%d does not fit in shared memory (M=%d A=%d C=%d K=%d)", L, M, A, C, K);
        return 0;
    }
    return LC;
}
int b200tts_attention_step_backward(int B, int L, int M, int A, int C, int K, const float* q, const float* memory,
                                    const float* memory_transform, const int32_t* text_lengths, const float* w_location,
                                    const float* w_loc_features, const float* bias, const float* w_energy, const float* cum_prev,
                                    const float* weights, const float* d_context, const float* d_weights, float* d_cum, float* d_q,
                                    float* d_memory_transform, float* d_w_location, float* d_w_loc_features, float* d_w_energy,
                                    float* workspace, void* stream) {
    B200_REQUIRE(q && memory && memory_transform && text_lengths && w_location && w_loc_features && bias && w_energy && cum_prev && weights &&
                 d_context && d_cum && d_q && d_memory_transform && d_w_location && d_w_loc_features && d_w_energy && workspace,
                 "attention_step_backward: null argument");
    B200_TRY(attention_step_backward_validate(B, L, M, A, C, K));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    float* dWloc_acc = workspace;
    float* dWc_acc = dWloc_acc + (size_t)B * A * C;
    float* dv_acc = dWc_acc + (size_t)B * C * K;
    float* dctx_tot = dv_acc + (size_t)B * A;
    B200_TRY(launch_fill(workspace, 0.f, (size_t)B * ((size_t)A * C + (size_t)C * K + A), st));
    AttnBwdArgs aa{};
    aa.q = q; aa.memT = memory_transform; aa.memory = memory; aa.lengths = text_lengths;
    aa.Wc = w_loc_features; aa.Wloc = w_location; aa.bias = bias; aa.v = w_energy; aa.cum_prev = cum_prev;
    aa.w = weights; aa.w_bstride = L; aa.dalign = d_weights; aa.dalign_bstride = L;
    aa.dctx_static = d_context; aa.part = nullptr; aa.nsplit = 0; aa.part_stride = 0; aa.ld_part = 0;
    aa.dcum = d_cum; aa.dctx_tot = dctx_tot; aa.dq = d_q; aa.dmemT = d_memory_transform;
    aa.dWloc_acc = dWloc_acc; aa.dWc_acc = dWc_acc; aa.dv_acc = dv_acc;
    aa.B = B; aa.L = L; aa.M = M; aa.A = A; aa.C = C; aa.K = K; aa.last = 0;
    B200_TRY(launch_attn_bwd(aa, st));
    batchsum_add_kernel<<<grid_for((size_t)A * C), 256, 0, st>>>(d_w_location, dWloc_acc, B, (size_t)A * C);
    B200_LAUNCH_CHECK();
    batchsum_add_kernel<<<grid_for((size_t)C * K), 256, 0, st>>>(d_w_loc_features, dWc_acc, B, (size_t)C * K);
    B200_LAUNCH_CHECK();
    batchsum_add_kernel<<<1, 256, 0, st>>>(d_w_energy, dv_acc, B, (size_t)A);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

// standalone backward of one forward-attention step: per-utterance d v partials in the workspace, reduced over the batch here
size_t b200tts_forward_attention_step_backward_workspace_elems(int B, int M, int A) { return (size_t)B * ((size_t)A + M); }
int b200tts_forward_attention_step_backward(int B, int L, int M, int A, const float* q, const float* memory, const float* memory_transform,
                                            const int32_t* text_lengths, const float* bias, const float* w_energy, const float* alpha_prev,
                                            const float* weights, const float* d_context, const float* d_weights, float* d_alpha,
                                            float* d_q, float* d_memory_transform, float* d_w_energy, float* workspace, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(q && memory && memory_transform && text_lengths && bias && w_energy && alpha_prev && weights && d_context && d_alpha &&
                 d_q && d_memory_transform && d_w_energy && workspace, "forward_attention_step_backward: null argument");
    B200_REQUIRE(B > 0 && L > 0 && A > 0 && A <= 128 && M > 0 && M <= 512,
                 "forward_attention_step_backward: unsupported dims B=%d L=%d A=%d M=%d", B, L, A, M);
    cudaStream_t st = (cudaStream_t)stream;
    float* dv_acc = workspace;
    float* dctx_tot = dv_acc + (size_t)B * A;
    B200_TRY(launch_fill(dv_acc, 0.f, (size_t)B * A, st));
    FwdAttnBwdArgs fa{};
    fa.q = q; fa.memT = memory_transform; fa.memory = memory; fa.lengths = text_lengths; fa.bias = bias; fa.v = w_energy;
    fa.alpha_prev = alpha_prev; fa.w = weights; fa.w_bstride = L; fa.dalign = d_weights; fa.dalign_bstride = L;
    fa.dctx_static = d_context; fa.part = nullptr; fa.nsplit = 0; fa.part_stride = 0; fa.ld_part = 0;
    fa.dalpha = d_alpha; fa.dctx_tot = dctx_tot; fa.dq = d_q; fa.dmemT = d_memory_transform; fa.dv_acc = dv_acc;
    fa.B = B; fa.L = L; fa.M = M; fa.A = A; fa.last = 0;
    B200_TRY(launch_fwd_attn_bwd(fa, st));
    batchsum_add_kernel<<<1, 256, 0, st>>>(d_w_energy, dv_acc, B, (size_t)A);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_lstm_cell_backward(int B, int D, int cell_kind, int training, float rate_h, float rate_c, const float* gates, const float* c_prev,
                               const uint8_t* mask_h, const uint8_t* mask_c, const float* d_h, float* d_c, float* d_h_prev, float* d_gates,
                               void* stream) {
    B200_REQUIRE(B > 0 && D > 0 && gates && c_prev && d_h && d_c && d_h_prev && d_gates, "lstm_cell_backward: bad argument");
    B200_REQUIRE(cell_kind == B200TTS_CELL_DROPOUT || cell_kind == B200TTS_CELL_ZONEOUT, "lstm_cell_backward: bad cell kind %d", cell_kind);
    B200_REQUIRE(rate_h >= 0.f && rate_h < 1.f && rate_c >= 0.f && rate_c < 1.f, "lstm_cell_backward: rates must be in [0, 1)");
    B200_TRY(require_device());
    B200_CUDA(cudaMemsetAsync(d_h_prev, 0, (size_t)B * D * sizeof(float), (cudaStream_t)stream));
    CellBwdArgs a{};
    a.gates = gates; a.c_prev = c_prev; a.dh_static = d_h; a.ld_dhs = D; a.part = nullptr; a.nsplit = 0;
    a.dc_state = d_c; a.dhz_state = d_h_prev;       // in: zero recurrent term; out: the direct (zoneout) gradient of h_prev
    a.mask_h = mask_h; a.mask_c = mask_c; a.kind = cell_kind; a.training = training; a.rate_h = rate_h; a.rate_c = rate_c;
    a.dgates = d_gates; a.B = B; a.D = D; a.last = 0;
    return launch_cell_bwd(a, (cudaStream_t)stream);
}

int b200tts_decoder_backward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                             const b200tts_decoder_inputs* inputs, const b200tts_decoder_outputs* fwd_outputs,
                             const b200tts_decoder_output_grads* output_grads, const void* fwd_workspace, void* bwd_workspace,
                             size_t bwd_workspace_bytes, const b200tts_decoder_params* d_params, float* d_memory,
                             void* stream) {
    B200_REQUIRE(shape && params && inputs && fwd_outputs && output_grads && fwd_workspace && bwd_workspace && d_params,
                 "decoder_backward: null argument");
    B200_REQUIRE(shape->att_window_back == 0 && shape->att_window_ahead == 0,
                 "decoder_backward: an attention window is for synthesis only (b200tts_decoder_forward_chunk)");
    B200_REQUIRE(!forced_inputs(*inputs), "decoder_backward: forced attention rows are for synthesis only (b200tts_decoder_forward_chunk)");
    B200_TRY(require_device());
    const b200tts_decoder_shape& frames = *shape;
    const b200tts_decoder_params& w = *params;
    const b200tts_decoder_params& dw = *d_params;
    const b200tts_decoder_inputs& in = *inputs;
    const b200tts_decoder_outputs& fwd_out = *fwd_outputs;
    const b200tts_decoder_output_grads& dout = *output_grads;
    const float* fws = static_cast<const float*>(fwd_workspace);
    float* bws = static_cast<float*>(bwd_workspace);
    const size_t bws_bytes = bwd_workspace_bytes;
    cudaStream_t st = (cudaStream_t)stream;
    B200_TRY(validate_decoder_shape(frames));
    const b200tts_decoder_shape s = step_shape(frames);     // T = decoder steps from here on; frames.T = target frames
    B200_REQUIRE(fwd_out.alignments, "decoder_backward: the forward alignments tensor is required");
    B200_REQUIRE(s.att_extent == 0, "decoder_backward: att_extent = 1 (attention over each utterance's own length) is for inference only; "
                 "training keeps the reference's softmax over the padded extent");
    const bool fwd_att = forward_attention(s);
    B200_REQUIRE(fwd_att || (s.A % 4 == 0 && s.C % 4 == 0 && (s.A / 4) * (s.C / 4) <= ATT_THREADS),
                 "decoder_backward: attention dims A=%d C=%d unsupported (need A%%4==0, C%%4==0, A*C<=4096)", s.A, s.C);
    B200_REQUIRE(!fwd_att || (!w.attn_location && !w.attn_loc_features && !dw.attn_location && !dw.attn_loc_features),
                 "decoder_backward: forward attention has no location weights (pass NULL)");
    // a decode with a free-running step ran its forward on the per-step chains (decoder_fwd.cu) and takes the segmented sweep below
    bool free_running = false;
    if (in.teacher)
        for (int i = 0; i < s.T; ++i) free_running |= (in.teacher[i] == 0);
    const DecoderLayout fl = decoder_layout(s);
    const BwdLayout l = bwd_layout(s);
    B200_REQUIRE(bws_bytes >= l.total * sizeof(float), "decoder_backward: workspace too small (%zu < %zu bytes)", bws_bytes,
                 l.total * sizeof(float));
    const int B = s.B, T = s.T, D = s.D, M = s.M, P = s.P, N = s.N, A = s.A, L = s.L, C = s.C, K = s.K, MD = M + D, N1 = fs_width(s);
    const size_t TB = (size_t)T * B;
    auto F = [&](size_t off) { return fws + off; };
    auto W = [&](size_t off) { return bws + off; };
    const BwdCtx c{s, w, in, fwd_out, dout, fl, l, fws, bws, st};
    const float* ai = F(fl.ai);                // [T+1, B, M+D]
    const float* ai1 = ai + (size_t)B * MD;    // rows 1..T
    // the segmented sweep runs on the per-step chains only: it reads neither the persistent workspace nor the bf16 operand rows, which a
    // sequential forward never wrote
    const PersistPlan plan = precision_mode() == B200TTS_PRECISION_BF16 && !free_running ? persist_plan(s) : PersistPlan{};
    // bf16 operand rows the wgmma forward loops left in the persistent workspace: aib [T+1, B, Kp_att] = [h_att | ctx | 0], hgb [T+1, B, Kp_gen]
    // = h_gen (row i+1 = state after step i, row 0 = 0).  The weight-gradient products read them in place (MN-major TMA operands).
    // A training forward ran those loops exactly when the attention reverse loop runs.
    const PersistLayout prl = persist_layout(s);
    const TcPersistGeom tcg = tc_persist_geom(s);
    const unsigned char* pws = reinterpret_cast<const unsigned char*>(F(fl.persist));
    const __nv_bfloat16* aib = plan.att_bwd ? reinterpret_cast<const __nv_bfloat16*>(pws + prl.aib) : nullptr;
    const __nv_bfloat16* hgb = plan.att_bwd ? reinterpret_cast<const __nv_bfloat16*>(pws + prl.hgb) : nullptr;
    const int ldab = tcg.Kp_att, ldhb = tcg.Kp_gen;
    const __nv_bfloat16* aib1 = aib ? aib + (size_t)B * ldab : nullptr;      // rows 1..T
    const __nv_bfloat16* hgb1 = hgb ? hgb + (size_t)B * ldhb : nullptr;

    // ---- 1. frame / stop projection backward (time-batched) ----
    gather_frame_grads_kernel<<<grid_for(TB * N1), 256, 0, st>>>(W(l.dfs), dout.d_spectrogram, dout.d_stop, B, T, frames.T, N, s.R);
    B200_LAUNCH_CHECK();
    // d h_gen (direct) and d ctx (projection part)
    B200_TRY(wgemm(st, l, bws, 0, 0, (int)TB, D, N1, W(l.dfs), N1, F(fl.wfs), D + M, W(l.dhgd), D, 0.f));
    B200_TRY(wgemm(st, l, bws, 0, 0, (int)TB, M, N1, W(l.dfs), N1, F(fl.wfs) + D, D + M, W(l.dctxs), M, 0.f));

    void* dgab = plan.att_bwd ? static_cast<void*>(W(l.dgab)) : nullptr;
    if (!free_running) {
        B200_TRY(frame_weight_grads(c, dw, hgb1, ldhb, aib1, ldab));

        // ---- 2. generator LSTM reverse loop ----
        // the persistent reverse loops keep their bf16 gate gradients as [T, B, 4D] histories: the time-batched products below read them
        // in place (K-major for dX, MN-major for dW) instead of converting the fp32 copies
        void* dggb = plan.gen_bwd ? static_cast<void*>(W(l.dggb)) : nullptr;
        if (plan.gen_bwd) {
            // bf16 perf mode: one cooperative weight-stationary TMA + wgmma kernel for the whole reverse recurrence (decoder_persist_bwd_tc.cu)
            B200_TRY(tc_persist_gen_bwd_loop(s, w, in, fl, fws, W(l.dhgd), W(l.dgg), reinterpret_cast<unsigned char*>(W(l.pextra)), st, dggb));
        } else {
            for (int i = T - 1; i >= 0; --i) B200_TRY(gen_bwd_step(c, i, W(l.part), W(l.dc), W(l.dhz)));
        }
        {
            // time-batched generator gradients.  The gate gradients are final now: their packed (transposed / K-contiguous) bf16 copies are
            // made once and shared by the three weight-gradient and the two input-gradient products (pack cache of the wgmma GEMM).
            PackScope pack_scope;
            B200_TRY(gen_weight_grads(c, dw, hgb, ldhb, aib1, ldab, dggb));
            B200_TRY(gen_input_grads(c, 0, T, dggb));
        }

        // ---- 3. attention LSTM + attention reverse loop ----
        if (plan.att_bwd) {
            // bf16 perf mode: cooperative weight-stationary kernel (tensor-core attention backward inside), then a parallel post pass
            B200_TRY(persist_att_bwd_loop(s, w, in, fl, fws, prl, pws, fwd_out.alignments,
                                          dout.d_alignments, W(l.dhas), W(l.dctxs), W(l.dga), W(l.dq), W(l.dctxt), W(l.dmemT),
                                          reinterpret_cast<unsigned char*>(W(l.pextra2)), dw, st, dgab));
        } else {
            B200_TRY(att_chain_init(c));
            for (int i = T - 1; i >= 0; --i) B200_TRY(att_bwd_step(c, i, W(l.part), W(l.dc), W(l.dhz)));
        }
    } else {
        // ---- 2-3. at least one free-running step: segmented reverse sweep on the per-step chains ----
        // A free-running step f >= 1 feeds prenet(frame_{f-1}) and autograd follows it (tacotron2.py:171,181: no detach), so the attention
        // reverse step f has to finish before the generator reverse step f-1 can start.  [0, T) is cut at every such f.  Each segment
        // [f, e), from the end: generator reverse steps e-1 .. f, the generator-input gradients of its rows, attention reverse steps
        // e-1 .. f, then the feedback of step f into row f-1 (dFS, d h_gen, d ctx).  Both recurrences carry state across segments at the
        // same time: the generator's lives in part_gen / dc_gen / dhz_gen, the attention's in part / dc / dhz / dcum.
        B200_TRY(att_chain_init(c));
        int e = T;
        for (int f = T - 1; f >= 0; --f) {
            if (f > 0 && !c.free_running(f)) continue;
            for (int i = e - 1; i >= f; --i) B200_TRY(gen_bwd_step(c, i, W(l.part_gen), W(l.dc_gen), W(l.dhz_gen)));
            B200_TRY(gen_input_grads(c, f, e, nullptr));
            for (int i = e - 1; i >= f; --i) B200_TRY(att_bwd_step(c, i, W(l.part), W(l.dc), W(l.dhz)));
            if (f > 0) B200_TRY(frame_feedback(c, f));       // step 0 was fed the zero frame: nothing to send
            e = f;
        }
        // dFS is final only now: the fed-back rows changed it after the products of section 1
        B200_TRY(frame_weight_grads(c, dw, nullptr, 0, nullptr, 0));
        {
            PackScope pack_scope;
            B200_TRY(gen_weight_grads(c, dw, nullptr, 0, nullptr, 0, nullptr));
        }
    }

    // ---- 4. time-batched gradients of the attention LSTM, attention parameters, prenet, memory ----
    {
        PackScope pack_scope;       // one transposed bf16 copy of the attention-LSTM gate gradients for the three weight-gradient products
        B200_TRY(wgemm16(st, l, bws, 4 * D, P, (int)TB, W(l.dga), 4 * D, F(fl.p1), P, nullptr, 0, dw.att_w_ih, P + M, 1.f, dgab, 4 * D));
        B200_TRY(wgemm16(st, l, bws, 4 * D, M, (int)TB, W(l.dga), 4 * D, ai, MD, aib ? aib + D : nullptr, ldab, dw.att_w_ih + P, P + M, 1.f, dgab, 4 * D));
        B200_TRY(wgemm16(st, l, bws, 4 * D, D, (int)TB, W(l.dga), 4 * D, ai + M, MD, aib, ldab, dw.att_w_hh, D, 1.f, dgab, 4 * D));
    }
    {
        B200_TRY(colsum_add(dw.att_b_ih, dw.att_b_hh, W(l.dga), TB, 4 * D, 4 * D, W(l.gpart), st));
        B200_TRY(colsum_add(dw.attn_bias, nullptr, W(l.dq), TB, A, A, W(l.gpart), st));
    }
    // d Wq = dQ^T . h_att
    B200_TRY(wgemm16(st, l, bws, A, D, (int)TB, W(l.dq), A, ai1 + M, MD, aib1, ldab, dw.attn_query, D, 1.f));
    if (!plan.att_bwd) {
        if (!fwd_att) {
            batchsum_add_kernel<<<grid_for((size_t)A * C), 256, 0, st>>>(dw.attn_location, W(l.dWloc_acc), B, (size_t)A * C);
            B200_LAUNCH_CHECK();
            batchsum_add_kernel<<<grid_for((size_t)C * K), 256, 0, st>>>(dw.attn_loc_features, W(l.dWc_acc), B, (size_t)C * K);
            B200_LAUNCH_CHECK();
        }
        batchsum_add_kernel<<<1, 256, 0, st>>>(dw.attn_energy, W(l.dv_acc), B, (size_t)A);
        B200_LAUNCH_CHECK();
    }
    // d Wm = dmemT^T . memory ; d memory = align^T . dctx (per utterance) + dmemT . Wm
    B200_TRY(wgemm(st, l, bws, 1, 0, A, M, B * L, W(l.dmemT), A, in.memory, M, dw.attn_memory, M, 1.f));
    if (d_memory) {
        B200_TRY(wgemm(st, l, bws, 1, 0, L, M, T, fwd_out.alignments, L, W(l.dctxt), B * M, d_memory, M, 0.f, B,
                       (long long)T * L, (long long)M, (long long)L * M));
        B200_TRY(wgemm(st, l, bws, 0, 0, B * L, M, A, W(l.dmemT), A, w.attn_memory, M, d_memory, M, 1.f));
    }
    // prenet: d P1 = dGA . W_ih[:, :P]; through dropout+relu; layer 1; layer 0.  Row i = step i's prenet, free-running ones included.
    {
        B200_TRY(xgemm16(st, l, bws, (int)TB, P, 4 * D, W(l.dga), 4 * D, dgab, 4 * D, w.att_w_ih, P + M, W(l.dp1), P, 0.f));
        B200_TRY(prenet_relu_bwd(c, W(l.dp1), F(fl.p1), in.mask_prenet1, in.mask_step_prenet1));
        B200_TRY(wgemm(st, l, bws, 1, 0, P, P, (int)TB, W(l.dp1), P, F(fl.p0), P, dw.prenet_w1, P, 1.f));
        B200_TRY(colsum_add(dw.prenet_b1, nullptr, W(l.dp1), TB, P, P, W(l.gpart), st));
        B200_TRY(wgemm(st, l, bws, 0, 0, (int)TB, P, P, W(l.dp1), P, w.prenet_w1, P, W(l.dp0), P, 0.f));
        B200_TRY(prenet_relu_bwd(c, W(l.dp0), F(fl.p0), in.mask_prenet0, in.mask_step_prenet0));
        B200_TRY(wgemm(st, l, bws, 1, 0, P, N, (int)TB, W(l.dp0), P, F(fl.xtm), N, dw.prenet_w0, N, 1.f));
        B200_TRY(colsum_add(dw.prenet_b0, nullptr, W(l.dp0), TB, P, P, W(l.gpart), st));
    }
    return B200TTS_OK;
}

}  // extern "C"
