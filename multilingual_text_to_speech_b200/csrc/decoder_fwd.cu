// Decoder forward: prenet, attention LSTM + location-sensitive attention loop, generator LSTM loop,
// frame / stop projections.  Restates Decoder._decode (reference modules/tacotron2.py:148-209) with the
// teacher-forced dependency structure exploited: everything that does not depend on the recurrence is a
// time-batched GEMM; the two recurrences run as short per-step kernel chains (GEMM -> cell -> attention).
#include "decoder_internal.cuh"

namespace b200tts {

int gemm_tc_try(const GemmDesc& d, cudaStream_t st, bool* handled);      // gemm_tc.cu

// =============================================================================================
// small utility kernels
// =============================================================================================
namespace {

__global__ void copy2d_kernel(float* __restrict__ dst, int ldd, const float* __restrict__ src, int lds, int rows, int cols) {
    const size_t total = (size_t)rows * cols;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int r = idx / cols, c = idx % cols;
        dst[(size_t)r * ldd + c] = src[(size_t)r * lds + c];
    }
}
__global__ void add_vec_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ b, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = a[i] + b[i];
}
__global__ void fill_kernel(float* __restrict__ dst, float v, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = v;
}

// Xtm[i, b, n] = (i == 0) ? 0 : target[b, n, i*R - 1]   (tacotron2.py:126-134 without the prenet; step i is fed the last frame of
// step i-1's group).  T = steps, Tf = frames of target.
__global__ void prep_target_kernel(float* __restrict__ xtm, const float* __restrict__ target, int B, int N, int T, int R, int Tf) {
    // tile transpose over (n, i) for one b: 32 x 32 tiles through shared memory
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int i0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int n = n0 + r, i = i0 + threadIdx.x;       // read along i (contiguous in target)
        float v = 0.f;
        if (n < N && i < T && i > 0) v = target[((size_t)b * N + n) * Tf + (size_t)i * R - 1];
        tile[r][threadIdx.x] = v;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int i = i0 + r, n = n0 + threadIdx.x;       // write along n (contiguous in xtm)
        if (i < T && n < N) xtm[((size_t)i * B + b) * N + n] = tile[threadIdx.x][r];
    }
}

// x = relu(x); x = x * keep * scale   (Prenet._layer_pass, tacotron2.py:37-41; GEMM already added the bias)
__global__ void relu_dropout_kernel(float* __restrict__ x, const uint8_t* __restrict__ keep, float scale, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float v = fmaxf(x[i], 0.f);
        if (keep) v = v * (float)keep[i] * scale;
        x[i] = v;
    }
}

// Frame k = i*R + j of utterance b (step i, slot j) from the step rows FS [S, B, R*(N+1)] = [R frames | R stop logits]:
// spec[b, k, n] = FS[i, b, j*N + n]; stop[b, k] = FS[i, b, R*N + j].  Only the T frames are written: the tail of the last step is dropped.
__global__ void split_frames_kernel(float* __restrict__ spec, float* __restrict__ stop, const float* __restrict__ fs,
                                    int B, int T, int N, int R) {
    const size_t total = (size_t)B * T * (N + 1);
    const int W = R * (N + 1);
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int n = idx % (N + 1);
        const int k = (idx / (N + 1)) % T;
        const int b = idx / ((size_t)(N + 1) * T);
        const int i = k / R, j = k - i * R;
        const float* row = fs + ((size_t)i * B + b) * W;
        if (n < N) spec[((size_t)b * T + k) * N + n] = row[j * N + n];
        else stop[(size_t)b * T + k] = row[R * N + j];
    }
}

// =============================================================================================
// LSTM cell (pointwise part) + regulariser + optional attention-query partial projection
//   gates: xproj (time-batched input projection incl. both biases) + sum of split-K partials of the
//   recurrent GEMM.  modules/layers.py:26-34 (zoneout), :44-47 (dropout), torch LSTMCell order i,f,g,o.
// =============================================================================================

__global__ void __launch_bounds__(256) lstm_cell_fwd_kernel(const CellFwdArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int Bp = (p.B + 7) & ~7;
    float* hsT = sm;                                  // [CELL_UNITS][Bp]
    float* wq = sm + CELL_UNITS * Bp;                 // [A][CELL_UNITS + 1]
    const int u0 = blockIdx.x * CELL_UNITS;
    const int D = p.D;
    const float inv_h = p.rate_h < 1.f ? 1.f / (1.f - p.rate_h) : 0.f;
    const float inv_c = p.rate_c < 1.f ? 1.f / (1.f - p.rate_c) : 0.f;
    for (int idx = threadIdx.x; idx < Bp * CELL_UNITS; idx += blockDim.x) {
        const int b = idx / CELL_UNITS, uu = idx % CELL_UNITS, u = u0 + uu;
        float hs = 0.f;
        if (b < p.B && u < D) {
            const size_t g0 = (size_t)b * 4 * D + u;
            float zi = p.xproj[g0], zf = p.xproj[g0 + D], zg = p.xproj[g0 + 2 * D], zo = p.xproj[g0 + 3 * D];
            for (int s = 0; s < p.nsplit; ++s) {
                const float* q = p.part + s * p.part_stride + g0;
                zi += q[0]; zf += q[D]; zg += q[2 * D]; zo += q[3 * D];
            }
            const float gi = sigmoidf_acc(zi), gf = sigmoidf_acc(zf), gg = tanhf(zg), go = sigmoidf_acc(zo);
            const float cp = p.c_prev[(size_t)b * D + u];
            float cn = gf * cp + gi * gg;
            float hn = go * tanhf(cn);
            p.gates[g0] = gi; p.gates[g0 + D] = gf; p.gates[g0 + 2 * D] = gg; p.gates[g0 + 3 * D] = go;
            if (p.kind == B200TTS_CELL_ZONEOUT) {
                const float hp = p.h_prev[(size_t)b * p.ld_hprev + u];
                if (p.training) {
                    float dh = hn - hp, dc = cn - cp;
                    if (p.mask_h) dh = dh * (float)p.mask_h[(size_t)b * D + u] * inv_h;
                    if (p.mask_c) dc = dc * (float)p.mask_c[(size_t)b * D + u] * inv_c;
                    hn = (1.f - p.rate_h) * dh + hp;
                    cn = (1.f - p.rate_c) * dc + cp;
                } else {
                    hn = p.rate_h * hp + (1.f - p.rate_h) * hn;
                    cn = p.rate_c * cp + (1.f - p.rate_c) * cn;
                }
            } else if (p.training && p.mask_h) {
                hn = hn * (float)p.mask_h[(size_t)b * D + u] * inv_h;
            }
            if (p.lengths) {                     // packed sequence: frozen state and zero output beyond the length
                const bool valid = p.step < p.lengths[b];
                if (p.y_out) p.y_out[(size_t)b * p.ld_y + u] = valid ? hn : 0.f;
                if (!valid) { cn = cp; hn = p.h_prev[(size_t)b * p.ld_hprev + u]; }
            }
            p.c_out[(size_t)b * D + u] = cn;
            p.h_out[(size_t)b * p.ld_hout + u] = hn;
            hs = hn;
        }
        if (p.Wq) hsT[uu * Bp + b] = hs;
    }
    if (!p.Wq) return;
    const int A = p.A;
    for (int idx = threadIdx.x; idx < A * CELL_UNITS; idx += blockDim.x) {
        const int a = idx / CELL_UNITS, uu = idx % CELL_UNITS;
        wq[a * (CELL_UNITS + 1) + uu] = (u0 + uu < D) ? p.Wq[(size_t)a * D + u0 + uu] : 0.f;
    }
    __syncthreads();
    const int nbg = Bp / 8;
    for (int idx = threadIdx.x; idx < A * nbg; idx += blockDim.x) {
        const int a = idx % A, bg = idx / A;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll 8
        for (int uu = 0; uu < CELL_UNITS; ++uu) {
            const float w = wq[a * (CELL_UNITS + 1) + uu];
            const float4 h0 = *reinterpret_cast<const float4*>(&hsT[uu * Bp + bg * 8]);
            const float4 h1 = *reinterpret_cast<const float4*>(&hsT[uu * Bp + bg * 8 + 4]);
            acc[0] = fmaf(w, h0.x, acc[0]); acc[1] = fmaf(w, h0.y, acc[1]); acc[2] = fmaf(w, h0.z, acc[2]); acc[3] = fmaf(w, h0.w, acc[3]);
            acc[4] = fmaf(w, h1.x, acc[4]); acc[5] = fmaf(w, h1.y, acc[5]); acc[6] = fmaf(w, h1.z, acc[6]); acc[7] = fmaf(w, h1.w, acc[7]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int b = bg * 8 + j;
            if (b < p.B) p.qpart[((size_t)blockIdx.x * p.B + b) * A + a] = acc[j];
        }
    }
}

// =============================================================================================
// Location-sensitive attention step (modules/attention.py:39-45, 67-86), one CTA per utterance.
// =============================================================================================
struct AttnFwdArgs {
    const float* qpart; int nq;        // [nq, B, A] partial queries (summed here)
    float* q_save;                     // [B, A] or null
    const float* memT;                 // [B, L, A]
    const float* memory;               // [B, L, M]
    const int* lengths;                // [B]
    const float* Wc;                   // [C, K]   location conv
    const float* Wloc;                 // [A, C]
    const float* bias; const float* v; // [A]
    const float* cum_prev; float* cum_next;   // [B, L]
    float* align; long long align_bstride;    // &align[0, i, 0]; stride between utterances
    float* ctx_out; int ld_ctx;        // [B, ld]
    float* ctx_out2; int ld_ctx2;      // optional second copy
    int B, L, M, A, C, K;
};

static inline size_t attn_fwd_smem_floats(int L, int M, int A, int C, int K) {
    const int Lp = (L + 3) & ~3;
    return (size_t)2 * A + ((L + K - 1 + 3) & ~3) + (size_t)C * A + ((C * K + 3) & ~3) + (size_t)C * Lp + Lp + 64 +
           (size_t)(ATT_THREADS / 32) * M;
}

__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const AttnFwdArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = ATT_THREADS / 32;
    const int L = p.L, A = p.A, C = p.C, K = p.K, M = p.M;
    const int half = (K - 1) / 2, Lp = (L + 3) & ~3;
    float* qb = sm;
    float* vv = qb + A;
    float* cump = vv + A;
    float* WlT = cump + ((L + K - 1 + 3) & ~3);
    float* Wcs = WlT + C * A;
    float* f = Wcs + ((C * K + 3) & ~3);
    float* e = f + C * Lp;
    float* red = e + Lp;
    float* cred = red + 64;
    int len = p.lengths[b];
    len = len < 0 ? 0 : (len > L ? L : len);

    for (int a = tid; a < A; a += ATT_THREADS) {
        float q = 0.f;
        for (int s = 0; s < p.nq; ++s) q += p.qpart[((size_t)s * p.B + b) * A + a];
        if (p.q_save) p.q_save[(size_t)b * A + a] = q;
        qb[a] = q + p.bias[a];
        vv[a] = p.v[a];
    }
    for (int j = tid; j < L + K - 1; j += ATT_THREADS) {
        const int l = j - half;
        cump[j] = (l >= 0 && l < L) ? p.cum_prev[(size_t)b * L + l] : 0.f;
    }
    for (int idx = tid; idx < A * C; idx += ATT_THREADS) {
        const int a = idx / C, c = idx % C;
        WlT[c * A + a] = p.Wloc[idx];
    }
    for (int idx = tid; idx < C * K; idx += ATT_THREADS) Wcs[idx] = p.Wc[idx];
    __syncthreads();

    // location features f[c, l] = sum_k Wc[c, k] * cum[l + k - half]
    for (int idx = tid; idx < C * Lp; idx += ATT_THREADS) {
        const int c = idx / Lp, l = idx % Lp;
        float acc = 0.f;
        if (l < L)
            for (int k = 0; k < K; ++k) acc = fmaf(Wcs[c * K + k], cump[l + k], acc);
        f[idx] = acc;
    }
    __syncthreads();

    // energies: warp = 4 consecutive positions, lane = attention dims {lane, lane+32, lane+64, lane+96}
    for (int l0 = warp * 4; l0 < len; l0 += NW * 4) {
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
        for (int c = 0; c < C; ++c) {
            const float4 fv = *reinterpret_cast<const float4*>(&f[c * Lp + l0]);
            float w[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) w[j] = (lane + 32 * j < A) ? WlT[c * A + lane + 32 * j] : 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s[0][j] = fmaf(fv.x, w[j], s[0][j]); s[1][j] = fmaf(fv.y, w[j], s[1][j]);
                s[2][j] = fmaf(fv.z, w[j], s[2][j]); s[3][j] = fmaf(fv.w, w[j], s[3][j]);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int l = l0 + i;
            if (l < len) {                      // warp-uniform
                float ep = 0.f;
                const float* mt = p.memT + ((size_t)b * L + l) * A;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int a = lane + 32 * j;
                    if (a < A) ep = fmaf(vv[a], tanhf(s[i][j] + qb[a] + mt[a]), ep);
                }
                ep = warp_sum(ep);
                if (lane == 0) e[l] = ep;
            }
        }
    }
    __syncthreads();

    // masked softmax over l < len (energies[~mask] = -inf, attention.py:77-83)
    float mx = -INFINITY;
    for (int l = tid; l < len; l += ATT_THREADS) mx = fmaxf(mx, e[l]);
    mx = block_max(mx, red);
    float sum = 0.f;
    for (int l = tid; l < len; l += ATT_THREADS) {
        const float ex = expf(e[l] - mx);
        e[l] = ex;
        sum += ex;
    }
    sum = block_sum(sum, red);
    for (int l = tid; l < L; l += ATT_THREADS) {
        const float w = l < len ? e[l] / sum : 0.f;
        e[l] = w;
        p.align[(size_t)b * p.align_bstride + l] = w;
        p.cum_next[(size_t)b * L + l] = cump[l + half] + w;
    }
    __syncthreads();

    // context[m] = sum_l w[l] * memory[b, l, m]
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    for (int l = warp; l < len; l += NW) {
        const float w = e[l];
        const float* row = p.memory + ((size_t)b * L + l) * M;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int m = lane + 32 * j;
            if (m < M) acc[j] = fmaf(w, row[m], acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int m = lane + 32 * j;
        if (m < M) cred[warp * M + m] = acc[j];
    }
    __syncthreads();
    for (int m = tid; m < M; m += ATT_THREADS) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) s += cred[w * M + m];
        p.ctx_out[(size_t)b * p.ld_ctx + m] = s;
        if (p.ctx_out2) p.ctx_out2[(size_t)b * p.ld_ctx2 + m] = s;
    }
}

// =============================================================================================
// Forward-attention step (modules/attention.py:23-45, 89-124), one CTA per utterance:
//   s = softmax(v . tanh(q + memT + bias)) over all L;  a = (alpha + alpha shifted by one) * s, zero at l >= length;
//   w = clamp(a, 1e-6) / max(sum, 1e-12);  context = w . memory over all L;  w is the alignment row and the next alpha.
// =============================================================================================
struct FwdAttnArgs {
    const float* qpart; int nq;        // [nq, B, A] partial queries (summed here)
    float* q_save;                     // [B, A] or null
    const float* memT;                 // [B, L, A]
    const float* memory;               // [B, L, M]
    const int* lengths;                // [B]
    const float* bias; const float* v; // [A]
    const float* alpha_prev; float* alpha_next;   // [B, L] (distinct buffers)
    float* align; long long align_bstride;        // &align[0, i, 0]; stride between utterances
    float* ctx_out; int ld_ctx;        // [B, ld]
    int B, L, M, A;
    int own_extent;                    // 1: every sum runs over l < lengths[b] instead of l < L (b200tts_decoder_shape.att_extent)
};

static inline size_t fwd_attn_smem_floats(int L, int M, int A) {
    return (size_t)2 * A + ((L + 3) & ~3) + 64 + (size_t)(ATT_THREADS / 32) * M;
}

__global__ void __launch_bounds__(ATT_THREADS) fwd_attn_fwd_kernel(const FwdAttnArgs p) {
    extern __shared__ __align__(16) float sm[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = ATT_THREADS / 32;
    const int L = p.L, A = p.A, M = p.M;
    float* qb = sm;
    float* vv = qb + A;
    float* s = vv + A;
    float* red = s + ((L + 3) & ~3);
    float* cred = red + 64;
    int len = p.lengths[b];
    len = len < 0 ? 0 : (len > L ? L : len);
    const float* alpha = p.alpha_prev + (size_t)b * L;
    // the extent of the softmax, the floor, the normalisation and the context: the padded L (the reference's training semantics) or
    // the utterance's own length, which gives a padded batch the loop bounds, and so the partial sums, of decoding it alone
    const int Le = p.own_extent ? len : L;

    for (int a = tid; a < A; a += ATT_THREADS) {
        float q = 0.f;
        for (int k = 0; k < p.nq; ++k) q += p.qpart[((size_t)k * p.B + b) * A + a];
        if (p.q_save) p.q_save[(size_t)b * A + a] = q;
        qb[a] = q + p.bias[a];
        vv[a] = p.v[a];
    }
    __syncthreads();
    fwd_att_transition(qb, vv, p.memT + (size_t)b * L * A, Le, A, s, red);

    float csum = 0.f;
    for (int l = tid; l < Le; l += ATT_THREADS) {
        const float c = fmaxf(fwd_att_product(alpha, s, l, len), FWD_ATT_FLOOR);
        s[l] = c;           // each thread rewrites only the positions it read
        csum += c;
    }
    const float denom = fmaxf(block_sum(csum, red), FWD_ATT_NORM_EPS);
    for (int l = tid; l < L; l += ATT_THREADS) {
        const float w = l < Le ? s[l] / denom : 0.f;
        s[l] = w;
        p.align[(size_t)b * p.align_bstride + l] = w;
        p.alpha_next[(size_t)b * L + l] = w;
    }
    __syncthreads();

    // context[m] = sum over every l < Le of w[l] * memory[b, l, m]
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    for (int l = warp; l < Le; l += NW) {
        const float w = s[l];
        const float* row = p.memory + ((size_t)b * L + l) * M;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int m = lane + 32 * j;
            if (m < M) acc[j] = fmaf(w, row[m], acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int m = lane + 32 * j;
        if (m < M) cred[warp * M + m] = acc[j];
    }
    __syncthreads();
    for (int m = tid; m < M; m += ATT_THREADS) {
        float acc_m = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) acc_m += cred[w * M + m];
        p.ctx_out[(size_t)b * p.ld_ctx + m] = acc_m;
    }
}

// alpha_0 = one-hot at position 0 (ForwardAttention.reset, attention.py:103-106): dst[r * ld] = 1 for every row r
__global__ void set_first_column_kernel(float* __restrict__ dst, int ld, int rows) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) dst[(size_t)r * ld] = 1.f;
}

}  // namespace
int launch_cell_fwd(const CellFwdArgs& a, cudaStream_t st) {
    const int Bp = (a.B + 7) & ~7;
    const size_t smem = a.Wq ? ((size_t)CELL_UNITS * Bp + (size_t)a.A * (CELL_UNITS + 1)) * sizeof(float) : 0;
    if (smem > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(lstm_cell_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    lstm_cell_fwd_kernel<<<cdiv(a.D, CELL_UNITS), 256, smem, st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}
namespace {

int launch_attn_fwd(const AttnFwdArgs& a, cudaStream_t st) {
    const size_t smem = attn_fwd_smem_floats(a.L, a.M, a.A, a.C, a.K) * sizeof(float);
    B200_REQUIRE(smem <= 227 * 1024, "attention step: shared memory %zu B exceeds 227 KB (L=%d M=%d)", smem, a.L, a.M);
    static size_t configured = 0;
    if (smem > configured) {
        B200_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    attn_fwd_kernel<<<a.B, ATT_THREADS, smem, st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int launch_fwd_attn(const FwdAttnArgs& a, cudaStream_t st) {
    const size_t smem = fwd_attn_smem_floats(a.L, a.M, a.A) * sizeof(float);
    B200_REQUIRE(smem <= 227 * 1024, "forward attention step: shared memory %zu B exceeds 227 KB (L=%d M=%d)", smem, a.L, a.M);
    static size_t configured = 48 * 1024;
    if (smem > configured) {
        B200_CUDA(cudaFuncSetAttribute(fwd_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    fwd_attn_fwd_kernel<<<a.B, ATT_THREADS, smem, st>>>(a);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

inline int grid_for(size_t n) {
    size_t g = (n + 255) / 256;
    return (int)(g > NUM_SMS * 16 ? NUM_SMS * 16 : (g < 1 ? 1 : g));
}

}  // namespace

int launch_copy2d(float* dst, int ldd, const float* src, int lds, int rows, int cols, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return B200TTS_OK;
    copy2d_kernel<<<grid_for((size_t)rows * cols), 256, 0, st>>>(dst, ldd, src, lds, rows, cols);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}
int launch_add_vec(float* dst, const float* a, const float* b, int n, cudaStream_t st) {
    add_vec_kernel<<<cdiv(n, 256), 256, 0, st>>>(dst, a, b, n);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}
int launch_fill(float* dst, float value, size_t n, cudaStream_t st) {
    if (n == 0) return B200TTS_OK;
    fill_kernel<<<grid_for(n), 256, 0, st>>>(dst, value, n);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int validate_decoder_shape(const b200tts_decoder_shape& s) {
    B200_REQUIRE(s.B > 0 && s.L > 0 && s.T > 0, "decoder: empty batch/sequence (B=%d L=%d T=%d)", s.B, s.L, s.T);
    B200_REQUIRE(s.R >= 0, "decoder: frames per step R=%d must be >= 1 (0 means 1)", s.R);
    B200_REQUIRE(s.att_kind == B200TTS_ATT_LOCATION || s.att_kind == B200TTS_ATT_FORWARD, "decoder: bad attention kind %d", s.att_kind);
    B200_REQUIRE(s.att_extent == 0 || s.att_extent == 1, "decoder: bad attention extent %d", s.att_extent);
    B200_REQUIRE(s.M > 0 && s.D > 0 && s.P > 0 && s.A > 0 && s.N > 0, "decoder: non-positive dimension");
    B200_REQUIRE(s.A <= 128 && s.A % 4 == 0, "decoder: attention dimension %d unsupported (need <= 128, multiple of 4)", s.A);
    if (!forward_attention(s)) {        // forward attention has no location features: C and K are ignored
        B200_REQUIRE(s.C > 0 && s.K > 0, "decoder: non-positive location dimension");
        B200_REQUIRE(s.K % 2 == 1, "decoder: attention kernel size must be odd (got %d)", s.K);
        B200_REQUIRE(s.C <= 32 && s.C % 4 == 0, "decoder: location channels %d unsupported (need <= 32, multiple of 4)", s.C);
    }
    B200_REQUIRE(s.M <= 512, "decoder: memory dimension %d > 512 unsupported", s.M);
    B200_REQUIRE(s.cell_kind == B200TTS_CELL_DROPOUT || s.cell_kind == B200TTS_CELL_ZONEOUT, "decoder: bad cell kind %d", s.cell_kind);
    B200_REQUIRE(s.rate_h >= 0.f && s.rate_h < 1.f && s.rate_c >= 0.f && s.rate_c < 1.f && s.prenet_rate >= 0.f && s.prenet_rate < 1.f,
                 "decoder: dropout / zoneout rates must be in [0, 1)");
    return B200TTS_OK;
}

// =============================================================================================
// host orchestration
// =============================================================================================
namespace {

struct FwdCtx {
    const b200tts_decoder_shape& s;
    const b200tts_decoder_params& w;
    const b200tts_decoder_inputs& in;
    DecoderLayout lay;
    float* ws;
    cudaStream_t st;
    float* at(size_t off) const { return ws + off; }
};

int run_gemm(cudaStream_t st, int M, int N, int K, const float* A, int lda, const float* B, int ldb, bool transB,
             float* C, int ldc, const float* bias, float beta, int splitk = 1, float* partial = nullptr, bool keep = false) {
    GemmDesc d;
    d.A = A; d.B = B; d.C = C; d.bias = bias; d.M = M; d.N = N; d.K = K; d.lda = lda; d.ldb = ldb; d.ldc = ldc;
    d.transA = 0; d.transB = transB ? 1 : 0; d.beta = beta; d.splitk = splitk; d.partial = partial; d.keep_partials = keep;
    if (keep && splitk == 1) {          // single split: the "partial" buffer simply receives the product
        d.C = partial; d.ldc = N; d.keep_partials = 0; d.partial = nullptr;
    }
    return gemm_run(d, st);
}

// prenet of one block of rows (time-batched or a single free-running step)
int prenet_rows(const FwdCtx& c, int rows, const float* x, float* p0, float* p1, const uint8_t* m0, const uint8_t* m1) {
    const auto& s = c.s;
    const float scale = 1.f / (1.f - s.prenet_rate);
    B200_TRY(run_gemm(c.st, rows, s.P, s.N, x, s.N, c.w.prenet_w0, s.N, true, p0, s.P, c.w.prenet_b0, 0.f));
    relu_dropout_kernel<<<grid_for((size_t)rows * s.P), 256, 0, c.st>>>(p0, m0, scale, (size_t)rows * s.P);
    B200_LAUNCH_CHECK();
    B200_TRY(run_gemm(c.st, rows, s.P, s.P, p0, s.P, c.w.prenet_w1, s.P, true, p1, s.P, c.w.prenet_b1, 0.f));
    relu_dropout_kernel<<<grid_for((size_t)rows * s.P), 256, 0, c.st>>>(p1, m1, scale, (size_t)rows * s.P);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int att_step(const FwdCtx& c, int i, float* align_out) {
    const auto& s = c.s; const auto& l = c.lay;
    const size_t BD = (size_t)s.B * s.D, B4D = 4 * BD, MD = s.M + s.D;
    float* ai_i = c.at(l.ai) + (size_t)i * s.B * MD;
    float* ai_n = ai_i + (size_t)s.B * MD;
    B200_TRY(run_gemm(c.st, s.B, 4 * s.D, (int)MD, ai_i, (int)MD, c.at(l.wcat_att), (int)MD, true, nullptr, 0, nullptr, 0.f,
                      l.split_att, c.at(l.part), true));
    CellFwdArgs ca{};
    ca.xproj = c.at(l.ga) + (size_t)i * B4D; ca.gates = c.at(l.ga) + (size_t)i * B4D;
    ca.part = c.at(l.part); ca.nsplit = l.split_att; ca.part_stride = B4D;
    ca.c_prev = c.at(l.ca) + (size_t)i * BD;
    ca.h_prev = ai_i + s.M; ca.ld_hprev = (int)MD;
    ca.c_out = c.at(l.ca) + (size_t)(i + 1) * BD;
    ca.h_out = ai_n + s.M; ca.ld_hout = (int)MD;
    ca.mask_h = c.in.mask_att_h ? c.in.mask_att_h + (size_t)i * BD : nullptr;
    ca.mask_c = c.in.mask_att_c ? c.in.mask_att_c + (size_t)i * BD : nullptr;
    ca.kind = s.cell_kind; ca.training = s.training; ca.rate_h = s.rate_h; ca.rate_c = s.rate_c;
    ca.Wq = c.w.attn_query; ca.A = s.A; ca.qpart = c.at(l.qpart);
    ca.B = s.B; ca.D = s.D;
    B200_TRY(launch_cell_fwd(ca, c.st));
    if (forward_attention(s)) {
        FwdAttnArgs fa{};
        fa.qpart = c.at(l.qpart); fa.nq = l.ncell_blocks;
        fa.q_save = c.at(l.q) + (size_t)i * s.B * s.A;
        fa.memT = c.at(l.memT); fa.memory = c.in.memory; fa.lengths = c.in.text_lengths;
        fa.bias = c.w.attn_bias; fa.v = c.w.attn_energy;
        fa.alpha_prev = c.at(l.cum) + (size_t)i * s.B * s.L; fa.alpha_next = c.at(l.cum) + (size_t)(i + 1) * s.B * s.L;
        fa.align = align_out + (size_t)i * s.L; fa.align_bstride = (long long)s.T * s.L;
        fa.ctx_out = ai_n; fa.ld_ctx = (int)MD;
        fa.B = s.B; fa.L = s.L; fa.M = s.M; fa.A = s.A; fa.own_extent = s.att_extent;
        return launch_fwd_attn(fa, c.st);
    }
    AttnFwdArgs aa{};
    aa.qpart = c.at(l.qpart); aa.nq = l.ncell_blocks;
    aa.q_save = c.at(l.q) + (size_t)i * s.B * s.A;
    aa.memT = c.at(l.memT); aa.memory = c.in.memory; aa.lengths = c.in.text_lengths;
    aa.Wc = c.w.attn_loc_features; aa.Wloc = c.w.attn_location; aa.bias = c.w.attn_bias; aa.v = c.w.attn_energy;
    aa.cum_prev = c.at(l.cum) + (size_t)i * s.B * s.L; aa.cum_next = c.at(l.cum) + (size_t)(i + 1) * s.B * s.L;
    aa.align = align_out + (size_t)i * s.L; aa.align_bstride = (long long)s.T * s.L;
    aa.ctx_out = ai_n; aa.ld_ctx = (int)MD; aa.ctx_out2 = nullptr; aa.ld_ctx2 = 0;
    aa.B = s.B; aa.L = s.L; aa.M = s.M; aa.A = s.A; aa.C = s.C; aa.K = s.K;
    B200_TRY(launch_attn_fwd(aa, c.st));
    return B200TTS_OK;
}

int gen_step(const FwdCtx& c, int i) {
    const auto& s = c.s; const auto& l = c.lay;
    const size_t BD = (size_t)s.B * s.D, B4D = 4 * BD;
    B200_TRY(run_gemm(c.st, s.B, 4 * s.D, s.D, c.at(l.hg) + (size_t)i * BD, s.D, c.w.gen_w_hh, s.D, true, nullptr, 0, nullptr, 0.f,
                      l.split_gen, c.at(l.part), true));
    CellFwdArgs ca{};
    ca.xproj = c.at(l.gg) + (size_t)i * B4D; ca.gates = c.at(l.gg) + (size_t)i * B4D;
    ca.part = c.at(l.part); ca.nsplit = l.split_gen; ca.part_stride = B4D;
    ca.c_prev = c.at(l.cg) + (size_t)i * BD;
    ca.h_prev = c.at(l.hg) + (size_t)i * BD; ca.ld_hprev = s.D;
    ca.c_out = c.at(l.cg) + (size_t)(i + 1) * BD;
    ca.h_out = c.at(l.hg) + (size_t)(i + 1) * BD; ca.ld_hout = s.D;
    ca.mask_h = c.in.mask_gen_h ? c.in.mask_gen_h + (size_t)i * BD : nullptr;
    ca.mask_c = c.in.mask_gen_c ? c.in.mask_gen_c + (size_t)i * BD : nullptr;
    ca.kind = s.cell_kind; ca.training = s.training; ca.rate_h = s.rate_h; ca.rate_c = s.rate_c;
    ca.Wq = nullptr; ca.A = 0; ca.qpart = nullptr; ca.B = s.B; ca.D = s.D;
    return launch_cell_fwd(ca, c.st);
}

// generator-LSTM input projection and frame/stop projection for `rows` consecutive (step, utterance) rows
int gen_input_proj(const FwdCtx& c, int step0, int nsteps) {
    const auto& s = c.s; const auto& l = c.lay;
    const int MD = s.M + s.D, rows = nsteps * s.B;
    const float* ai = c.at(l.ai) + (size_t)(step0 + 1) * s.B * MD;
    float* gg = c.at(l.gg) + (size_t)step0 * s.B * 4 * s.D;
    B200_TRY(run_gemm(c.st, rows, 4 * s.D, s.D, ai + s.M, MD, c.w.gen_w_ih, s.D + s.M, true, gg, 4 * s.D, c.at(l.bsum_gen), 0.f));
    B200_TRY(run_gemm(c.st, rows, 4 * s.D, s.M, ai, MD, c.w.gen_w_ih + s.D, s.D + s.M, true, gg, 4 * s.D, nullptr, 1.f));
    return B200TTS_OK;
}
int frame_proj(const FwdCtx& c, int step0, int nsteps) {
    const auto& s = c.s; const auto& l = c.lay;
    const int MD = s.M + s.D, rows = nsteps * s.B, N1 = fs_width(s);
    const float* hg = c.at(l.hg) + (size_t)(step0 + 1) * s.B * s.D;
    const float* ai = c.at(l.ai) + (size_t)(step0 + 1) * s.B * MD;
    float* fs = c.at(l.fs) + (size_t)step0 * s.B * N1;
    B200_TRY(run_gemm(c.st, rows, N1, s.D, hg, s.D, c.at(l.wfs), s.D + s.M, true, fs, N1, c.at(l.bfs), 0.f));
    B200_TRY(run_gemm(c.st, rows, N1, s.M, ai, MD, c.at(l.wfs) + s.D, s.D + s.M, true, fs, N1, nullptr, 1.f));
    return B200TTS_OK;
}

}  // namespace

int decoder_forward_impl(const b200tts_decoder_shape& frames, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                         const b200tts_decoder_outputs& out, float* ws, size_t ws_bytes, cudaStream_t st,
                         const b200tts_decoder_state* state, int first) {
    B200_TRY(validate_decoder_shape(frames));
    const b200tts_decoder_shape s = step_shape(frames);     // T = decoder steps from here on; Tf = target frames
    const bool resume = state != nullptr && !first;       // chunked decode: start from the carried state
    FwdCtx c{s, w, in, decoder_layout(s), ws, st};
    const auto& l = c.lay;
    B200_REQUIRE(ws != nullptr && ws_bytes >= l.total * sizeof(float), "decoder_forward: workspace too small (%zu < %zu bytes)",
                 ws_bytes, l.total * sizeof(float));
    B200_REQUIRE(in.memory && in.text_lengths && in.target, "decoder_forward: memory / text_lengths / target must be given");
    B200_REQUIRE(out.spectrogram && out.stop && out.alignments, "decoder_forward: null output");
    if (forward_attention(s))
        B200_REQUIRE(!w.attn_location && !w.attn_loc_features, "decoder_forward: forward attention has no location weights (pass NULL)");
    else
        B200_REQUIRE(w.attn_location && w.attn_loc_features, "decoder_forward: location-sensitive attention needs its location weights");
    const int B = s.B, T = s.T, D = s.D, M = s.M, P = s.P, N = s.N, MD = M + D;
    const int R = s.R, Tf = frames.T, RN = R * N, W = fs_width(s);
    const size_t BD = (size_t)B * D;
    bool sequential = false;
    if (in.teacher)
        for (int i = 0; i < T; ++i) sequential |= (in.teacher[i] == 0);

    // ---- derived parameters ----
    B200_TRY(launch_copy2d(c.at(l.wcat_att), MD, w.att_w_ih + P, P + M, 4 * D, M, st));
    B200_TRY(launch_copy2d(c.at(l.wcat_att) + M, MD, w.att_w_hh, D, 4 * D, D, st));
    B200_TRY(launch_add_vec(c.at(l.bsum_att), w.att_b_ih, w.att_b_hh, 4 * D, st));
    B200_TRY(launch_add_vec(c.at(l.bsum_gen), w.gen_b_ih, w.gen_b_hh, 4 * D, st));
    B200_TRY(launch_copy2d(c.at(l.wfs), D + M, w.frame_w, D + M, RN, D + M, st));
    B200_TRY(launch_copy2d(c.at(l.wfs) + (size_t)RN * (D + M), D + M, w.stop_w, D + M, R, D + M, st));
    B200_TRY(launch_copy2d(c.at(l.bfs), RN, w.frame_b, RN, 1, RN, st));
    B200_TRY(launch_copy2d(c.at(l.bfs) + RN, R, w.stop_b, R, 1, R, st));

    // ---- time-batched prologue: prenet over all frames, attention-LSTM input projection, memory projection ----
    {
        dim3 grid(cdiv(T, 32), cdiv(N, 32), B), block(32, 8);
        prep_target_kernel<<<grid, block, 0, st>>>(c.at(l.xtm), in.target, B, N, T, R, Tf);
        B200_LAUNCH_CHECK();
    }
    B200_TRY(prenet_rows(c, T * B, c.at(l.xtm), c.at(l.p0), c.at(l.p1), in.mask_prenet0, in.mask_prenet1));
    B200_TRY(run_gemm(st, T * B, 4 * D, P, c.at(l.p1), P, w.att_w_ih, P + M, true, c.at(l.ga), 4 * D, c.at(l.bsum_att), 0.f));
    B200_TRY(run_gemm(st, B * s.L, s.A, M, in.memory, M, w.attn_memory, M, true, c.at(l.memT), s.A, nullptr, 0.f));
    if (resume) {
        B200_TRY(launch_copy2d(c.at(l.ai), MD, state->context, M, B, M, st));
        B200_TRY(launch_copy2d(c.at(l.ai) + M, MD, state->att_h, D, B, D, st));
        B200_TRY(launch_copy2d(c.at(l.ca), D, state->att_c, D, B, D, st));
        B200_TRY(launch_copy2d(c.at(l.hg), D, state->gen_h, D, B, D, st));
        B200_TRY(launch_copy2d(c.at(l.cg), D, state->gen_c, D, B, D, st));
        B200_TRY(launch_copy2d(c.at(l.cum), s.L, state->cum_weights, s.L, B, s.L, st));
    } else {
    B200_TRY(launch_fill(c.at(l.ai), 0.f, (size_t)B * MD, st));
    B200_TRY(launch_fill(c.at(l.ca), 0.f, BD, st));
    B200_TRY(launch_fill(c.at(l.hg), 0.f, BD, st));
    B200_TRY(launch_fill(c.at(l.cg), 0.f, BD, st));
    B200_TRY(launch_fill(c.at(l.cum), 0.f, (size_t)B * s.L, st));
    if (forward_attention(s)) {
        set_first_column_kernel<<<cdiv(B, 128), 128, 0, st>>>(c.at(l.cum), s.L, B);
        B200_LAUNCH_CHECK();
    }
    }

    const bool persistent = !sequential && state == nullptr && precision_mode() == B200TTS_PRECISION_BF16 && persist_plan(s).fwd;
    if (persistent) {
        // bf16 perf mode: one cooperative, weight-stationary TMA + wgmma kernel per recurrence (decoder_persist_tc.cu)
        unsigned char* pws = reinterpret_cast<unsigned char*>(c.at(l.persist));
        const TcPersistGeom g = tc_persist_geom(s);
        const PersistLayout pl = persist_layout(s);
        B200_TRY(persist_att_prep(s, w, in, l, ws, pws, st));
        B200_TRY(tc_persist_att_loop(s, w, in, l, ws, pws, out.alignments, st));
        {
            // the attention loop left [h_att | ctx] of every step as bf16 operand rows in exactly the column order of W_ih of the
            // generator LSTM: ONE product, its A operand read by TMA straight from those rows (no packing, no second accumulate pass)
            GemmDesc d;
            d.A = c.at(l.ai); d.lda = MD;           // (unused by the wgmma path)
            d.A16 = pws + pl.aib + (size_t)B * g.Kp_att * 2; d.lda16 = g.Kp_att;      // operand row 1 (bf16)
            d.B = w.gen_w_ih; d.ldb = D + M; d.transB = 1; d.C = c.at(l.gg); d.ldc = 4 * D; d.bias = c.at(l.bsum_gen);
            d.M = T * B; d.N = 4 * D; d.K = MD; d.beta = 0.f;
            bool handled = false;
            B200_TRY(gemm_tc_try(d, st, &handled));
            if (!handled) B200_TRY(gen_input_proj(c, 0, T));
        }
        B200_TRY(tc_persist_gen_loop(s, w, in, l, ws, pws, st));
        {       // frame / stop projection straight from the bf16 operand rows of the two loops (h_gen, then ctx accumulated on top)
            const int N1 = W;
            GemmDesc d;
            d.A = c.at(l.hg) + BD; d.lda = D;
            d.A16 = pws + pl.hgb + (size_t)B * g.Kp_gen * 2; d.lda16 = g.Kp_gen;
            d.B = c.at(l.wfs); d.ldb = D + M; d.transB = 1; d.C = c.at(l.fs); d.ldc = N1; d.bias = c.at(l.bfs);
            d.M = T * B; d.N = N1; d.K = D; d.beta = 0.f;
            bool h1 = false, h2 = false;
            B200_TRY(gemm_tc_try(d, st, &h1));
            if (h1) {
                GemmDesc e;
                e.A = c.at(l.ai) + (size_t)B * MD; e.lda = MD;
                e.A16 = pws + pl.aib + ((size_t)B * g.Kp_att + D) * 2; e.lda16 = g.Kp_att;
                e.B = c.at(l.wfs) + D; e.ldb = D + M; e.transB = 1; e.C = c.at(l.fs); e.ldc = N1;
                e.M = T * B; e.N = N1; e.K = M; e.beta = 1.f;
                B200_TRY(gemm_tc_try(e, st, &h2));
                if (!h2) {      // second half on the generic path
                    B200_TRY(run_gemm(c.st, T * B, N1, M, c.at(l.ai) + (size_t)B * MD, MD, c.at(l.wfs) + D, D + M, true, c.at(l.fs), N1, nullptr, 1.f));
                }
            } else {
                B200_TRY(frame_proj(c, 0, T));
            }
        }
    } else if (!sequential) {
        for (int i = 0; i < T; ++i) B200_TRY(att_step(c, i, out.alignments));
        B200_TRY(gen_input_proj(c, 0, T));
        for (int i = 0; i < T; ++i) B200_TRY(gen_step(c, i));
        B200_TRY(frame_proj(c, 0, T));
    } else {
        // at least one free-running step: the previous frame feeds the prenet, so everything is sequential
        for (int i = 0; i < T; ++i) {
            if (!in.teacher[i]) {
                float* x = c.at(l.xtm) + (size_t)i * B * N;
                if (i == 0 && resume) B200_TRY(launch_copy2d(x, N, state->frame, N, B, N, st));
                else if (i == 0) B200_TRY(launch_fill(x, 0.f, (size_t)B * N, st));
                else B200_TRY(launch_copy2d(x, N, c.at(l.fs) + (size_t)(i - 1) * B * W + RN - N, W, B, N, st));
                const uint8_t* m0 = in.mask_step_prenet0 ? in.mask_step_prenet0 + (size_t)i * B * P : nullptr;
                const uint8_t* m1 = in.mask_step_prenet1 ? in.mask_step_prenet1 + (size_t)i * B * P : nullptr;
                B200_TRY(prenet_rows(c, B, x, c.at(l.p0) + (size_t)i * B * P, c.at(l.p1) + (size_t)i * B * P, m0, m1));
                B200_TRY(run_gemm(st, B, 4 * D, P, c.at(l.p1) + (size_t)i * B * P, P, w.att_w_ih, P + M, true,
                                  c.at(l.ga) + (size_t)i * 4 * BD, 4 * D, c.at(l.bsum_att), 0.f));
            }
            B200_TRY(att_step(c, i, out.alignments));
            B200_TRY(gen_input_proj(c, i, 1));
            B200_TRY(gen_step(c, i));
            B200_TRY(frame_proj(c, i, 1));
        }
    }
    split_frames_kernel<<<grid_for((size_t)B * Tf * (N + 1)), 256, 0, st>>>(out.spectrogram, out.stop, c.at(l.fs), B, Tf, N, R);
    B200_LAUNCH_CHECK();
    if (state) {        // state after the last step of the chunk
        const float* ai_T = c.at(l.ai) + (size_t)T * B * MD;
        B200_TRY(launch_copy2d(state->context, M, ai_T, MD, B, M, st));
        B200_TRY(launch_copy2d(state->att_h, D, ai_T + M, MD, B, D, st));
        B200_TRY(launch_copy2d(state->att_c, D, c.at(l.ca) + (size_t)T * BD, D, B, D, st));
        B200_TRY(launch_copy2d(state->gen_h, D, c.at(l.hg) + (size_t)T * BD, D, B, D, st));
        B200_TRY(launch_copy2d(state->gen_c, D, c.at(l.cg) + (size_t)T * BD, D, B, D, st));
        B200_TRY(launch_copy2d(state->cum_weights, s.L, c.at(l.cum) + (size_t)T * B * s.L, s.L, B, s.L, st));
        B200_TRY(launch_copy2d(state->frame, N, c.at(l.fs) + (size_t)(T - 1) * B * W + RN - N, W, B, N, st));
    }
    return B200TTS_OK;
}

// ---- standalone attention step (module-level parity of LocationSensitiveAttention.forward) ----
int attention_step_impl(int B, int L, int M, int D, int A, int C, int K, const float* query, const float* memory,
                        const float* memT, const int* lengths, const float* Wq, const float* Wloc, const float* Wc,
                        const float* bias, const float* v, float* cum, float* ctx, float* weights, float* workspace,
                        cudaStream_t st) {
    B200_REQUIRE(A <= 128 && M <= 512 && (K % 2) == 1, "attention_step: unsupported dims A=%d M=%d K=%d", A, M, K);
    // q = query . Wq^T into workspace[0 : B*A]; new cum into workspace[B*A : B*A + B*L] then copied back
    float* q = workspace;
    float* cum_next = workspace + (size_t)B * A;
    B200_TRY(run_gemm(st, B, A, D, query, D, Wq, D, true, q, A, nullptr, 0.f));
    AttnFwdArgs aa{};
    aa.qpart = q; aa.nq = 1; aa.q_save = nullptr; aa.memT = memT; aa.memory = memory; aa.lengths = lengths;
    aa.Wc = Wc; aa.Wloc = Wloc; aa.bias = bias; aa.v = v; aa.cum_prev = cum; aa.cum_next = cum_next;
    aa.align = weights; aa.align_bstride = L; aa.ctx_out = ctx; aa.ld_ctx = M; aa.ctx_out2 = nullptr; aa.ld_ctx2 = 0;
    aa.B = B; aa.L = L; aa.M = M; aa.A = A; aa.C = C; aa.K = K;
    B200_TRY(launch_attn_fwd(aa, st));
    B200_TRY(launch_copy2d(cum, L, cum_next, L, B, L, st));
    return B200TTS_OK;
}

// ---- standalone forward-attention step (module-level parity of ForwardAttention.forward) ----
int forward_attention_step_impl(int B, int L, int M, int D, int A, const float* query, const float* memory, const float* memT,
                                const int* lengths, const float* Wq, const float* bias, const float* v, float* alpha, float* ctx,
                                float* weights, float* workspace, cudaStream_t st) {
    B200_REQUIRE(B > 0 && L > 0 && D > 0 && A > 0 && A <= 128 && M > 0 && M <= 512,
                 "forward_attention_step: unsupported dims B=%d L=%d D=%d A=%d M=%d", B, L, D, A, M);
    // q = query . Wq^T into workspace[0 : B*A]; the new alpha into workspace[B*A : B*A + B*L], then copied back
    float* q = workspace;
    float* alpha_next = workspace + (size_t)B * A;
    B200_TRY(run_gemm(st, B, A, D, query, D, Wq, D, true, q, A, nullptr, 0.f));
    FwdAttnArgs fa{};
    fa.qpart = q; fa.nq = 1; fa.q_save = nullptr; fa.memT = memT; fa.memory = memory; fa.lengths = lengths;
    fa.bias = bias; fa.v = v; fa.alpha_prev = alpha; fa.alpha_next = alpha_next;
    fa.align = weights; fa.align_bstride = L; fa.ctx_out = ctx; fa.ld_ctx = M;
    fa.B = B; fa.L = L; fa.M = M; fa.A = A;
    B200_TRY(launch_fwd_attn(fa, st));
    B200_TRY(launch_copy2d(alpha, L, alpha_next, L, B, L, st));
    return B200TTS_OK;
}

}  // namespace b200tts
