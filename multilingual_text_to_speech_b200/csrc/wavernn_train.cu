// WaveRNN training (fatchord architecture): the kernels of the teacher-forced forward, the loss and the backward that the library's
// existing ops (GEMM, convolution block) do not cover.
//
//   * gru_seq_fwd_kernel / gru_seq_bwd_kernel: the persistent GRU sequence loop (torch.nn.GRU, gate order r, z, n, h0 = 0), forward and
//     reverse, one cooperative launch of 128 CTAs each.  The input products gi = W_ih x + b_ih of all steps are a time-batched GEMM before
//     the forward loop; the weight, bias and input gradients are time-batched GEMMs / reductions over the dgi / dgh histories after the
//     reverse loop.  Both loops run in fp32 (weights, state, arithmetic) in both precision modes.
//   * wavernn_upsample_bwd_*: the adjoint of one upsampling layer pair (nearest stretch x s, FIR of 2s+1 taps): d in, and d fir += as a
//     fixed-order two-pass reduction.
//   * wavernn_stretch_bwd_kernel: the adjoint of the aux stretch (sum over each frame's hop positions).
//   * wavernn_loss_{raw,mol}_kernel + wavernn_loss_sum_kernel: per-row loss and d logits / N, then one fixed-order sum (no atomics).
//   * column_sum_*: fixed-order column sums (the GRUs' bias gradients over the dgi / dgh histories).
//
// The loops.  CTA c owns hidden units [c U, (c + 1) U), U = R / 128.  Forward: its 3U rows of W_hh (r, z, n of its units) stay in shared
// memory; per step it stages h_{t-1} of a group of utterances from the h history (L2) into shared memory, each warp forms the 3U dot
// products of one utterance (lanes split K, fixed-order warp sums), then one thread per (utterance, unit) runs the cell and writes h_t, r,
// z, n and W_hn h + b_hn.  Reverse: its U columns of W_hh stay in shared memory; per step it stages dgh_{t+1} and forms W_hh^T dgh_{t+1} for
// its units the same way, then one thread per (utterance, unit) adds the external dh_t and the carried z dh, and writes dgi_t, dgh_t and the
// new carry.  One grid barrier per step.  Every reduction has a fixed order, so identical calls give identical bits.
#include <math.h>
#include <type_traits>
#include "decoder_internal.cuh"
#include "tc_ptx.cuh"

namespace b200tts {

namespace {

using namespace tcx;

constexpr int GS_CTAS = 128;
constexpr int GS_THREADS = 256;
constexpr int GS_WARPS = GS_THREADS / 32;
constexpr int GS_MAX_B = 64;
constexpr int GS_MAX_T = 4400;
constexpr int GS_MAX_U = 5;            // R <= 640

struct GruSeqArgs {
    int B, T, G;                        // G: utterances staged per group
    const float* gi;                    // [B, T, 3R]
    const float* w_hh;                  // [3R, R]
    const float* b_hh;                  // [3R]
    float* h;                           // [B, T, R] (forward out; reverse in)
    float* saved;                       // [B, T, 4R]: r, z, n, W_hn h + b_hn (forward out; reverse in)
    const float* dh_ext;                // [B, T, R]
    float* dgi;                         // [B, T, 3R]
    float* dgh;                         // [B, T, 3R]
    float* dh_dbg;                      // [B, T, R] or null: the total dh of every step
    float* carry;                       // [B, R]: z dh of the later step, read and written by the unit's owner only
    unsigned* bar;
    int* abort_flag;
};

template <int U>
__global__ void __launch_bounds__(GS_THREADS, 1) gru_seq_fwd_kernel(GruSeqArgs a) {
    constexpr int R = 128 * U, Q = 3 * U, KL = R / 32;
    extern __shared__ __align__(16) float smem[];
    float* s_w = smem;                          // [3U][R]
    float* s_x = s_w + Q * R;                   // [G][R]
    float* s_acc = s_x + (size_t)a.G * R;       // [G][3U]
    __shared__ int s_ok;
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int B = a.B, T = a.T;
    for (int i = threadIdx.x; i < Q * R; i += GS_THREADS) {
        const int q = i / R, k = i - q * R, g = q / U, j = q - g * U;
        s_w[i] = a.w_hh[(size_t)(g * R + c * U + j) * R + k];
    }
    __syncthreads();
    unsigned target = 0;
    for (int t = 0; t < T; ++t) {
        for (int g0 = 0; g0 < B; g0 += a.G) {
            const int nb = min(a.G, B - g0);
            if (t > 0) {
                for (int i = threadIdx.x; i < nb * (R / 4); i += GS_THREADS) {
                    const int bb = i / (R / 4), k4 = i - bb * (R / 4);
                    reinterpret_cast<float4*>(s_x)[i] =
                        __ldcg(reinterpret_cast<const float4*>(a.h + ((size_t)(g0 + bb) * T + t - 1) * R) + k4);
                }
                __syncthreads();
                for (int bb = warp; bb < nb; bb += GS_WARPS) {
                    float acc[Q];
#pragma unroll
                    for (int q = 0; q < Q; ++q) acc[q] = 0.f;
                    const float* x = s_x + (size_t)bb * R;
#pragma unroll
                    for (int i = 0; i < KL; ++i) {
                        const float v = x[lane + 32 * i];
#pragma unroll
                        for (int q = 0; q < Q; ++q) acc[q] = fmaf(s_w[q * R + lane + 32 * i], v, acc[q]);
                    }
#pragma unroll
                    for (int q = 0; q < Q; ++q) acc[q] = warp_sum(acc[q]);
                    if (lane == 0) {
#pragma unroll
                        for (int q = 0; q < Q; ++q) s_acc[bb * Q + q] = acc[q];
                    }
                }
                __syncthreads();
            }
            for (int e = threadIdx.x; e < nb * U; e += GS_THREADS) {
                const int bb = e / U, j = e - bb * U, u = c * U + j;
                const size_t row = (size_t)(g0 + bb) * T + t;
                const float* gi = a.gi + row * 3 * R;
                float ghr = a.b_hh[u], ghz = a.b_hh[R + u], ghn = a.b_hh[2 * R + u], hp = 0.f;
                if (t > 0) {
                    ghr += s_acc[bb * Q + j];
                    ghz += s_acc[bb * Q + U + j];
                    ghn += s_acc[bb * Q + 2 * U + j];
                    hp = __ldcg(a.h + (row - 1) * R + u);
                }
                const float r = sigmoidf_acc(gi[u] + ghr), z = sigmoidf_acc(gi[R + u] + ghz);
                const float n = tanhf(fmaf(r, ghn, gi[2 * R + u]));
                a.h[row * R + u] = fmaf(z, hp - n, n);       // (1 - z) n + z h
                float* sv = a.saved + row * 4 * R;
                sv[u] = r;
                sv[R + u] = z;
                sv[2 * R + u] = n;
                sv[3 * R + u] = ghn;
            }
            __syncthreads();
        }
        if (t + 1 < T && !grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
    }
}

template <int U>
__global__ void __launch_bounds__(GS_THREADS, 1) gru_seq_bwd_kernel(GruSeqArgs a) {
    constexpr int R = 128 * U, K3 = 3 * R, KL = K3 / 32;
    extern __shared__ __align__(16) float smem[];
    float* s_w = smem;                          // [U][3R]: column c U + j of W_hh
    float* s_x = s_w + U * K3;                  // [G][3R]
    float* s_acc = s_x + (size_t)a.G * K3;      // [G][U]
    __shared__ int s_ok;
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int B = a.B, T = a.T;
    for (int i = threadIdx.x; i < U * K3; i += GS_THREADS) {
        const int j = i / K3, k = i - j * K3;
        s_w[i] = a.w_hh[(size_t)k * R + c * U + j];
    }
    __syncthreads();
    unsigned target = 0;
    for (int t = T - 1; t >= 0; --t) {
        for (int g0 = 0; g0 < B; g0 += a.G) {
            const int nb = min(a.G, B - g0);
            if (t + 1 < T) {
                for (int i = threadIdx.x; i < nb * (K3 / 4); i += GS_THREADS) {
                    const int bb = i / (K3 / 4), k4 = i - bb * (K3 / 4);
                    reinterpret_cast<float4*>(s_x)[i] =
                        __ldcg(reinterpret_cast<const float4*>(a.dgh + ((size_t)(g0 + bb) * T + t + 1) * K3) + k4);
                }
                __syncthreads();
                for (int bb = warp; bb < nb; bb += GS_WARPS) {
                    float acc[U];
#pragma unroll
                    for (int j = 0; j < U; ++j) acc[j] = 0.f;
                    const float* x = s_x + (size_t)bb * K3;
#pragma unroll 4
                    for (int i = 0; i < KL; ++i) {
                        const float v = x[lane + 32 * i];
#pragma unroll
                        for (int j = 0; j < U; ++j) acc[j] = fmaf(s_w[j * K3 + lane + 32 * i], v, acc[j]);
                    }
#pragma unroll
                    for (int j = 0; j < U; ++j) acc[j] = warp_sum(acc[j]);
                    if (lane == 0) {
#pragma unroll
                        for (int j = 0; j < U; ++j) s_acc[bb * U + j] = acc[j];
                    }
                }
                __syncthreads();
            }
            for (int e = threadIdx.x; e < nb * U; e += GS_THREADS) {
                const int bb = e / U, j = e - bb * U, b = g0 + bb, u = c * U + j;
                const size_t row = (size_t)b * T + t;
                float dh = a.dh_ext[row * R + u];
                if (t + 1 < T) dh += a.carry[(size_t)b * R + u] + s_acc[bb * U + j];
                const float* sv = a.saved + row * 4 * R;
                const float r = sv[u], z = sv[R + u], n = sv[2 * R + u], ghn = sv[3 * R + u];
                const float hp = t > 0 ? a.h[(row - 1) * R + u] : 0.f;
                const float dn = dh * (1.f - z), dz = dh * (hp - n);
                const float dnh = dn * (1.f - n * n);
                const float drh = dnh * ghn * (r * (1.f - r));
                const float dzh = dz * (z * (1.f - z));
                float* gi = a.dgi + row * K3;
                float* gh = a.dgh + row * K3;
                gi[u] = drh; gi[R + u] = dzh; gi[2 * R + u] = dnh;
                gh[u] = drh; gh[R + u] = dzh; gh[2 * R + u] = r * dnh;
                a.carry[(size_t)b * R + u] = z * dh;
                if (a.dh_dbg) a.dh_dbg[row * R + u] = dh;
            }
            __syncthreads();
        }
        if (t > 0 && !grid_barrier(a.bar, target, gridDim.x, a.abort_flag, &s_ok, false)) return;
    }
}

// ---- upsampling layer adjoint ----
// forward (wavernn.cu): out[c, i] = sum_{k=-s..s} w[k + s] in[c, (i + k) / s] over 0 <= i + k < lo = len s.
// din[c, j] = sum_{p = j s .. j s + s - 1} sum_k [0 <= p - k < lo] w[k + s] dout[c, p - k]
__global__ void wavernn_upsample_bwd_in_kernel(int C, int len, int s, const float* __restrict__ w, const float* __restrict__ dout,
                                               float* __restrict__ din) {
    const long long n = (long long)C * len;
    const int lo = len * s;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx / len), j = (int)(idx - (long long)c * len);
        const float* d = dout + (size_t)c * lo;
        float acc = 0.f;
        for (int p = j * s; p < j * s + s; ++p)
            for (int k = -s; k <= s; ++k) {
                const int i = p - k;
                if (i >= 0 && i < lo) acc = fmaf(w[k + s], d[i], acc);
            }
        din[idx] = acc;
    }
}

constexpr int UPS_CHUNKS = 64;
// part[tap][chunk] = sum over the chunk's slice of the flat (c, i) range of dout[c, i] in[c, (i + k) / s], 0 <= i + k < lo
__global__ void __launch_bounds__(256) wavernn_upsample_bwd_fir_part_kernel(int C, int len, int s, const float* __restrict__ in,
                                                                            const float* __restrict__ dout, float* __restrict__ part) {
    __shared__ float red[33];
    const int tap = blockIdx.x, chunk = blockIdx.y, k = tap - s, lo = len * s;
    const long long n = (long long)C * lo, per = (n + UPS_CHUNKS - 1) / UPS_CHUNKS;
    const long long e0 = chunk * per, e1 = min(n, e0 + per);
    float acc = 0.f;
    for (long long e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
        const int c = (int)(e / lo), i = (int)(e - (long long)c * lo), p = i + k;
        if (p >= 0 && p < lo) acc = fmaf(dout[e], in[(size_t)c * len + p / s], acc);
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) part[tap * UPS_CHUNKS + chunk] = acc;
}
__global__ void wavernn_upsample_bwd_fir_sum_kernel(int taps, const float* __restrict__ part, float* __restrict__ dfir) {
    const int tap = blockIdx.x * blockDim.x + threadIdx.x;
    if (tap >= taps) return;
    float acc = 0.f;
    for (int q = 0; q < UPS_CHUNKS; ++q) acc += part[tap * UPS_CHUNKS + q];
    dfir[tap] += acc;
}

// ---- aux stretch adjoint: dup [B, F hop, C] -> daux [B, F, C], daux[b, f, c] = sum_{q < hop} dup[b, f hop + q, c] ----
__global__ void wavernn_stretch_bwd_kernel(int B, int F, int C, int hop, const float* __restrict__ dup, float* __restrict__ daux) {
    const long long n = (long long)B * F * C;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int cc = (int)(idx % C);
        const long long bf = idx / C;                  // b F + f
        const float* d = dup + (size_t)bf * hop * C + cc;
        float acc = 0.f;
        for (int q = 0; q < hop; ++q) acc += d[(size_t)q * C];
        daux[idx] = acc;
    }
}

// ---- fixed-order column sums: part[chunk][col] over the chunk's rows, then out[col] += the chunks in order ----
constexpr int COLSUM_CHUNKS = 64;
__global__ void column_sum_part_kernel(long long rows, int cols, const float* __restrict__ x, float* __restrict__ part) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x, chunk = blockIdx.y;
    if (col >= cols) return;
    const long long per = (rows + COLSUM_CHUNKS - 1) / COLSUM_CHUNKS, r0 = chunk * per, r1 = min(rows, r0 + per);
    float acc = 0.f;
    for (long long r = r0; r < r1; ++r) acc += x[(size_t)r * cols + col];
    part[(size_t)chunk * cols + col] = acc;
}
__global__ void column_sum_add_kernel(int cols, const float* __restrict__ part, float* __restrict__ out) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= cols) return;
    float acc = 0.f;
    for (int q = 0; q < COLSUM_CHUNKS; ++q) acc += part[(size_t)q * cols + col];
    out[col] += acc;
}

// ---- losses ----
__device__ __forceinline__ float softplus_t(float x) { return x > 20.f ? x : log1pf(expf(x)); }     // F.softplus (beta 1, threshold 20)
__device__ __forceinline__ float dsoftplus_t(float x) { return x > 20.f ? 1.f : sigmoidf_acc(x); }

// cross entropy, one warp per row: loss[row] = logsumexp - logit[y], dlogits[row] = (softmax - onehot(y)) / N; a label outside [0, n)
// gives a NaN loss
__global__ void wavernn_loss_raw_kernel(long long N, int n, const float* __restrict__ logits, const int* __restrict__ y,
                                        float* __restrict__ loss, float* __restrict__ dlogits) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    const float invN = (float)(1.0 / (double)N);
    for (long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
        const float* l = logits + (size_t)row * n;
        float* d = dlogits + (size_t)row * n;
        const int lab = y[row];
        float mx = -INFINITY;
        for (int k = lane; k < n; k += 32) mx = fmaxf(mx, l[k]);
        mx = warp_max(mx);
        float s = 0.f;
        for (int k = lane; k < n; k += 32) s += expf(l[k] - mx);
        s = warp_sum(s);
        const float inv_s = 1.f / s;
        for (int k = lane; k < n; k += 32) d[k] = (expf(l[k] - mx) * inv_s - (k == lab ? 1.f : 0.f)) * invN;
        if (lane == 0) loss[row] = (lab >= 0 && lab < n) ? logf(s) + mx - l[lab] : NAN;
    }
}

// discretized mixture of logistics (fatchord's discretized_mix_logistic_loss, 65536 classes), one warp per row, lane j < nr: mixture j
__global__ void wavernn_loss_mol_kernel(long long N, int nr, const float* __restrict__ logits, const float* __restrict__ y,
                                        float* __restrict__ loss, float* __restrict__ dlogits) {
    const float LOG_SCALE_MIN = -32.23619130191664f;      // log(1e-14)
    const float HALF_BIN = 1.f / 65535.f;
    const float LOG_HALF_CLASSES = 10.3971924f;            // log(65535 / 2) = log(32767.5)
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    const float invN = (float)(1.0 / (double)N);
    for (long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
        const float* l = logits + (size_t)row * 3 * nr;
        float* d = dlogits + (size_t)row * 3 * nr;
        const float yv = y[row];
        const bool on = lane < nr;
        float lp = -INFINITY, logprob = 0.f, dmu_l = 0.f, dls_l = 0.f;     // dmu_l / dls_l: d logprob / d mean, d log_scale
        if (on) {
            lp = l[lane];
            const float mu = l[nr + lane], lsr = l[2 * nr + lane];
            const float ls = fmaxf(lsr, LOG_SCALE_MIN);
            const float cy = yv - mu, inv = expf(-ls);
            const float plus = inv * (cy + HALF_BIN), mn = inv * (cy - HALF_BIN), mid = inv * cy;
            float dplus = 0.f, dmin = 0.f, dmid = 0.f, dls_direct = 0.f;
            if (yv < -0.999f) {
                logprob = plus - softplus_t(plus);
                dplus = 1.f - dsoftplus_t(plus);
            } else if (yv > 0.999f) {
                logprob = -softplus_t(mn);
                dmin = -dsoftplus_t(mn);
            } else {
                const float cp = sigmoidf_acc(plus), cm = sigmoidf_acc(mn), cd = cp - cm;
                if (cd > 1e-5f) {
                    logprob = logf(fmaxf(cd, 1e-12f));
                    dplus = cp * (1.f - cp) / cd;
                    dmin = -cm * (1.f - cm) / cd;
                } else {
                    logprob = mid - ls - 2.f * softplus_t(mid) - LOG_HALF_CLASSES;
                    dmid = 1.f - 2.f * dsoftplus_t(mid);
                    dls_direct = -1.f;
                }
            }
            dmu_l = -inv * (dplus + dmin + dmid);
            dls_l = lsr >= LOG_SCALE_MIN ? dls_direct - (plus * dplus + mn * dmin + mid * dmid) : 0.f;
        }
        const float m = warp_max(lp);
        const float e = on ? expf(lp - m) : 0.f;
        const float s = warp_sum(e);
        const float a = on ? logprob + (lp - m - logf(s)) : -INFINITY;
        const float M = warp_max(a);
        const float ea = on ? expf(a - M) : 0.f;
        const float S = warp_sum(ea);
        if (on) {
            const float w = ea / S, sm = e / s, g = -w * invN;
            d[lane] = (sm - w) * invN;
            d[nr + lane] = g * dmu_l;
            d[2 * nr + lane] = g * dls_l;
        }
        if (lane == 0) loss[row] = -(M + logf(S));
    }
}

// out[0] = sum(rows) / N in a fixed order: thread i sums rows i, i + 1024, ..., then one block reduction
__global__ void __launch_bounds__(1024) wavernn_loss_sum_kernel(long long N, const float* __restrict__ rows, float* __restrict__ out) {
    __shared__ float red[33];
    float acc = 0.f;
    for (long long i = threadIdx.x; i < N; i += blockDim.x) acc += rows[i];
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) out[0] = (float)((double)acc / (double)N);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int gru_seq_validate(const b200tts_gru_seq_shape& s) {
    B200_REQUIRE(s.B >= 1 && s.B <= GS_MAX_B, "gru_seq: batch %d outside [1, %d]", s.B, GS_MAX_B);
    B200_REQUIRE(s.R >= GS_CTAS && s.R % GS_CTAS == 0 && s.R <= GS_MAX_U * GS_CTAS, "gru_seq: hidden size %d must be a multiple of %d, at most %d",
                 s.R, GS_CTAS, GS_MAX_U * GS_CTAS);
    B200_REQUIRE(s.T >= 1 && s.T <= GS_MAX_T, "gru_seq: %d steps outside [1, %d]", s.T, GS_MAX_T);
    return B200TTS_OK;
}

static int gru_seq_check(const b200tts_gru_seq_shape& s, const void* ws, size_t ws_bytes) {
    B200_TRY(gru_seq_validate(s));
    const size_t need = b200tts_gru_seq_workspace_bytes(&s);
    B200_REQUIRE(ws && ws_bytes >= need, "gru_seq: workspace of %zu bytes is smaller than the %zu required", ws_bytes, need);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "gru_seq: workspace must be 256-byte aligned");
    return B200TTS_OK;
}

// utterances per staged group: as many as fit beside the weights (one CTA per SM)
static int gru_seq_group(int B, size_t weight_floats, size_t row_floats, size_t acc_floats) {
    const size_t avail = (PERSIST_SMEM_LIMIT - weight_floats * sizeof(float)) / sizeof(float);
    const int g = (int)(avail / (row_floats + acc_floats));
    return g < B ? g : B;
}

template <typename F>
static const void* gru_seq_pick(int U, F pick) {
    switch (U) {
        case 1: return pick(std::integral_constant<int, 1>());
        case 2: return pick(std::integral_constant<int, 2>());
        case 3: return pick(std::integral_constant<int, 3>());
        case 4: return pick(std::integral_constant<int, 4>());
        default: return pick(std::integral_constant<int, 5>());
    }
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_gru_seq_saved_bytes(const b200tts_gru_seq_shape* shape) {
    if (!shape) { set_last_error("gru_seq_saved_bytes: null shape"); return 0; }
    const b200tts_gru_seq_shape& s = *shape;
    if (gru_seq_validate(s) != B200TTS_OK) return 0;
    return (size_t)s.B * s.T * 4 * s.R * sizeof(float);
}

// workspace: barrier counter (+ abort flag at +128), then the reverse loop's carry [B, R]
size_t b200tts_gru_seq_workspace_bytes(const b200tts_gru_seq_shape* shape) {
    if (!shape) { set_last_error("gru_seq_workspace_bytes: null shape"); return 0; }
    const b200tts_gru_seq_shape& s = *shape;
    if (gru_seq_validate(s) != B200TTS_OK) return 0;
    return 256 + align_up_sz((size_t)s.B * s.R * sizeof(float), 256);
}

int b200tts_gru_seq_forward(const b200tts_gru_seq_shape* shape, const float* gi, const float* w_hh, const float* b_hh, float* h, void* saved,
                            void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && gi && w_hh && b_hh && h && saved, "gru_seq_forward: null argument");
    const b200tts_gru_seq_shape& s = *shape;
    B200_TRY(gru_seq_check(s, workspace, workspace_bytes));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const int U = s.R / GS_CTAS;
    GruSeqArgs a{};
    a.B = s.B; a.T = s.T;
    a.G = gru_seq_group(s.B, (size_t)3 * U * s.R, s.R, 3 * U);
    a.gi = gi; a.w_hh = w_hh; a.b_hh = b_hh; a.h = h; a.saved = static_cast<float*>(saved);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    a.bar = reinterpret_cast<unsigned*>(base);
    a.abort_flag = reinterpret_cast<int*>(base + 128);
    a.carry = reinterpret_cast<float*>(base + 256);
    B200_CUDA(cudaMemsetAsync(base, 0, sizeof(unsigned), st));     // the barrier counter; the abort flag stays until the caller clears it
    const size_t smem = ((size_t)3 * U * s.R + (size_t)a.G * (s.R + 3 * U)) * sizeof(float);
    const void* fn = gru_seq_pick(U, [](auto u) { return (const void*)gru_seq_fwd_kernel<decltype(u)::value>; });
    void* params[] = {&a};
    return launch_persistent("gru_seq_fwd", fn, GS_CTAS, GS_THREADS, smem, false, params, st);
}

int b200tts_gru_seq_backward(const b200tts_gru_seq_shape* shape, const float* w_hh, const float* h, const void* saved, const float* dh_ext,
                             float* dgi, float* dgh, float* dh_dbg, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && w_hh && h && saved && dh_ext && dgi && dgh, "gru_seq_backward: null argument");
    const b200tts_gru_seq_shape& s = *shape;
    B200_TRY(gru_seq_check(s, workspace, workspace_bytes));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const int U = s.R / GS_CTAS;
    GruSeqArgs a{};
    a.B = s.B; a.T = s.T;
    a.G = gru_seq_group(s.B, (size_t)3 * U * s.R, 3 * s.R, U);
    a.w_hh = w_hh; a.h = const_cast<float*>(h); a.saved = static_cast<float*>(const_cast<void*>(saved));
    a.dh_ext = dh_ext; a.dgi = dgi; a.dgh = dgh; a.dh_dbg = dh_dbg;
    unsigned char* base = static_cast<unsigned char*>(workspace);
    a.bar = reinterpret_cast<unsigned*>(base);
    a.abort_flag = reinterpret_cast<int*>(base + 128);
    a.carry = reinterpret_cast<float*>(base + 256);
    B200_CUDA(cudaMemsetAsync(base, 0, sizeof(unsigned), st));
    const size_t smem = ((size_t)3 * U * s.R + (size_t)a.G * (3 * s.R + U)) * sizeof(float);
    const void* fn = gru_seq_pick(U, [](auto u) { return (const void*)gru_seq_bwd_kernel<decltype(u)::value>; });
    void* params[] = {&a};
    return launch_persistent("gru_seq_bwd", fn, GS_CTAS, GS_THREADS, smem, false, params, st);
}

int b200tts_gru_seq_aborted(const b200tts_gru_seq_shape* shape, const void* workspace, size_t workspace_bytes, int* aborted, void* stream) {
    B200_REQUIRE(shape && aborted, "gru_seq_aborted: null argument");
    B200_TRY(require_device());
    B200_TRY(gru_seq_check(*shape, workspace, workspace_bytes));
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaMemcpyAsync(aborted, static_cast<const unsigned char*>(workspace) + 128, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200TTS_OK;
}

int b200tts_gru_seq_abort_flag_copy(const b200tts_gru_seq_shape* shape, const void* workspace, size_t workspace_bytes, int* dst, void* stream) {
    B200_REQUIRE(shape && dst, "gru_seq_abort_flag_copy: null argument");
    B200_TRY(gru_seq_check(*shape, workspace, workspace_bytes));
    B200_TRY(require_device());
    B200_CUDA(cudaMemcpyAsync(dst, static_cast<const unsigned char*>(workspace) + 128, sizeof(int), cudaMemcpyDefault, (cudaStream_t)stream));
    return B200TTS_OK;
}

size_t b200tts_wavernn_upsample_layer_backward_workspace_bytes(int C, int len, int scale) {
    if (wavernn_upsample_layer_check(C, len, scale) != B200TTS_OK) return 0;
    return (size_t)(2 * scale + 1) * UPS_CHUNKS * sizeof(float);
}

int b200tts_wavernn_upsample_layer_backward(int C, int len, int scale, const float* fir, const float* in, const float* dout, float* din,
                                            float* dfir, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(fir && dout && (din || dfir), "wavernn_upsample_layer_backward: null argument");
    B200_TRY(wavernn_upsample_layer_check(C, len, scale));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wavernn_upsample_bwd", st);
    if (din) {
        wavernn_upsample_bwd_in_kernel<<<grid_for((size_t)C * len), 256, 0, st>>>(C, len, scale, fir, dout, din);
        B200_LAUNCH_CHECK();
    }
    if (dfir) {
        const size_t need = b200tts_wavernn_upsample_layer_backward_workspace_bytes(C, len, scale);
        B200_REQUIRE(in && workspace && workspace_bytes >= need, "wavernn_upsample_layer_backward: d fir needs the layer input and %zu workspace bytes",
                     need);
        float* part = static_cast<float*>(workspace);
        wavernn_upsample_bwd_fir_part_kernel<<<dim3(2 * scale + 1, UPS_CHUNKS), 256, 0, st>>>(C, len, scale, in, dout, part);
        B200_LAUNCH_CHECK();
        wavernn_upsample_bwd_fir_sum_kernel<<<1, 64, 0, st>>>(2 * scale + 1, part, dfir);
        B200_LAUNCH_CHECK();
    }
    return B200TTS_OK;
}

int b200tts_wavernn_stretch_backward(int B, int F, int C, int hop, const float* dup, float* daux, void* stream) {
    B200_REQUIRE(dup && daux, "wavernn_stretch_backward: null argument");
    B200_REQUIRE(B >= 1 && F >= 1 && C >= 1 && hop >= 1 && (long long)B * F * hop * C < (1ll << 40),
                 "wavernn_stretch_backward: bad dimensions (B = %d, frames = %d, C = %d, hop = %d)", B, F, C, hop);
    B200_TRY(require_device());
    wavernn_stretch_bwd_kernel<<<grid_for((size_t)B * F * C), 256, 0, (cudaStream_t)stream>>>(B, F, C, hop, dup, daux);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

size_t b200tts_column_sum_workspace_bytes(int cols) { return cols >= 1 ? (size_t)COLSUM_CHUNKS * cols * sizeof(float) : 0; }

int b200tts_column_sum(long long rows, int cols, const float* x, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(x && out, "column_sum: null argument");
    B200_REQUIRE(rows >= 1 && cols >= 1 && rows * cols < (1ll << 40), "column_sum: bad dimensions (rows = %lld, cols = %d)", rows, cols);
    B200_TRY(require_device());
    const size_t need = b200tts_column_sum_workspace_bytes(cols);
    B200_REQUIRE(workspace && workspace_bytes >= need, "column_sum: workspace of %zu bytes is smaller than the %zu required", workspace_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    float* part = static_cast<float*>(workspace);
    column_sum_part_kernel<<<dim3((cols + 255) / 256, COLSUM_CHUNKS), 256, 0, st>>>(rows, cols, x, part);
    B200_LAUNCH_CHECK();
    column_sum_add_kernel<<<(cols + 255) / 256, 256, 0, st>>>(cols, part, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

size_t b200tts_wavernn_loss_workspace_bytes(long long N) { return N >= 1 ? (size_t)N * sizeof(float) : 0; }

int b200tts_wavernn_loss(int mode, long long N, int n_out, const float* logits, const void* target, float* loss, float* dlogits, void* workspace,
                         size_t workspace_bytes, void* stream) {
    B200_REQUIRE(logits && target && loss && dlogits, "wavernn_loss: null argument");
    B200_REQUIRE(N >= 1 && N < (1ll << 40), "wavernn_loss: %lld rows", N);
    if (mode == B200TTS_WAVERNN_RAW) {
        B200_REQUIRE(n_out >= 2 && n_out <= 65536, "wavernn_loss: RAW needs 2 to 65536 classes (n_out = %d)", n_out);
    } else {
        B200_REQUIRE(mode == B200TTS_WAVERNN_MOL, "wavernn_loss: unknown mode %d", mode);
        B200_REQUIRE(n_out % 3 == 0 && n_out >= 3 && n_out <= 96, "wavernn_loss: MOL needs 3 x (1..32) outputs (n_out = %d)", n_out);
    }
    B200_TRY(require_device());
    const size_t need = b200tts_wavernn_loss_workspace_bytes(N);
    B200_REQUIRE(workspace && workspace_bytes >= need, "wavernn_loss: workspace of %zu bytes is smaller than the %zu required", workspace_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("wavernn_loss", st);
    float* rows = static_cast<float*>(workspace);
    const int blocks = (int)((N + 7) / 8 > NUM_SMS * 16 ? NUM_SMS * 16 : (N + 7) / 8);
    if (mode == B200TTS_WAVERNN_RAW)
        wavernn_loss_raw_kernel<<<blocks, 256, 0, st>>>(N, n_out, logits, static_cast<const int*>(target), rows, dlogits);
    else
        wavernn_loss_mol_kernel<<<blocks, 256, 0, st>>>(N, n_out / 3, logits, static_cast<const float*>(target), rows, dlogits);
    B200_LAUNCH_CHECK();
    wavernn_loss_sum_kernel<<<1, 1024, 0, st>>>(N, rows, loss);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
