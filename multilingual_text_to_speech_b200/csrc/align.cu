// Forced alignment: the monotonic alignment search (Glow-TTS MAS) over attention probabilities, and per-utterance alignment scores.
//
// One CTA per utterance reads only its own rows of P in a fixed order with no global atomics, so an utterance's result does not depend
// on the batch it is computed in.
#include <float.h>
#include <algorithm>
#include "common.cuh"

namespace b200tts {

namespace {

constexpr int MAS_THREADS = 256;
constexpr int MAS_CPT = B200TTS_ALIGN_MAX_SYMBOLS / MAS_THREADS;      // symbols per thread and step
constexpr int SCORE_THREADS = 256;
constexpr size_t MAS_SMEM_LIMIT = 227 * 1024;
// two fp64 rows of the DP at the largest text length, then one back-pointer bit per cell
constexpr size_t MAS_ROWS_BYTES = 2 * sizeof(double) * B200TTS_ALIGN_MAX_SYMBOLS;
static_assert(B200TTS_ALIGN_MAX_SYMBOLS % MAS_THREADS == 0, "whole symbol chunks per thread");
static_assert(B200TTS_ALIGN_MAX_CELLS == (int)((MAS_SMEM_LIMIT - MAS_ROWS_BYTES) * 8), "B200TTS_ALIGN_MAX_CELLS follows from 227 KB");
static_assert(B200TTS_ALIGN_MAX_CELLS % 32 == 0, "whole back-pointer words");

__device__ __forceinline__ bool lengths_ok(int Lb, int Sb, int L, int S, int cells) {
    return Lb >= 1 && Lb <= L && Sb >= Lb && Sb <= S && (long long)Sb * Lb <= cells;
}

// Q[s][l] = log max(P[s, l], 1e-8) + max(Q[s-1][l], Q[s-1][l-1]) in fp64, Q[0][0] = log max(P[0, 0], 1e-8), every other cell of row 0
// and Q[s][-1] at -inf.  The back-pointer bit of cell (s, l) is 1 (advance: the path came from symbol l - 1) only when
// Q[s-1][l-1] > Q[s-1][l]; on equal values the path stays on symbol l.  Cells above the diagonal (l > s) stay -inf, and cells from which
// (S_b - 1, L_b - 1) cannot be reached are never on the path the backtrack follows, so neither needs a mask.  Bits are packed
// contiguously, cell s L_b + l, and set by one shared-memory atomicOr per warp and touched word; the backtrack is one thread's walk.
__global__ void __launch_bounds__(MAS_THREADS) mas_kernel(int S, int L, long long ld, long long bstride, int cells,
                                                          const float* __restrict__ P, const int* __restrict__ text_lengths,
                                                          const int* __restrict__ step_lengths, int* __restrict__ durations,
                                                          double* __restrict__ path_logp, int* __restrict__ path) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* rows = reinterpret_cast<double*>(smem_raw);                       // [2][L]
    unsigned* bits = reinterpret_cast<unsigned*>(rows + 2 * L);                 // [ceil(cells / 32)]
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int Lb = text_lengths[b], Sb = step_lengths[b];
    int* dur = durations + (size_t)b * L;
    int* pth = path ? path + (size_t)b * S : nullptr;
    if (!lengths_ok(Lb, Sb, L, S, cells)) {
        // lengths the host would have refused: a marked result, no access past the buffers
        for (int l = tid; l < L; l += blockDim.x) dur[l] = -1;
        if (pth) for (int s = tid; s < S; s += blockDim.x) pth[s] = -1;
        if (tid == 0) path_logp[b] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    const float* Pb = P + (size_t)b * bstride;
    const int words = (int)(((long long)Sb * Lb + 31) >> 5);
    for (int w = tid; w < words; w += blockDim.x) bits[w] = 0u;
    for (int l = tid; l < L; l += blockDim.x) {
        if (l >= Lb) dur[l] = 0;
        rows[l] = l == 0 ? log(fmax((double)Pb[0], 1e-8)) : -INFINITY;
    }
    if (pth) for (int s = Sb + tid; s < S; s += blockDim.x) pth[s] = -1;

    float p[MAS_CPT];
#pragma unroll
    for (int k = 0; k < MAS_CPT; ++k) {
        const int l = k * MAS_THREADS + tid;
        p[k] = (Sb > 1 && l < Lb) ? Pb[ld + l] : 0.f;
    }
    __syncthreads();
    for (int s = 1; s < Sb; ++s) {
        const double* prev = rows + ((s - 1) & 1) * L;
        double* cur = rows + (s & 1) * L;
        float pn[MAS_CPT];
#pragma unroll
        for (int k = 0; k < MAS_CPT; ++k) {                                        // next step's weights, off this step's chain
            const int l = k * MAS_THREADS + tid;
            pn[k] = (s + 1 < Sb && l < Lb) ? Pb[(size_t)(s + 1) * ld + l] : 0.f;
        }
        const long long row0 = (long long)s * Lb;
#pragma unroll
        for (int k = 0; k < MAS_CPT; ++k) {
            const int l0 = k * MAS_THREADS;
            if (l0 >= Lb) break;                                                   // uniform over the block
            const int l = l0 + tid;
            bool adv = false;
            if (l < Lb) {
                const double stay = prev[l], diag = l > 0 ? prev[l - 1] : -INFINITY;
                adv = diag > stay;
                cur[l] = log(fmax((double)p[k], 1e-8)) + (adv ? diag : stay);
            }
            const unsigned m = __ballot_sync(0xffffffffu, adv);
            if (lane == 0 && m) {
                const long long i0 = row0 + l0 + (tid & ~31);
                const int w = (int)(i0 >> 5), o = (int)(i0 & 31);
                atomicOr(bits + w, m << o);
                if (o && (m >> (32 - o))) atomicOr(bits + w + 1, m >> (32 - o));
            }
        }
#pragma unroll
        for (int k = 0; k < MAS_CPT; ++k) p[k] = pn[k];
        __syncthreads();
    }
    if (tid != 0) return;
    path_logp[b] = rows[((Sb - 1) & 1) * L + Lb - 1];
    int l = Lb - 1, run = 0;
    for (int s = Sb - 1; s >= 0; --s) {
        if (pth) pth[s] = l;
        ++run;
        const long long i = (long long)s * Lb + l;
        if (s > 0 && ((bits[i >> 5] >> (i & 31)) & 1u)) {
            dur[l] = run;
            run = 0;
            --l;
        }
    }
    dur[l] = run;       // l == 0: every cell on the walk lies in the reachable band
}

// Scores over steps s < S_b and symbols l < L_b.  Warp w takes steps w, w + 8, ...: the step's max weight and its first argmax; eight
// steps at a time go through shared memory so the argmax moves are taken between consecutive steps in order.  Each thread then sums
// whole columns for the coverage.
__global__ void __launch_bounds__(SCORE_THREADS) scores_kernel(int S, int L, long long ld, long long bstride, const float* __restrict__ P,
                                                               const int* __restrict__ text_lengths, const int* __restrict__ step_lengths,
                                                               float* __restrict__ focus, float* __restrict__ coverage,
                                                               int* __restrict__ max_jump, int* __restrict__ moves_back) {
    constexpr int WARPS = SCORE_THREADS / 32;
    __shared__ int am[WARPS + 1];
    __shared__ double red_d[SCORE_THREADS];
    __shared__ int red_i[3][SCORE_THREADS];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Lb = text_lengths[b], Sb = step_lengths[b];
    if (!(Lb >= 1 && Lb <= L && Sb >= 1 && Sb <= S)) {
        if (tid == 0) {
            focus[b] = coverage[b] = __int_as_float(0x7fc00000);
            max_jump[b] = moves_back[b] = -1;
        }
        return;
    }
    const float* Pb = P + (size_t)b * bstride;
    double fsum = 0.0;
    int jump = 0, back = 0;
    if (tid == 0) am[WARPS] = -1;
    for (int s0 = 0; s0 < Sb; s0 += WARPS) {
        __syncthreads();                                                          // am[WARPS] holds the previous tile's last argmax
        const int s = s0 + warp;
        if (s < Sb) {
            float mx = -INFINITY;
            int ix = 0;
            for (int l = lane; l < Lb; l += 32) {
                const float v = Pb[(size_t)s * ld + l];
                if (v > mx) { mx = v; ix = l; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float om = __shfl_xor_sync(0xffffffffu, mx, o);
                const int oi = __shfl_xor_sync(0xffffffffu, ix, o);
                if (om > mx || (om == mx && oi < ix)) { mx = om; ix = oi; }
            }
            if (lane == 0) { am[warp] = ix; fsum += (double)mx; }
        }
        __syncthreads();
        if (tid < WARPS && s0 + tid < Sb) {
            const int before = tid == 0 ? am[WARPS] : am[tid - 1];
            if (before >= 0) {
                const int d = am[tid] - before;
                jump = max(jump, d);
                back |= d < 0;
            }
        }
        __syncthreads();
        if (tid == 0) am[WARPS] = am[min(WARPS, Sb - s0) - 1];
    }
    int covered = 0;
    for (int l = tid; l < Lb; l += blockDim.x) {
        double c = 0.0;
        for (int s = 0; s < Sb; ++s) c += (double)Pb[(size_t)s * ld + l];
        covered += c >= 0.5;
    }
    red_d[tid] = fsum;
    red_i[0][tid] = covered;
    red_i[1][tid] = jump;
    red_i[2][tid] = back;
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
        if (tid < h) {
            red_d[tid] += red_d[tid + h];
            red_i[0][tid] += red_i[0][tid + h];
            red_i[1][tid] = max(red_i[1][tid], red_i[1][tid + h]);
            red_i[2][tid] |= red_i[2][tid + h];
        }
        __syncthreads();
    }
    if (tid == 0) {
        focus[b] = (float)(red_d[0] / Sb);
        coverage[b] = (float)((double)red_i[0][0] / Lb);
        max_jump[b] = red_i[1][0];
        moves_back[b] = red_i[2][0];
    }
}

}  // namespace

static int align_validate(const b200tts_align_shape& s) {
    B200_REQUIRE(s.B >= 1 && s.S >= 1, "align: need B >= 1 and S >= 1 (B = %d, S = %d)", s.B, s.S);
    B200_REQUIRE(s.L >= 1 && s.L <= B200TTS_ALIGN_MAX_SYMBOLS, "align: L = %d must be in [1, %d]", s.L, B200TTS_ALIGN_MAX_SYMBOLS);
    B200_REQUIRE(s.ld >= s.L && s.batch_stride >= 0, "align: need ld >= L and batch_stride >= 0 (ld = %lld, L = %d, batch_stride = %lld)",
                 s.ld, s.L, s.batch_stride);
    return B200TTS_OK;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

int b200tts_monotonic_alignment(const b200tts_align_shape* shape, const float* P, const int32_t* text_lengths, const int32_t* step_lengths,
                                int32_t* durations_out, double* path_logp_out, int32_t* path_out, void* stream) {
    B200_REQUIRE(shape && P && text_lengths && step_lengths && durations_out && path_logp_out, "monotonic_alignment: null argument");
    const b200tts_align_shape& s = *shape;
    B200_TRY(align_validate(s));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const int cells = (int)std::min<long long>((long long)s.S * s.L, B200TTS_ALIGN_MAX_CELLS);
    const size_t smem = 2 * sizeof(double) * s.L + (size_t)(cells + 31) / 32 * sizeof(unsigned);
    B200_CUDA(cudaFuncSetAttribute(mas_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt("monotonic_alignment", st);
    mas_kernel<<<s.B, MAS_THREADS, smem, st>>>(s.S, s.L, s.ld, s.batch_stride, cells, P, text_lengths, step_lengths, durations_out,
                                               path_logp_out, path_out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_alignment_scores(const b200tts_align_shape* shape, const float* P, const int32_t* text_lengths, const int32_t* step_lengths,
                             float* focus_out, float* coverage_out, int32_t* max_jump_out, int32_t* moves_back_out, void* stream) {
    B200_REQUIRE(shape && P && text_lengths && step_lengths && focus_out && coverage_out && max_jump_out && moves_back_out,
                 "alignment_scores: null argument");
    const b200tts_align_shape& s = *shape;
    B200_TRY(align_validate(s));
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("alignment_scores", st);
    scores_kernel<<<s.B, SCORE_THREADS, 0, st>>>(s.S, s.L, s.ld, s.batch_stride, P, text_lengths, step_lengths, focus_out, coverage_out,
                                                 max_jump_out, moves_back_out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
