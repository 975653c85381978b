// Shared device/host helpers for the b200tts hot-path library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b200tts.h"

namespace b200tts {

void set_last_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what, const char* file, int line);
// B200TTS_OK when the current device is a usable sm_90 GPU (cached once it is); entry points call it before any device work
int require_device();

#define B200_CUDA(call)                                                             \
    do {                                                                            \
        int _st = ::b200tts::check_cuda((call), #call, __FILE__, __LINE__);         \
        if (_st != B200TTS_OK) return _st;                                          \
    } while (0)

#define B200_LAUNCH_CHECK() B200_CUDA(cudaGetLastError())

#define B200_REQUIRE(cond, ...)                                                     \
    do {                                                                            \
        if (!(cond)) {                                                              \
            ::b200tts::set_last_error(__VA_ARGS__);                                 \
            return B200TTS_ERR_INVALID;                                             \
        }                                                                           \
    } while (0)

#define B200_TRY(expr)                                                              \
    do {                                                                            \
        int _st = (expr);                                                           \
        if (_st != B200TTS_OK) return _st;                                          \
    } while (0)

// Named kernel timers (b200tts_kernel_timing): when enabled, CUDA events are recorded on the launching stream around the dominant kernels;
// bench.py reads per-name totals after a synchronize.  Disabled (the default) they cost one relaxed load.
void ktimer_start(const char* name, cudaStream_t st);
void ktimer_stop(const char* name, cudaStream_t st);
struct KernelTimer {
    const char* name; cudaStream_t st;
    KernelTimer(const char* n, cudaStream_t s) : name(n), st(s) { ktimer_start(n, s); }
    ~KernelTimer() { ktimer_stop(name, st); }
};

// WaveRNN upsampling layer (wavernn.cu): the shape check its forward and backward entry points share
int wavernn_upsample_layer_check(int C, int len, int scale);
// y[r, :] = lfilter([1], [1, -a], y[r, :]) for each of `rows` rows of `len` samples, no normalisation (vocoder.cu; the WaveRNN folds)
int deemphasis_rows(int rows, int len, float a, float* y, cudaStream_t st);

// SMs of the H100 SXM the library is built for: grid sizes of the grid-stride kernels and the co-residency limit of the persistent loops
constexpr int NUM_SMS = 132;

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline size_t align_up_sz(size_t x, size_t a) { return (x + a - 1) / a * a; }
// grid of a 256-thread grid-stride kernel over n elements: one thread per element, at most 16 CTAs per SM
static inline int grid_for(size_t n) {
    size_t g = (n + 255) / 256;
    return (int)(g > NUM_SMS * 16 ? NUM_SMS * 16 : (g < 1 ? 1 : g));
}

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum / max; `scratch` must hold >= 33 floats; every thread gets the result.
__device__ __forceinline__ float block_sum(float v, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = lane < nw ? scratch[lane] : 0.f;
        t = warp_sum(t);
        if (lane == 0) scratch[32] = t;
    }
    __syncthreads();
    return scratch[32];
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = lane < nw ? scratch[lane] : -INFINITY;
        t = warp_max(t);
        if (lane == 0) scratch[32] = t;
    }
    __syncthreads();
    return scratch[32];
}

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.f / (1.f + expf(-x)); }

// ---------------------------------------------------------------------------------------------
// GEMM (gemm.cu):  C = alpha * op(A) . op(B) + beta * C + bias[n]
//   op(A)(m,k) = transA ? A[k*lda+m] : A[m*lda+k];  op(B)(k,n) = transB ? B[n*ldb+k] : B[k*ldb+n]
//   batch > 1: pointers advance by stride{A,B,C}.  splitk > 1: raw partial sums are written to
//   `partial` as [splitk][batch][M][N] (dense) and, unless `keep_partials`, reduced into C.
// ---------------------------------------------------------------------------------------------
struct GemmDesc {
    const float* A = nullptr;
    const float* B = nullptr;
    float* C = nullptr;
    const float* bias = nullptr;
    int M = 0, N = 0, K = 0;
    int lda = 0, ldb = 0, ldc = 0;
    int transA = 0, transB = 0;
    float alpha = 1.f, beta = 0.f;
    int batch = 1;
    long long strideA = 0, strideB = 0, strideC = 0;
    int a_batch_mod = 0;          // > 0: A advances by strideA * (batch_index % a_batch_mod)
    int splitk = 1;
    float* partial = nullptr;     // required when splitk > 1
    int keep_partials = 0;        // 1: leave the reduction to the consumer kernel (C untouched)
    // optional (wgmma path, batch == 1): op(A) already available as bf16, read through TMA directly (no packing pass); A / lda are then
    // ignored by that path, the other paths still multiply A.  !transA: [M, K] rows, K contiguous, row stride lda16 (multiple of 8,
    // 16-byte aligned base).  transA (and kin == 0): [K, M] rows, M contiguous, row stride lda16 (multiple of 64, 16-byte aligned base),
    // an MN-major operand like B16: the columns up to the next multiple of 64 beyond M must be readable (their products are never stored)
    const void* A16 = nullptr;
    int lda16 = 0;
    // optional (wgmma path, !transB, batch == 1): op(B) = B [K, N] already available as bf16 rows, row stride ldb16 elements (multiple of
    // 64, 16-byte aligned base); the columns up to the next multiple of 64 beyond N must be readable (their products are never stored).
    // Read in place through TMA as an MN-major operand: no packing pass
    const void* B16 = nullptr;
    int ldb16 = 0;
    // optional two-level K (wgmma path only; needs !transA && transB): K = kouter * kin, element (row, q * kin + l) of op(A) lives at
    // A[q * kosA + row * lda + l] (op(B) likewise with kosB): sums a product over `kouter` separately stored slabs in ONE GEMM.
    // the SIMT and mma.sync kernels reject kin > 0 (B200TTS_ERR_INVALID) when the wgmma path does not take the product
    int kin = 0;
    long long kosA = 0, kosB = 0;
};

// pack cache of the wgmma GEMM (gemm_tc.cu): operands packed inside a begin / end scope are reused by later products of the scope
void tc_pack_cache_begin();
void tc_pack_cache_end();
// the wgmma GEMM's packing scratch (b200tts_set_scratch; null disables the path) and its on / off switch (b200tts_set_tensor_core_gemm)
void set_tc_scratch(void* ptr, size_t bytes);
void set_tc_enabled(int on);

// Arguments of the SIMT (gemm.cu) and mma.sync (gemm_bf16.cu) kernels, filled from a GemmDesc by gemm.cu.  kcontig: the operand is
// contiguous along k; vec: 16-byte vector loads are legal; kchunk: k range of one split, a multiple of the kernel's k-block.
struct GemmKernelArgs {
    const float* A; const float* B; float* C; const float* bias; float* partial;
    int M, N, K, lda, ldb, ldc;
    int a_kcontig, b_kcontig, a_vec, b_vec;
    float alpha, beta;
    int batch, splitk, kchunk, a_batch_mod;
    long long strideA, strideB, strideC;
};
constexpr int GEMM_MMA_BK = 32;     // k-block of the mma.sync kernel
int launch_gemm_mma(const GemmKernelArgs& p, cudaStream_t stream);
// Split-K reduction shared by every GEMM path: C[b] = alpha * sum_{z = 0 .. splitk - 1} partial[z][b] + bias[n] + beta * C[b], summed in
// that fixed order (deterministic); partial is [splitk][batch][M][N] (dense), C[b] starts at C + b * strideC with row stride ldc
int splitk_reduce(const float* partial, float* C, const float* bias, int M, int N, int ldc, int batch, int splitk, long long strideC,
                  float alpha, float beta, cudaStream_t stream);
// wgmma path (gemm_tc.cu): returns B200TTS_OK and sets *handled = true when it ran; *handled = false: the shape is not one it takes, the
// caller runs its own path
int gemm_tc_try(const GemmDesc& d, cudaStream_t st, bool* handled);
// bf16 tensor maps with SWIZZLE_128B (gemm_tc.cu).  map3: dims {d0, d1, d2} (d0 contiguous), byte strides of d1 / d2, box {b0, b1, b2}.
// mapN: rank <= 5; dims / box: `rank` entries (innermost first), strides: rank - 1 byte strides
int tc_make_map3_bf16(void* map, const void* base, int d0, int d1, int d2, size_t stride1, size_t stride2, int b0, int b1, int b2);
int tc_make_mapN_bf16(void* map, const void* base, int rank, const unsigned long long* dims, const unsigned long long* strides, const unsigned* box);
// implicit convolutions on the wgmma GEMM (gemm_tc.cu), for the encoder's conv blocks: *handled = false when the shape is not one they take
int gemm_tc_conv(const float* weight, const float* in, float* out, int NB, int G, int Cout, int Cin, int L, int k, int dil, int pad, int bwd,
                 float beta, cudaStream_t st, bool* handled);
int gemm_tc_conv_dw(const float* dz, const float* x, float* dweight, int NB, int G, int Cout, int Cin, int L, int k, int dil, int pad,
                    cudaStream_t st, bool* handled);
// Precision mode of the library (b200tts_set_precision): 0 = fp32-exact (parity mode), 1 = bf16 tensor-core operands.
int precision_mode();
void set_precision_mode(int mode);
// Dispatch on the precision mode: bf16 mode tries the wgmma path, then runs mma.sync; fp32 mode runs the SIMT kernel.
int gemm_run(const GemmDesc& d, cudaStream_t stream);
int gemm_run_auto(GemmDesc d, float* scratch, size_t scratch_elems, cudaStream_t stream);
// The SIMT kernel whatever the precision mode.
int gemm_f32(const GemmDesc& d, cudaStream_t stream);
int gemm_f32_auto(GemmDesc d, float* scratch, size_t scratch_elems, cudaStream_t stream);

}  // namespace b200tts
