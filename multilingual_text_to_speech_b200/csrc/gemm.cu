// GEMM host layer: the precision mode, the descriptor check, the choice among the wgmma (gemm_tc.cu), mma.sync (gemm_bf16.cu) and
// SIMT kernels, the auto split-K policy and the split-K reduction every path shares.
// The SIMT kernel, for the parity (fp32-exact) mode and for all skinny / odd-shaped contractions, is here as well: register-tiled,
// shared-memory double buffered (register prefetch), optional split-K with a deterministic reduction (no atomics anywhere ->
// bit-reproducible run to run).
#include "common.cuh"

namespace b200tts {

namespace {

constexpr int BK = 16;
constexpr int PAD = 4;

// Load a ROWS x BK tile of an operand into registers.
//   kcontig: element (r, k) at base[r*ld + k]   (row-major along k)
//   else   : element (r, k) at base[k*ld + r]
template <int ROWS, int NT>
__device__ __forceinline__ void tile_load(const float* __restrict__ base, int ld, bool kcontig, bool vec,
                                          int row0, int rows_total, int k0, int k_end, float (&regs)[ROWS * BK / NT]) {
    constexpr int PER = ROWS * BK / NT;
    const int tid = threadIdx.x;
    if (vec) {
#pragma unroll
        for (int j = 0; j < PER / 4; ++j) {
            const int v = tid + j * NT;
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kcontig) {
                const int r = v / (BK / 4), kq = v % (BK / 4);
                if (row0 + r < rows_total && k0 + kq * 4 < k_end)
                    val = *reinterpret_cast<const float4*>(base + (size_t)(row0 + r) * ld + k0 + kq * 4);
            } else {
                const int k = v / (ROWS / 4), r4 = v % (ROWS / 4);
                if (k0 + k < k_end && row0 + r4 * 4 < rows_total)
                    val = *reinterpret_cast<const float4*>(base + (size_t)(k0 + k) * ld + row0 + r4 * 4);
            }
            regs[j * 4 + 0] = val.x; regs[j * 4 + 1] = val.y; regs[j * 4 + 2] = val.z; regs[j * 4 + 3] = val.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const int idx = tid + j * NT;
            float val = 0.f;
            if (kcontig) {
                const int r = idx / BK, k = idx % BK;
                if (row0 + r < rows_total && k0 + k < k_end) val = base[(size_t)(row0 + r) * ld + k0 + k];
            } else {
                const int k = idx / ROWS, r = idx % ROWS;
                if (k0 + k < k_end && row0 + r < rows_total) val = base[(size_t)(k0 + k) * ld + row0 + r];
            }
            regs[j] = val;
        }
    }
}

template <int ROWS, int NT>
__device__ __forceinline__ void tile_store(float (*sm)[ROWS + PAD], bool kcontig, bool vec,
                                           const float (&regs)[ROWS * BK / NT]) {
    constexpr int PER = ROWS * BK / NT;
    const int tid = threadIdx.x;
    if (vec) {
#pragma unroll
        for (int j = 0; j < PER / 4; ++j) {
            const int v = tid + j * NT;
            if (kcontig) {
                const int r = v / (BK / 4), kq = v % (BK / 4);
#pragma unroll
                for (int e = 0; e < 4; ++e) sm[kq * 4 + e][r] = regs[j * 4 + e];
            } else {
                const int k = v / (ROWS / 4), r4 = v % (ROWS / 4);
                *reinterpret_cast<float4*>(&sm[k][r4 * 4]) =
                    make_float4(regs[j * 4 + 0], regs[j * 4 + 1], regs[j * 4 + 2], regs[j * 4 + 3]);
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const int idx = tid + j * NT;
            if (kcontig) sm[idx % BK][idx / BK] = regs[j];
            else sm[idx / ROWS][idx % ROWS] = regs[j];
        }
    }
}

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_f32_kernel(const GemmKernelArgs p) {
    constexpr int NT = (BM / TM) * (BN / TN);
    static_assert(NT == 256, "tile configs are written for 256 threads");
    static_assert(TM % 4 == 0 && TN % 4 == 0, "micro tile must be a multiple of 4");
    __shared__ __align__(16) float As[2][BK][BM + PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + PAD];

    const int z = blockIdx.z;
    const int bz = z / p.splitk, ks = z % p.splitk;
    const float* A = p.A + (size_t)(p.a_batch_mod > 0 ? bz % p.a_batch_mod : bz) * p.strideA;
    const float* B = p.B + (size_t)bz * p.strideB;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int k_begin = ks * p.kchunk;
    const int k_end = min(p.K, k_begin + p.kchunk);

    const int tid = threadIdx.x;
    const int tx = tid % (BN / TN), ty = tid / (BN / TN);

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    float ra[BM * BK / NT], rb[BN * BK / NT];
    const int ntiles = (k_end > k_begin) ? (k_end - k_begin + BK - 1) / BK : 0;
    if (ntiles > 0) {
        tile_load<BM, NT>(A, p.lda, p.a_kcontig, p.a_vec, m0, p.M, k_begin, k_end, ra);
        tile_load<BN, NT>(B, p.ldb, p.b_kcontig, p.b_vec, n0, p.N, k_begin, k_end, rb);
        tile_store<BM, NT>(As[0], p.a_kcontig, p.a_vec, ra);
        tile_store<BN, NT>(Bs[0], p.b_kcontig, p.b_vec, rb);
    }
    __syncthreads();
    for (int t = 0; t < ntiles; ++t) {
        const int cur = t & 1;
        if (t + 1 < ntiles) {
            const int k0 = k_begin + (t + 1) * BK;
            tile_load<BM, NT>(A, p.lda, p.a_kcontig, p.a_vec, m0, p.M, k0, k_end, ra);
            tile_load<BN, NT>(B, p.ldb, p.b_kcontig, p.b_vec, n0, p.N, k0, k_end, rb);
        }
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
            // rows/cols of this thread: chunks of 4, interleaved across the tile for conflict-free LDS.128
#pragma unroll
            for (int c = 0; c < TM / 4; ++c) {
                const float4 v = *reinterpret_cast<const float4*>(&As[cur][k][c * (BM / (TM / 4)) + ty * 4]);
                a[c * 4 + 0] = v.x; a[c * 4 + 1] = v.y; a[c * 4 + 2] = v.z; a[c * 4 + 3] = v.w;
            }
#pragma unroll
            for (int c = 0; c < TN / 4; ++c) {
                const float4 v = *reinterpret_cast<const float4*>(&Bs[cur][k][c * (BN / (TN / 4)) + tx * 4]);
                b[c * 4 + 0] = v.x; b[c * 4 + 1] = v.y; b[c * 4 + 2] = v.z; b[c * 4 + 3] = v.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (t + 1 < ntiles) {
            tile_store<BM, NT>(As[cur ^ 1], p.a_kcontig, p.a_vec, ra);
            tile_store<BN, NT>(Bs[cur ^ 1], p.b_kcontig, p.b_vec, rb);
        }
        __syncthreads();
    }

    // epilogue
    float* out;
    size_t ldo;
    const bool raw = p.splitk > 1;
    if (raw) {
        out = p.partial + ((size_t)ks * p.batch + bz) * (size_t)p.M * p.N;
        ldo = p.N;
    } else {
        out = p.C + (size_t)bz * p.strideC;
        ldo = p.ldc;
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + (i / 4) * (BM / (TM / 4)) + ty * 4 + (i % 4);
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + (j / 4) * (BN / (TN / 4)) + tx * 4 + (j % 4);
            if (n >= p.N) continue;
            float v = acc[i][j];
            if (!raw) {
                v *= p.alpha;
                if (p.bias) v += p.bias[n];
                if (p.beta != 0.f) v += p.beta * out[(size_t)m * ldo + n];
            }
            out[(size_t)m * ldo + n] = v;
        }
    }
}

__global__ void splitk_reduce_kernel(const float* __restrict__ partial, float* __restrict__ C, const float* __restrict__ bias,
                                     int M, int N, int ldc, int batch, int splitk, long long strideC, float alpha,
                                     float beta) {
    const size_t total = (size_t)batch * M * N;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int n = idx % N;
        const int m = (idx / N) % M;
        const int b = idx / ((size_t)M * N);
        float s = 0.f;
        for (int k = 0; k < splitk; ++k) s += partial[(size_t)k * total + idx];
        s *= alpha;
        if (bias) s += bias[n];
        float* c = C + (size_t)b * strideC + (size_t)m * ldc + n;
        if (beta != 0.f) s += beta * *c;
        *c = s;
    }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int launch_gemm_simt(const GemmKernelArgs& p, cudaStream_t stream) {
    dim3 block(256);
    if (p.M > 64 && p.N > 64) {
        dim3 grid(cdiv(p.N, 128), cdiv(p.M, 128), p.batch * p.splitk);
        gemm_f32_kernel<128, 128, 8, 8><<<grid, block, 0, stream>>>(p);
    } else {
        dim3 grid(cdiv(p.N, 64), cdiv(p.M, 64), p.batch * p.splitk);
        gemm_f32_kernel<64, 64, 4, 4><<<grid, block, 0, stream>>>(p);
    }
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

// d on the mma.sync kernel (bf16 operands) or the SIMT kernel, then the split-K reduction unless the consumer keeps the partials
int gemm_mma_or_simt(const GemmDesc& d, bool mma, cudaStream_t stream) {
    if (d.M <= 0 || d.N <= 0 || d.batch <= 0) return B200TTS_OK;
    B200_REQUIRE(d.A && d.B && (d.C || (d.splitk > 1 && d.keep_partials)), "gemm: null operand");
    B200_REQUIRE(d.splitk >= 1 && (d.splitk == 1 || d.partial), "gemm: split-K needs a partial workspace");
    B200_REQUIRE(d.kin == 0, "gemm: two-level K (kin = %d) is taken by the wgmma path only", d.kin);
    GemmKernelArgs p;
    p.A = d.A; p.B = d.B; p.C = d.C; p.bias = d.bias; p.partial = d.partial;
    p.M = d.M; p.N = d.N; p.K = d.K; p.lda = d.lda; p.ldb = d.ldb; p.ldc = d.ldc;
    p.a_kcontig = !d.transA; p.b_kcontig = d.transB;
    p.alpha = d.alpha; p.beta = d.beta; p.batch = d.batch; p.splitk = d.splitk;
    p.strideA = d.strideA; p.strideB = d.strideB; p.strideC = d.strideC; p.a_batch_mod = d.a_batch_mod;
    const int bk = mma ? GEMM_MMA_BK : BK;
    p.kchunk = cdiv(cdiv(d.K > 0 ? d.K : 1, d.splitk), bk) * bk;
    // vector loads need 16B-aligned rows; the contiguous extent must be a multiple of 4 as well
    auto vec_ok = [&](const float* ptr, int ld, long long stride, bool kcontig, int rows) {
        if (!aligned16(ptr) || (ld & 3) || (stride & 3)) return false;
        return kcontig ? ((d.K & 3) == 0) : ((rows & 3) == 0);
    };
    p.a_vec = vec_ok(d.A, d.lda, d.strideA, p.a_kcontig, d.M);
    p.b_vec = vec_ok(d.B, d.ldb, d.strideB, p.b_kcontig, d.N);
    B200_TRY(mma ? launch_gemm_mma(p, stream) : launch_gemm_simt(p, stream));
    if (d.splitk > 1 && !d.keep_partials)
        B200_TRY(splitk_reduce(d.partial, d.C, d.bias, d.M, d.N, d.ldc, d.batch, d.splitk, d.strideC, d.alpha, d.beta, stream));
    return B200TTS_OK;
}

}  // namespace

int splitk_reduce(const float* partial, float* C, const float* bias, int M, int N, int ldc, int batch, int splitk, long long strideC,
                  float alpha, float beta, cudaStream_t stream) {
    const size_t total = (size_t)batch * M * N;
    int blocks = (int)((total + 255) / 256);
    if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
    splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(partial, C, bias, M, N, ldc, batch, splitk, strideC, alpha, beta);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

static int g_precision = 0;
int precision_mode() { return g_precision; }
void set_precision_mode(int mode) { g_precision = mode ? 1 : 0; }

int gemm_f32(const GemmDesc& d, cudaStream_t stream) { return gemm_mma_or_simt(d, false, stream); }

int gemm_run(const GemmDesc& d, cudaStream_t stream) {
    if (g_precision) {      // the wgmma kernel takes the large products; it declines what it cannot take
        bool handled = false;
        B200_TRY(gemm_tc_try(d, stream, &handled));
        if (handled) return B200TTS_OK;
    }
    return gemm_mma_or_simt(d, g_precision != 0, stream);
}

// Picks a split-K factor so that small-output / long-K products still fill the NUM_SMS SMs, bounded by the
// scratch the caller provides for the partial sums.
static int gemm_auto_impl(GemmDesc d, float* scratch, size_t scratch_elems, cudaStream_t stream, bool bf16) {
    if (bf16) {     // long-K products run un-split on the wgmma kernel (no partial round trip); it declines what it cannot take
        d.splitk = 1; d.partial = nullptr; d.keep_partials = 0;
        bool handled = false;
        B200_TRY(gemm_tc_try(d, stream, &handled));
        if (handled) return B200TTS_OK;
    }
    const bool big = bf16 || (d.M > 64 && d.N > 64);
    const long long tiles = (long long)(big ? cdiv(d.M, 128) * cdiv(d.N, 128) : cdiv(d.M, 64) * cdiv(d.N, 64)) * d.batch;
    int s = 1;
    if (tiles < NUM_SMS && scratch) {
        s = (int)((2 * NUM_SMS + tiles - 1) / tiles);
        const int kmax = cdiv(d.K, 128);
        if (s > kmax) s = kmax;
        if (s > 160) s = 160;
        if (s < 1) s = 1;
        while (s > 1 && (size_t)s * d.batch * d.M * d.N > scratch_elems) --s;
    }
    d.splitk = s;
    d.partial = s > 1 ? scratch : nullptr;
    d.keep_partials = 0;
    return gemm_mma_or_simt(d, bf16, stream);
}

int gemm_f32_auto(GemmDesc d, float* scratch, size_t scratch_elems, cudaStream_t stream) {
    return gemm_auto_impl(d, scratch, scratch_elems, stream, false);
}
int gemm_run_auto(GemmDesc d, float* scratch, size_t scratch_elems, cudaStream_t stream) {
    return gemm_auto_impl(d, scratch, scratch_elems, stream, g_precision != 0);
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

int b200tts_gemm_f32(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
                     int ldb, float beta, float* C, int ldc, const float* bias, int batch, long long strideA,
                     long long strideB, long long strideC, int splitk, float* workspace, void* stream) {
    B200_TRY(require_device());
    GemmDesc d;
    d.A = A; d.B = B; d.C = C; d.bias = bias; d.M = M; d.N = N; d.K = K; d.lda = lda; d.ldb = ldb; d.ldc = ldc;
    d.transA = transA; d.transB = transB; d.alpha = alpha; d.beta = beta; d.batch = batch < 1 ? 1 : batch;
    d.strideA = strideA; d.strideB = strideB; d.strideC = strideC; d.splitk = splitk < 1 ? 1 : splitk; d.partial = workspace;
    return gemm_run(d, (cudaStream_t)stream);
}

static_assert(sizeof(b200tts_gemm_desc) == sizeof(GemmDesc), "b200tts_gemm_desc must list the fields of GemmDesc");
int b200tts_debug_gemm(const b200tts_gemm_desc* desc, int route, float* partial, size_t partial_elems, void* stream) {
    B200_REQUIRE(desc, "debug_gemm: null descriptor");
    B200_REQUIRE(route == 0 || route == 1, "debug_gemm: unknown route %d", route);
    B200_TRY(require_device());
    const b200tts_gemm_desc& s = *desc;
    GemmDesc d;
    d.A = s.A; d.B = s.B; d.C = s.C; d.bias = s.bias;
    d.M = s.M; d.N = s.N; d.K = s.K; d.lda = s.lda; d.ldb = s.ldb; d.ldc = s.ldc;
    d.transA = s.transA; d.transB = s.transB; d.alpha = s.alpha; d.beta = s.beta;
    d.batch = s.batch; d.strideA = s.strideA; d.strideB = s.strideB; d.strideC = s.strideC; d.a_batch_mod = s.a_batch_mod;
    d.splitk = s.splitk; d.partial = s.partial; d.keep_partials = s.keep_partials;
    d.A16 = s.A16; d.lda16 = s.lda16; d.B16 = s.B16; d.ldb16 = s.ldb16;
    d.kin = s.kin; d.kosA = s.kosA; d.kosB = s.kosB;
    if (route == 0) return gemm_run(d, (cudaStream_t)stream);
    return gemm_run_auto(d, partial, partial ? partial_elems : 0, (cudaStream_t)stream);
}

}  // extern "C"
