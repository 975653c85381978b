// bf16 tensor-core GEMM (fp32 in / fp32 out, operands rounded to bf16 on the way into shared memory,
// fp32 accumulation) for the perf mode ("bf16 fwd / fp32 master", BASELINE.json configs[1]).
// Same GemmDesc contract as the SIMT kernel (transposes, batch strides, a_batch_mod, split-K); host setup in gemm.cu.
// 128x128x32 CTA tile, 8 warps (2 x 4), each warp 64x32 through mma.sync.m16n8k16 fed by ldmatrix.
#include <cuda_bf16.h>
#include "common.cuh"
#include "tc_ptx.cuh"

namespace b200tts {

namespace {

using namespace tcx;

constexpr int BM = 128, BN = 128, BK = GEMM_MMA_BK, LDS = BK + 8;   // smem row stride in bf16 (80 B: conflict-free ldmatrix)
constexpr int NT = 256;

// Stage a 128 x 32 operand tile: global fp32 -> registers (16 floats / thread).
//   kcontig: element (r, k) at base[r*ld + k]; else at base[k*ld + r].
__device__ __forceinline__ void tile_load(const float* __restrict__ base, int ld, bool kcontig, bool vec, int row0, int rows_total,
                                          int k0, int k_end, float (&regs)[16]) {
    const int tid = threadIdx.x;
    if (vec) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int v = tid + j * NT;                 // 1024 float4 per tile
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kcontig) {
                const int r = v >> 3, kq = v & 7;       // 8 float4 per row of 32 k
                if (row0 + r < rows_total && k0 + kq * 4 < k_end)
                    val = *reinterpret_cast<const float4*>(base + (size_t)(row0 + r) * ld + k0 + kq * 4);
            } else {
                const int k = v >> 5, r4 = v & 31;      // 32 float4 per k row of 128
                if (k0 + k < k_end && row0 + r4 * 4 < rows_total)
                    val = *reinterpret_cast<const float4*>(base + (size_t)(k0 + k) * ld + row0 + r4 * 4);
            }
            regs[j * 4 + 0] = val.x; regs[j * 4 + 1] = val.y; regs[j * 4 + 2] = val.z; regs[j * 4 + 3] = val.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int idx = tid + j * NT;
            float val = 0.f;
            if (kcontig) {
                const int r = idx >> 5, k = idx & 31;
                if (row0 + r < rows_total && k0 + k < k_end) val = base[(size_t)(row0 + r) * ld + k0 + k];
            } else {
                const int k = idx >> 7, r = idx & 127;
                if (k0 + k < k_end && row0 + r < rows_total) val = base[(size_t)(k0 + k) * ld + row0 + r];
            }
            regs[j] = val;
        }
    }
}

// registers -> shared memory tile sm[row][k] (bf16, k contiguous) regardless of the global orientation
__device__ __forceinline__ void tile_store(__nv_bfloat16* sm, bool kcontig, bool vec, const float (&regs)[16]) {
    const int tid = threadIdx.x;
    if (vec) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int v = tid + j * NT;
            if (kcontig) {
                const int r = v >> 3, kq = v & 7;
                uint2 w;
                w.x = pack2(regs[j * 4 + 0], regs[j * 4 + 1]);
                w.y = pack2(regs[j * 4 + 2], regs[j * 4 + 3]);
                *reinterpret_cast<uint2*>(sm + r * LDS + kq * 4) = w;
            } else {
                const int k = v >> 5, r4 = v & 31;
#pragma unroll
                for (int e = 0; e < 4; ++e) sm[(r4 * 4 + e) * LDS + k] = __float2bfloat16_rn(regs[j * 4 + e]);
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int idx = tid + j * NT;
            if (kcontig) sm[(idx >> 5) * LDS + (idx & 31)] = __float2bfloat16_rn(regs[j]);
            else sm[(idx & 127) * LDS + (idx >> 7)] = __float2bfloat16_rn(regs[j]);
        }
    }
}

__global__ void __launch_bounds__(NT) gemm_bf16_kernel(const GemmKernelArgs p) {
    __shared__ __align__(16) __nv_bfloat16 As[2][BM * LDS];
    __shared__ __align__(16) __nv_bfloat16 Bs[2][BN * LDS];
    const int z = blockIdx.z;
    const int bz = z / p.splitk, ks = z % p.splitk;
    const float* A = p.A + (size_t)(p.a_batch_mod > 0 ? bz % p.a_batch_mod : bz) * p.strideA;
    const float* B = p.B + (size_t)bz * p.strideB;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int k_begin = ks * p.kchunk;
    const int k_end = min(p.K, k_begin + p.kchunk);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = (warp >> 2) * 64, wn = (warp & 3) * 32;     // warp tile origin inside the CTA tile

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

    float ra[16], rb[16];
    const int ntiles = (k_end > k_begin) ? (k_end - k_begin + BK - 1) / BK : 0;
    if (ntiles > 0) {
        tile_load(A, p.lda, p.a_kcontig, p.a_vec, m0, p.M, k_begin, k_end, ra);
        tile_load(B, p.ldb, p.b_kcontig, p.b_vec, n0, p.N, k_begin, k_end, rb);
        tile_store(As[0], p.a_kcontig, p.a_vec, ra);
        tile_store(Bs[0], p.b_kcontig, p.b_vec, rb);
    }
    __syncthreads();
    for (int t = 0; t < ntiles; ++t) {
        const int cur = t & 1;
        if (t + 1 < ntiles) {
            const int k0 = k_begin + (t + 1) * BK;
            tile_load(A, p.lda, p.a_kcontig, p.a_vec, m0, p.M, k0, k_end, ra);
            tile_load(B, p.ldb, p.b_kcontig, p.b_vec, n0, p.N, k0, k_end, rb);
        }
#pragma unroll
        for (int kk = 0; kk < BK; kk += 16) {
            uint32_t af[4][4], bf[2][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
                ldmatrix_x4(af[i][0], af[i][1], af[i][2], af[i][3], &As[cur][(wm + i * 16 + (lane & 15)) * LDS + kk + (lane >> 4) * 8]);
#pragma unroll
            for (int j = 0; j < 2; ++j)
                ldmatrix_x4(bf[j][0], bf[j][1], bf[j][2], bf[j][3],
                            &Bs[cur][(wn + j * 16 + (lane & 7) + ((lane >> 4) << 3)) * LDS + kk + ((lane >> 3) & 1) * 8]);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_bf16(acc[i][j], af[i], bf[j >> 1][(j & 1) * 2], bf[j >> 1][(j & 1) * 2 + 1]);
        }
        if (t + 1 < ntiles) {
            tile_store(As[cur ^ 1], p.a_kcontig, p.a_vec, ra);
            tile_store(Bs[cur ^ 1], p.b_kcontig, p.b_vec, rb);
        }
        __syncthreads();
    }

    // epilogue: accumulator element e of tile (i, j): row = g + 8*(e>>1), col = 2*tq + (e&1)
    float* out;
    size_t ldo;
    const bool raw = p.splitk > 1;
    if (raw) { out = p.partial + ((size_t)ks * p.batch + bz) * (size_t)p.M * p.N; ldo = p.N; }
    else { out = p.C + (size_t)bz * p.strideC; ldo = p.ldc; }
    const int g = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = m0 + wm + i * 16 + g + 8 * (e >> 1);
                const int n = n0 + wn + j * 8 + 2 * tq + (e & 1);
                if (m < p.M && n < p.N) {
                    float v = acc[i][j][e];
                    if (!raw) {
                        v *= p.alpha;
                        if (p.bias) v += p.bias[n];
                        if (p.beta != 0.f) v += p.beta * out[(size_t)m * ldo + n];
                    }
                    out[(size_t)m * ldo + n] = v;
                }
            }
}

}  // namespace

int launch_gemm_mma(const GemmKernelArgs& p, cudaStream_t stream) {
    dim3 grid(cdiv(p.N, BN), cdiv(p.M, BM), p.batch * p.splitk);
    gemm_bf16_kernel<<<grid, NT, 0, stream>>>(p);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // namespace b200tts
