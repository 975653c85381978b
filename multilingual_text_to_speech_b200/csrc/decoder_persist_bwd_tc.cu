// Persistent generator-LSTM BACKWARD loop of the bf16 perf mode on TMA + wgmma (sm_90a).
//
// Reverse step i needs  d h_{i-1}[b, n] = sum_r dgates_i[b, r] . W_hh[r, n]  (r over the 4D gate rows): the transpose of the forward
// product.  CTA (gate g, n-block nb, batch half bh) keeps W_hh^T[n-block (64 outputs), gate g (D rows of K)] in shared memory as
// K-major SWIZZLE_128B tiles (A operand, M = 64); per step the bf16 gate gradients [32 utterances x D] of its gate arrive by TMA
// (B operand, N = 32); D / 16 wgmma instructions accumulate in registers; the fp32 partial [gate][b][n] that the next
// step's cell backward sums over the 4 gates (fixed order, no atomics) is stored straight from them.  The launch is cooperative
// with clusters of 2: the CTAs of a pair share (gate, batch half), differ in the n-block, and each issues ONE multicast TMA box of
// half the operand's k-blocks into both CTAs, so every operand byte leaves L2 once per pair.  Per step:
//   P1  cell backward of this CTA's 16 hidden units x 32 utterances (operands prefetched during the previous product)
//   --  grid barrier (gate gradients of all units visible)
//   P2  multicast TMA + wgmma product, registers -> partial store
//   --  grid barrier.
// Warp roles as in decoder_persist_tc.cu: warps 0-7 compute, warps 8-11 = the MMA warpgroup (an elected lane of warp 8 issues the TMA).
// Reference semantics: autograd replay of modules/layers.py:18-47 (train.py:83).
#include <cuda.h>
#include <cuda_bf16.h>
#include "decoder_internal.cuh"
#include "tc_ptx.cuh"

namespace b200tts {

int tc_make_map3_bf16(void* map, const void* base, int d0, int d1, int d2, size_t stride1, size_t stride2, int b0, int b1, int b2);

namespace {

constexpr int NCW = 8;
constexpr int CT = 32 * NCW;
constexpr int PT = CT + 128;            // + the MMA warpgroup
constexpr int UNITS = 16;               // hidden units of the cell backward per CTA
constexpr int ROWS = 64;                // outputs (n) per CTA = MMA M
constexpr int BT = 32;                  // utterances per CTA = MMA N
constexpr int KB = 64;
constexpr int WTILE = ROWS * KB * 2;
constexpr int ATILE = BT * KB * 2;
constexpr int NG = 4;                   // gates = K blocks of the product

struct TcBwdArgs {
    int B, T, D, NNB, NBH;                    // NNB = D / 64 n-blocks
    const float* W; int ldw;                  // fp32 [4D, ldw]: dgates . W
    const float* gates; const float* cstate; const float* dh_static;
    const uint8_t* mask_h; const uint8_t* mask_c;
    int kind, training; float rate_h, rate_c;
    float* dgates;                            // [T, B, 4D] out (fp32)
    __nv_bfloat16* dgb;                       // [T, B, 4D] out: bf16 history of the gate gradients, TMA source of the product
    long long dgb_step; int dgb_rows;         // elements (B * 4D) and TMA rows (B) of one step of the history
    float* part;                              // [NG, B, D] partial products of the previous reverse step
    unsigned* barrier; int* abort_flag;
    long long* prof;
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers (mbarrier, TMA, fences and the cluster barrier: tc_ptx.cuh)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void l2_prefetch(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// tanh of the recomputed cell state in the reverse loops: the same ex2-based form the forward loops of the bf16 mode use (~1e-6 relative)
__device__ __forceinline__ float tanh_exp(float x) { return 2.f * __fdividef(1.f, 1.f + __expf(-2.f * x)) - 1.f; }
// named barrier among the compute warps only
__device__ __forceinline__ void csync() { asm volatile("bar.sync 1, %0;" ::"n"(CT) : "memory"); }

__device__ __forceinline__ bool grid_barrier(unsigned* counter, unsigned& target, unsigned nblocks, int* abort_flag, int* s_ok) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += nblocks;
        tcx::proxy_fence_global();          // the bf16 gate gradients written above are read by other CTAs through TMA (async proxy)
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
        int ok = 1;
        const long long t0 = clock64();
        unsigned polls = 0;
        for (;;) {
            unsigned v;
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            if (v >= target) break;
            if ((++polls & 255u) == 0 && (clock64() - t0 > 4000000000ll || *reinterpret_cast<volatile int*>(abort_flag))) {
                ok = 0; *abort_flag = 1; break;
            }
        }
        asm volatile("fence.acquire.gpu;" ::: "memory");
        *s_ok = ok;
    }
    __syncthreads();
    return *s_ok != 0;
}

__global__ void __launch_bounds__(PT, 1) lstm_bwd_loop_tc_kernel(const __grid_constant__ CUtensorMap tmG, const TcBwdArgs p) {
    extern __shared__ __align__(1024) unsigned char smem_raw0[];
    unsigned char* smem_raw = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw0) + 1023) & ~(uintptr_t)1023);
    __shared__ uint64_t full_bar;
    __shared__ int s_ok;

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int cta = blockIdx.x;
    // the CTA pair (2k, 2k+1) = one cluster shares (gate, batch half) and takes two n-blocks: both need the same operand every step
    const int gsel = (cta >> 1) % NG, nb = 2 * ((cta >> 3) % (p.NNB / 2)) + (cta & 1), bh = cta / (NG * p.NNB);
    const int B = p.B, D = p.D, NNB = p.NNB;
    const int b0 = bh * BT, n0 = nb * ROWS;
    const int u0 = (gsel * NNB + nb) * UNITS;                 // hidden units whose cell backward this CTA owns
    // batch halves are independent (cell backward and product of a CTA serve the same 32 utterances): one barrier counter per half
    // (the cost of a barrier is its latency chain -- store acks, atomic round trip, poll -- not the number of arrivals, so one grid-wide
    // counter is used)
    const unsigned nblocks = gridDim.x;
    unsigned* const bar_counter = p.barrier;
    const bool compute = warp < NCW, is_mma = warp >= NCW;

    unsigned char* sW = smem_raw;                              // [NNB][64 rows (n)][128 B] swizzled: W^T[n0 + r, gate gsel, k]
    unsigned char* ring = smem_raw + (size_t)NNB * WTILE;      // [NNB][32 rows (b)][128 B] swizzled (one TMA box)

    // ---- one-time: resident transposed weight block, fp32 -> bf16, canonical K-major SWIZZLE_128B layout (n fastest: coalesced reads) ----
    for (int idx = tid; idx < ROWS * D; idx += PT) {
        const int k = idx / ROWS, r = idx % ROWS;
        const float w = (n0 + r < D) ? p.W[(size_t)(gsel * D + k) * p.ldw + n0 + r] : 0.f;
        const int kb = k / KB, kc = k % KB, chunk = kc >> 3, e = kc & 7;
        *reinterpret_cast<__nv_bfloat16*>(sW + (size_t)kb * WTILE + r * 128 + ((chunk ^ (r & 7)) << 4) + e * 2) = __float2bfloat16_rn(w);
    }
    if (tid == 0) {
        tcx::mbar_init(&full_bar, 1);
        tcx::mbar_init_fence();
    }
    tcx::proxy_fence_shared();              // the weight tiles were written through the generic proxy; wgmma reads them through the async proxy
    __syncthreads();
    tcx::cluster_arrive(); tcx::cluster_wait();     // one-time: the peer's mbarrier is initialised before this CTA's first multicast targets it

    const float inv_h = 1.f / (1.f - p.rate_h), inv_c = 1.f / (1.f - p.rate_c);
    // cell-backward operands of this thread's two (b, u) pairs, fetched one step ahead (during the previous product)
    float gi_[2], gf_[2], gg_[2], go_[2], cp_[2], dhs_[2];
    uint8_t mh_[2], mc_[2];
    float dc_reg[2] = {0.f, 0.f}, dhz_reg[2] = {0.f, 0.f};
    auto prefetch = [&](int step) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int idx = tid + e * CT;
            const int bl = idx / UNITS, uu = idx % UNITS, b = b0 + bl, u = u0 + uu;
            gi_[e] = gf_[e] = gg_[e] = go_[e] = cp_[e] = dhs_[e] = 0.f; mh_[e] = 1; mc_[e] = 1;
            if (b < B && u < D) {
                const size_t g0 = ((size_t)step * B + b) * 4 * D + u, mi = ((size_t)step * B + b) * D + u;
                gi_[e] = p.gates[g0]; gf_[e] = p.gates[g0 + D]; gg_[e] = p.gates[g0 + 2 * D]; go_[e] = p.gates[g0 + 3 * D];
                cp_[e] = p.cstate[mi];
                dhs_[e] = p.dh_static[mi];
                if (p.training && p.mask_h) mh_[e] = p.mask_h[mi];
                if (p.training && p.mask_c) mc_[e] = p.mask_c[mi];
            }
        }
    };
    auto prefetch_l2 = [&](int step) {
        if (step < 0) return;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int idx = tid + e * CT;
            const int bl = idx / UNITS, uu = idx % UNITS, b = b0 + bl, u = u0 + uu;
            if (b < B && u < D && (uu & 7) == 0) {
                const size_t g0 = ((size_t)step * B + b) * 4 * D + u, mi = ((size_t)step * B + b) * D + u;
                l2_prefetch(p.gates + g0); l2_prefetch(p.gates + g0 + D); l2_prefetch(p.gates + g0 + 2 * D); l2_prefetch(p.gates + g0 + 3 * D);
                l2_prefetch(p.cstate + mi); l2_prefetch(p.dh_static + mi);
                if (uu == 0 && p.training && p.mask_h) l2_prefetch(p.mask_h + mi);
                if (uu == 0 && p.training && p.mask_c) l2_prefetch(p.mask_c + mi);
            }
        }
    };
    if (compute) { prefetch(p.T - 1); prefetch_l2(p.T - 2); }

    unsigned target = 0;
    uint32_t it = 0;                         // products done (mbarrier phase)
    long long prof_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long prof_t = clock64();
#define PROF_MARK(slot)                                                      \
    do {                                                                     \
        if (p.prof && tid == 0) { const long long now = clock64(); prof_acc[slot] += now - prof_t; prof_t = now; } \
    } while (0)

    for (int i = p.T - 1; i >= 0; --i) {
        const bool last = (i == p.T - 1);
        // ---------------- P1: LSTM cell backward (2 (b, u) pairs per compute thread) ----------------
        if (compute) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int idx = tid + e * CT;
                const int bl = idx / UNITS, uu = idx % UNITS, b = b0 + bl, u = u0 + uu;
                if (b < B && u < D) {
                    const size_t g0 = ((size_t)i * B + b) * 4 * D + u;
                    float dh = dhs_[e];
                    float dc_in = 0.f;
                    if (!last) {
                        float r4[NG];
#pragma unroll
                        for (int k2 = 0; k2 < NG; ++k2) r4[k2] = __ldcg(p.part + ((size_t)k2 * B + b) * D + u);
                        dh += ((r4[0] + r4[1]) + (r4[2] + r4[3])) + dhz_reg[e];
                        dc_in = dc_reg[e];
                    }
                    const float gi = gi_[e], gf = gf_[e], gg = gg_[e], go = go_[e], cp = cp_[e];
                    const float tc = tanh_exp(gf * cp + gi * gg);
                    float dhn, dcn, dc_prev_direct = 0.f, dh_prev_direct = 0.f;
                    if (p.kind == B200TTS_CELL_ZONEOUT) {
                        float kh, kc;
                        if (p.training) {
                            kh = (1.f - p.rate_h) * (p.mask_h ? (float)mh_[e] * inv_h : 1.f);
                            kc = (1.f - p.rate_c) * (p.mask_c ? (float)mc_[e] * inv_c : 1.f);
                        } else { kh = 1.f - p.rate_h; kc = 1.f - p.rate_c; }
                        dhn = dh * kh; dh_prev_direct = dh - dhn;
                        dcn = dc_in * kc + dhn * go * (1.f - tc * tc);
                        dc_prev_direct = dc_in - dc_in * kc;
                    } else {
                        dhn = (p.training && p.mask_h) ? dh * (float)mh_[e] * inv_h : dh;
                        dcn = dc_in + dhn * go * (1.f - tc * tc);
                    }
                    const float di = dcn * gg * gi * (1.f - gi), df = dcn * cp * gf * (1.f - gf);
                    const float dg = dcn * gi * (1.f - gg * gg), dO = dhn * tc * go * (1.f - go);
                    p.dgates[g0] = di; p.dgates[g0 + D] = df; p.dgates[g0 + 2 * D] = dg; p.dgates[g0 + 3 * D] = dO;
                    __nv_bfloat16* db = p.dgb + (size_t)i * p.dgb_step + (size_t)b * 4 * D + u;
                    db[0] = __float2bfloat16_rn(di); db[D] = __float2bfloat16_rn(df);
                    db[2 * D] = __float2bfloat16_rn(dg); db[3 * D] = __float2bfloat16_rn(dO);
                    dc_reg[e] = dcn * gf + dc_prev_direct;
                    dhz_reg[e] = dh_prev_direct;
                }
            }
        }
        PROF_MARK(0);
        if (!grid_barrier(bar_counter, target, nblocks, p.abort_flag, &s_ok)) break;
        PROF_MARK(1);
        if (i == 0) break;

        // ---------------- P2: partial[gate] = dgates[:, gate block] . W[gate block, n-block]  (TMA + wgmma) ----------------
        // the operand is fetched once per CTA pair: rank r issues k-blocks [r NNB/2, (r+1) NNB/2) of the gate's D columns with multicast
        // into both rings, and each CTA arms its barrier with the whole NNB tiles.  The peer may write into this ring now: both CTAs'
        // previous products completed before they arrived at the grid barriers in between.
        if (is_mma) {
            if (warp == NCW) {
                tcx::proxy_fence_global();
                if (tcx::elect_one()) {
                    const int r = cta & 1;
                    tcx::mbar_expect_tx(&full_bar, (uint32_t)NNB * ATILE);
                    tcx::tma_load_3d_mc(ring + (size_t)r * (NNB / 2) * ATILE, &tmG, &full_bar, 0x3, 0, i * p.dgb_rows + b0, gsel * NNB + r * (NNB / 2));
                }
                __syncwarp();
            }
            tcx::mbar_wait(&full_bar, it & 1);
            float acc[16];                   // the first instruction overwrites (scale-d = 0)
            tcx::wgmma_fence();
            for (int c = 0; c < NNB; ++c) {
                const uint64_t adesc = tcx::make_sw128_desc(tcx::smem_u32(sW + (size_t)c * WTILE));
                const uint64_t bdesc = tcx::make_sw128_desc(tcx::smem_u32(ring + (size_t)c * ATILE));
#pragma unroll
                for (int k = 0; k < KB / 16; ++k) tcx::wgmma_m64n32<0, 0>(acc, adesc + 2 * k, bdesc + 2 * k, (c | k) != 0);
            }
            tcx::wgmma_commit();
            tcx::wgmma_wait<0>();
            tcx::wgmma_fence_acc(acc);
            // accumulator row = output n0 + row, column = utterance b0 + column (fragment layout: tc_ptx.cuh)
            const int row = 16 * (warp - NCW) + (lane >> 2), n = n0 + row;
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const int b = b0 + 8 * (r >> 2) + 2 * (lane & 3) + (r & 1), nn = n + 8 * ((r >> 1) & 1);
                if (b < B && nn < D) p.part[((size_t)gsel * B + b) * D + nn] = acc[r];
            }
        }
        if (compute) {
            prefetch(i - 1);                 // operands of the next cell backward: their latency hides behind the product
            prefetch_l2(i - 2);
            PROF_MARK(2);
        }
        ++it;
        PROF_MARK(3);
        if (!grid_barrier(bar_counter, target, nblocks, p.abort_flag, &s_ok)) break;
        PROF_MARK(4);
    }
    if (p.prof && tid == 0)
        for (int k = 0; k < 8; ++k) p.prof[(size_t)cta * 8 + k] = prof_acc[k];
#undef PROF_MARK
    // no CTA exits while a multicast it issued may still be landing in its peer.  A watchdog abort leaves the loop through the shared abort
    // flag, which every CTA checks at each grid barrier, so both ranks of a pair stop at the same barrier -- unless the flag is raised just
    // as that barrier completes: the rank that went on then waits for the peer's half of the next operand and ends in the trap of
    // mbar_wait (~2 s), not in a hang
    tcx::cluster_arrive(); tcx::cluster_wait();
}

size_t bwd_tc_smem_bytes(int D) { return 1024 + (size_t)(D / KB) * (WTILE + ATILE); }
size_t part_bytes(const b200tts_decoder_shape& s) { return ((size_t)NG * s.B * s.D * 4 + 255) / 256 * 256; }

}  // namespace

bool tc_persist_gen_bwd_supported(const b200tts_decoder_shape& s) {
    if (s.D % 128 != 0 || s.D > 2048 || s.B > 64) return false;                      // the shapes this loop is validated on
    if (s.D % KB != 0 || s.D % (NG * (s.D / KB) * UNITS) != 0) return false;       // 4 x D/64 CTAs per batch half x 16 units = D
    if ((s.D / KB) % 2 != 0) return false;                                          // the n-blocks pair up (one operand half per rank)
    const int NBH = (s.B + BT - 1) / BT;
    if (NG * (s.D / KB) * NBH > NUM_SMS) return false;
    return bwd_tc_smem_bytes(s.D) <= 227 * 1024 - 1088;
}

size_t persist_bwd_gen_extra_bytes(const b200tts_decoder_shape& s) { return part_bytes(s) + 256 + NUM_SMS * 8 * 8; }

// dgates for all T steps of the generator LSTM, and their bf16 [T, B, 4D] history `dgb_hist`; `extra` = persist_bwd_gen_extra_bytes
// scratch: the partial buffer [NG, B, D], then barrier + profile counters.
int tc_persist_gen_bwd_loop(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                            const DecoderLayout& fl, const float* fws, const float* dh_static, float* dgates, unsigned char* extra,
                            cudaStream_t st, void* dgb_hist) {
    const int B = s.B, D = s.D;
    TcBwdArgs a{};
    a.B = B; a.T = s.T; a.D = D; a.NNB = D / KB; a.NBH = (B + BT - 1) / BT;
    a.W = w.gen_w_hh; a.ldw = D;
    a.gates = fws + fl.gg; a.cstate = fws + fl.cg; a.dh_static = dh_static;
    a.mask_h = in.mask_gen_h; a.mask_c = in.mask_gen_c; a.kind = s.cell_kind; a.training = s.training; a.rate_h = s.rate_h; a.rate_c = s.rate_c;
    a.dgates = dgates;
    a.dgb = static_cast<__nv_bfloat16*>(dgb_hist); a.dgb_step = (long long)B * 4 * D; a.dgb_rows = B;
    a.part = reinterpret_cast<float*>(extra);
    a.barrier = reinterpret_cast<unsigned*>(extra + part_bytes(s));
    a.abort_flag = reinterpret_cast<int*>(a.barrier + 32);
    a.prof = reinterpret_cast<long long*>(extra + part_bytes(s) + 256);
    B200_CUDA(cudaMemsetAsync(a.barrier, 0, 256, st));
    // {64 columns, T * B rows, 4D/64 k-blocks}: k-block stride 128 B, row stride 4D * 2 B; a box is half of one gate (NNB/2 k-blocks)
    CUtensorMap tm;
    B200_TRY(tc_make_map3_bf16(&tm, a.dgb, KB, s.T * B, 4 * D / KB, (size_t)4 * D * 2, 128, KB, BT, a.NNB / 2));
    const size_t smem = bwd_tc_smem_bytes(D);
    void* fn = (void*)lstm_bwd_loop_tc_kernel;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = NG * a.NNB * a.NBH;
    void* params[] = {&tm, &a};
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(PT); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeCooperative;
    attrs[0].val.cooperative = 1;
    attrs[1].id = cudaLaunchAttributeClusterDimension;          // CTA pairs share the per-step operand (multicast TMA)
    attrs[1].val.clusterDim.x = 2; attrs[1].val.clusterDim.y = 1; attrs[1].val.clusterDim.z = 1;
    cfg.attrs = attrs; cfg.numAttrs = 2;
    int nclusters = 0;
    B200_CUDA(cudaOccupancyMaxActiveClusters(&nclusters, fn, &cfg));
    B200_REQUIRE(nclusters * 2 >= grid, "wgmma persistent backward: only %d CTA pairs can be co-resident, %d needed", nclusters, grid / 2);
    KernelTimer kt("lstm_bwd_loop_tc_kernel", st);
    B200_CUDA(cudaLaunchKernelExC(&cfg, fn, params));
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // namespace b200tts
