// Persistent attention-LSTM + attention reverse loop of the bf16 perf mode (TMA + wgmma + CTA pairs), and its parallel post pass.
//
// Reverse step i needs  [d ctx | d h_att]_{i-1} = dgates_i . [W_ih[:, P:] | W_hh]  (K = 4D gate rows -> M + D output columns), the
// transpose of the forward product.  CTA (kb, nb) of 8 x 16 keeps W^T[n-block of 80 outputs (96 for memory dim 512), K-slice kb of
// 4 x D/8 gate rows] in shared memory as K-major SWIZZLE_128B tiles (wgmma B operand) for the whole sequence.  Per step:
//   PA  attention backward of one utterance per CTA pair (cluster of 2): d weights, softmax backward, energies backward and d cum on
//       the tensor cores (mma.sync), the two ranks exchanging partials through distributed shared memory;
//   --  grid barrier
//   PB  LSTM-cell backward of 8 hidden units x every utterance (CTAs < D/8): gate gradients -> fp32 for the weight-gradient products
//       and a bf16 [T, B, 4D] history;
//   --  grid barrier (gate gradients of all units visible)
//   P2  the bf16 gate gradients of the K-slice for the whole batch (<= 64 utterances, rows beyond B zero-filled), the A operand
//       (M = 64), arrive as two 5-D TMA boxes of two gates each: the CTAs of a pair share the K-slice (and differ in the n-block), and
//       each issues one box with multicast into both; warpgroup 0 runs wgmma m64n80k16 / m64n96k16 and stores the fp32 partial
//       [B x n-block] that the next step sums over the 8 K-slices (fixed order, no atomics);
//   --  grid barrier.
// The post pass then accumulates, in parallel over all steps, what the recurrence does not need: d memT, d Wcomb, d v.
// Reference semantics: autograd replay of modules/layers.py:18-47 and modules/attention.py:39-86 (train.py:83).
#include <cuda_bf16.h>
#include "decoder_internal.cuh"
#include "tc_ptx.cuh"

namespace b200tts {

namespace {

constexpr int PT = 256;

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    const uint32_t addr = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
struct NoOverlap { __device__ __forceinline__ void operator()() const {} };
// `overlap` runs on every thread BETWEEN the CTA's arrival and its wait: work that does not depend on other CTAs (next step's operand
// prefetch) hides under the barrier latency instead of delaying the arrival
template <typename Overlap = NoOverlap>
__device__ __forceinline__ bool grid_barrier(unsigned* counter, unsigned& target, unsigned nblocks, int* abort_flag, bool async_fence = false,
                                             Overlap overlap = Overlap()) {
    __shared__ int s_ok;
    __syncthreads();
    if (threadIdx.x == 0) {
        target += nblocks;
        if (async_fence) tcx::proxy_fence_global();     // global data written above is read by other CTAs through TMA (async proxy)
        // arrival = ONE release-reduction (cumulative over the CTA's writes, which the __syncthreads above made visible to thread 0);
        // the wait polls with relaxed loads and issues a single acquire fence after the last one
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
    }
    overlap();
    if (threadIdx.x == 0) {
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
        s_ok = ok;
    }
    __syncthreads();
    return s_ok != 0;
}

__device__ __forceinline__ void l2_prefetch(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// asynchronous global -> shared copies: 16 bytes bypassing L1 (.cg; also right for data other CTAs wrote during the launch), and 8 bytes.
// The thread that issued them waits with cp_async_wait_all; a CTA barrier after that wait makes them visible to the other threads
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// remote store that completes its 4 bytes on the PEER's mbarrier (data + signal in one instruction): the pair exchanges need no cluster
// barrier and none of the memory fence its release semantics imply
__device__ __forceinline__ void st_async_peer_f32(const float* local_smem, const uint64_t* local_bar, uint32_t peer_rank, float v) {
    uint32_t ra, rb;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"((uint32_t)__cvta_generic_to_shared(local_smem)), "r"(peer_rank));
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"((uint32_t)__cvta_generic_to_shared(local_bar)), "r"(peer_rank));
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(ra), "r"(__float_as_uint(v)), "r"(rb) : "memory");
}
// tanh of the recomputed cell state in the reverse loops: the same ex2-based form the forward loops of the bf16 mode use (~1e-6 relative)
__device__ __forceinline__ float tanh_exp(float x) { return 2.f * __fdividef(1.f, 1.f + __expf(-2.f * x)) - 1.f; }

#define BPROF_DECL long long prof_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}; long long prof_t = clock64();
#define BPROF_MARK(slot)                                                                                         \
    do {                                                                                                         \
        if (p.prof && threadIdx.x == 0) { const long long now = clock64(); prof_acc[slot] += now - prof_t; prof_t = now; } \
    } while (0)
#define BPROF_FLUSH                                                                                              \
    do {                                                                                                         \
        if (p.prof && threadIdx.x == 0)                                                                          \
            for (int k9 = 0; k9 < 8; ++k9) p.prof[(size_t)blockIdx.x * 8 + k9] = prof_acc[k9];                   \
    } while (0)

// =================================================================================================
// Attention-LSTM + attention reverse loop
// =================================================================================================
constexpr int KBA = 8;            // K-slices of the product (over hidden units)
constexpr int GLD = 33;           // row stride of the G tile buffer (floats)
constexpr int NBT = 16;           // n-blocks of the product  -> 8 x 16 = 128 CTAs (64 pairs): one per SM of the 132
constexpr int TUN = 80;           // outputs per n-block (wgmma N); TUN_WIDE when M + D > NBT * TUN (memory dim 512)
constexpr int TUN_WIDE = 96;

struct AttBwdArgs {
    int B, T, D, M, L, A, KC, NOUT, UK, UN, MT;           // NOUT = M + D, UK = D / KBA, MT = ceil(L / 16)
    const float* W; int ldw;                              // wcat_att fp32 [4D, M + D]
    const float* gates; const float* cstate;              // forward saves
    const float* dh_static;                               // [T, B, D]   (from the generator input projection)
    const float* dctx_static;                             // [T, B, M]
    const uint8_t* mask_h; const uint8_t* mask_c;
    int kind, training; float rate_h, rate_c;
    float* dgates;                                        // [T, B, 4D] out (fp32)
    __nv_bfloat16* dgb;                                   // [T, B, 4D] out: bf16 history of the gate gradients, TMA source of the product
    long long dgb_step; int dgb_rows;                     // elements (B * 4D) and TMA rows (B) of one step of the history
    float* part;                                          // [KBA, B, NOUT] partial products of the previous reverse step
    // attention
    const float* q; const float* cum; const float* align; long long align_bstride;
    const float* dalign; long long dalign_bstride;        // may be null
    const float* bias; const float* v; const float* Wq;   // [A], [A], [A, D]
    const __nv_bfloat16* WcB;                             // [A][40]   Wcomb[a][k], k contiguous (k >= KC zero)
    const __nv_bfloat16* WcB2;                            // [32][A+8] Wcomb^T[k][a], a contiguous
    const __nv_bfloat16* memTf;                           // [B][MT][32 lanes][64] fragment-major memory projection
    const uint4* memFb; int M16;                          // [B][MT][M16][32] A fragments (rows = positions, k = memory dims), bf16
    const int* lengths;
    float* dctx_tot;                                      // [T, B, M] out
    float* dq;                                            // [T, B, A] out
    float* de;                                            // [T, B, L] out (softmax-backward energies, consumed by the post pass)
    unsigned* barrier; int* abort_flag;
    long long* prof;
};

__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float tanh_fast(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// UNC: outputs per n-block of the product (wgmma N), compile-time: 80, or 96 for memory dim 512
template <int UNC>
__global__ void __launch_bounds__(PT, 1) att_bwd_loop_kernel(const __grid_constant__ CUtensorMap tmG, const AttBwdArgs p) {
    extern __shared__ __align__(1024) unsigned char smem_raw0[];
    unsigned char* smem_raw = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw0) + 1023) & ~(uintptr_t)1023);
    __shared__ uint64_t full_bar[2], xb1, xb2;   // full_bar[r]: rank r's half of the P2 operand; xb1 / xb2: arrival of the peer's softmax dot /
                                                 // query-gradient partial + G halo tile
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x;
    // the CTA pair (2k, 2k+1) = one cluster shares the K-slice kb and takes two n-blocks: both need the same operand in P2
    const int kb = (cta >> 1) % KBA, nb = 2 * (cta >> 4) + (cta & 1);
    const int B = p.B, D = p.D, UK = p.UK, UN = p.UN, KROWS = 4 * UK, M = p.M, L = p.L, A = p.A;
    const int n0 = nb * UN;
    const int NKT = KROWS / 64;                                                      // k-block tiles of the K-slice
    // sW [NKT][UN rows][128 B] swizzled, slot As [NKT][64 rows][128 B] (one TMA box).  The slot doubles as the attention scratch and
    // the query-gradient staging.
    unsigned char* sW = smem_raw;
    __nv_bfloat16* As = reinterpret_cast<__nv_bfloat16*>(smem_raw + (size_t)NKT * UN * 128);
    unsigned char* extra = reinterpret_cast<unsigned char*>(As) + (size_t)NKT * 8192;
    __nv_bfloat16* sWcB = reinterpret_cast<__nv_bfloat16*>(extra);                   // [A][40]
    __nv_bfloat16* sWcB2 = sWcB + (size_t)A * 40;                                    // [32][A+8]
    float* dcum = reinterpret_cast<float*>(sWcB2 + (size_t)32 * (A + 8));            // [L16 + 32] persistent d cum
    uint4* wqf = reinterpret_cast<uint4*>(dcum + (p.MT * 16 + 32));                  // [A / 16][32 lanes] Wq B fragments of this CTA's 8 units
    float* s_dhq = reinterpret_cast<float*>(wqf + (size_t)(A / 16) * 32);            // [2 halves of A][64][8] query part of d h
    // cell-backward staging (owner CTAs), [..][B][8 units] each, outside the TMA slot: the operands of the next step are in flight while
    // P2's TMA refills the slot
    float* s_pbo = s_dhq + 2 * 64 * 8;                                               // [6][B][8] gates i, f, g, o, c, d h static
    uint8_t* s_pbm = reinterpret_cast<uint8_t*>(s_pbo + (size_t)6 * B * 8);          // [2][B][8] zoneout / dropout keep bytes h, c
    float* s_rp = reinterpret_cast<float*>(s_pbm + (size_t)2 * B * 8);               // [KBA][B][8] recurrent partial sums
    const unsigned nblocks = gridDim.x;
    const int L16 = p.MT * 16;

    for (int idx = tid; idx < KROWS * UN; idx += PT) {
        const int r = idx / UN, n = idx % UN;
        const int g = r / UK, uk = r % UK;
        float w = 0.f;
        if (n0 + n < p.NOUT) w = p.W[(size_t)(g * D + kb * UK + uk) * p.ldw + n0 + n];
        // W^T[n][k] of k-block tile c = r / 64 (same order as the TMA box: gate-major, then 64-row halves), SWIZZLE_128B
        const int c = r >> 6, kc = r & 63;
        *reinterpret_cast<__nv_bfloat16*>(sW + (size_t)c * UN * 128 + n * 128 + ((((kc >> 3) ^ (n & 7))) << 4) + (kc & 7) * 2) = __float2bfloat16_rn(w);
    }
    for (int idx = tid; idx < A * 40; idx += PT) sWcB[idx] = p.WcB[idx];
    for (int idx = tid; idx < 32 * (A + 8); idx += PT) sWcB2[idx] = p.WcB2[idx];
    for (int idx = tid; idx < L16 + 32; idx += PT) dcum[idx] = 0.f;
    // cell-backward ownership: CTA c < D/8 owns hidden units [8c, 8c+8) for every utterance
    const int UOWN = 8;
    const bool owner = cta * UOWN < D;
    const int uo0 = cta * UOWN;
    // B fragments (bf16 hi / lo split) of Wq[:, 8 owned units] for the query term of the cell backward: constant over the loop, built once.
    // Entry (k-step kk, lane): {hi, hi, lo, lo} of rows a = 16 kk + 2 (lane % 4) (+1) (+8), column lane / 4
    if (owner)
        for (int idx = tid; idx < (A / 16) * 32; idx += PT) {
            const int kk = idx >> 5, g = (idx >> 2) & 7, tq = idx & 3;
            uint32_t f[4];
#pragma unroll
            for (int r2 = 0; r2 < 2; ++r2) {
                const int a = kk * 16 + 2 * tq + 8 * r2;
                const float x0 = p.Wq[(size_t)a * D + uo0 + g], x1 = p.Wq[(size_t)(a + 1) * D + uo0 + g];
                const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
                __nv_bfloat162 hp; hp.x = h0; hp.y = h1;
                f[r2] = *reinterpret_cast<uint32_t*>(&hp);
                f[2 + r2] = pack2(x0 - __bfloat162float(h0), x1 - __bfloat162float(h1));
            }
            wqf[idx] = make_uint4(f[0], f[1], f[2], f[3]);
        }
    uint32_t prod_it = 0;
    if (tid == 0) { tcx::mbar_init(&xb1, 1); tcx::mbar_init(&xb2, 1); tcx::mbar_init_fence(); }
    if (tid == 0) { tcx::mbar_init(&full_bar[0], 1); tcx::mbar_init(&full_bar[1], 1); tcx::mbar_init_fence(); }
    tcx::proxy_fence_shared();           // the weight tiles were written through the generic proxy; wgmma reads them through the async proxy
    __syncthreads();
    // one-time: the peer's mbarriers are initialised before the first remote st.async or multicast TMA of this CTA targets them
    tcx::cluster_arrive(); tcx::cluster_wait();

    const float inv_h = 1.f / (1.f - p.rate_h), inv_c = 1.f / (1.f - p.rate_c);
    constexpr int MAXE = 3;               // (b, u) pairs per thread: B * 8 / 256 <= 3 for B <= 64... (B <= 96)
    float dc_reg[MAXE], dhz_reg[MAXE];
#pragma unroll
    for (int e = 0; e < MAXE; ++e) { dc_reg[e] = 0.f; dhz_reg[e] = 0.f; }
    unsigned target = 0;

    // attention scratch (aliases As): floats
    float* scr = reinterpret_cast<float*>(As);
    float* s_dctx = scr;                                  // [M (+3)]
    float* s_w = s_dctx + ((M + 3) & ~3);                 // [L16]
    float* s_de = s_w + L16;                              // [L16]
    float* s_qb = s_de + L16;                             // [A]
    float* s_vv = s_qb + A;                               // [A]
    uint32_t* s_Ph = reinterpret_cast<uint32_t*>(s_vv + A);   // [L16 + 48]
    uint32_t* s_Pl = s_Ph + (L16 + 48);
    float* s_red = reinterpret_cast<float*>(s_Pl + (L16 + 48));   // [64]
    // attention backward runs on CTA PAIRS (cluster of 2): rank hf = cta & 1 owns the position tiles [t_lo, t_hi) of utterance cta >> 1
    const int hf = cta & 1, HT0 = (p.MT + 1) / 2;
    const int t_lo = hf ? HT0 : 0, t_hi = hf ? p.MT : HT0;
    const int g_lo = hf ? (HT0 - 1) * 16 : 0;             // first G row held locally: the own tiles plus ONE halo tile of the peer
    float* s_G = s_red + 64;                              // [(HT0 + 1) * 16][GLD], row l stored at l - g_lo
    float* s_dqp = s_G + (size_t)(HT0 + 1) * 16 * GLD;    // [8][A] per-warp query-gradient partials
    float* s_dqx = s_dqp + 8 * A;                         // [A]  the peer's partial (written through distributed shared memory)
    float* s_dotx = s_dqx + A;                            // [4]  the peer's partial softmax dot
    float* s_stage = s_dotx + 4;                          // [L16] d cum staging
    uint2* s_bf = reinterpret_cast<uint2*>(s_stage + L16); // [M16][32] B fragments (hi / lo split of d ctx) of the dw product, shared by all warps
    BPROF_DECL

    const int pc = cta >> 1;
    // cell-backward operands of the owned units x every utterance: copied into s_pbo / s_pbm a whole reverse step ahead, under the grid
    // barrier that ends the previous cell phase, so that neither their DRAM latency nor registers to hold them sit on the loop.  Each
    // (utterance, operand) is one 32-byte run of 8 floats (uo0 = 8 cta) and 8 mask bytes; the keep masks are read only when training with
    // masks, so only then copied
    auto pb_stage = [&](int step) {
        if (!owner || step < 0) return;
        const size_t row = (size_t)step * B;
        for (int c = tid; c < 12 * B; c += PT) {
            const int k = c / (2 * B), r = c - k * 2 * B, b = r >> 1, h4 = (r & 1) * 4;
            const float* src = k < 4 ? p.gates + (row + b) * 4 * D + (size_t)k * D : (k == 4 ? p.cstate : p.dh_static) + (row + b) * D;
            cp_async16(s_pbo + (k * B + b) * UOWN + h4, src + uo0 + h4);
        }
        if (p.training)
            for (int c = tid; c < 2 * B; c += PT) {
                const int k = c / B, b = c - k * B;
                const uint8_t* m = k ? p.mask_c : p.mask_h;
                if (m) cp_async8(s_pbm + (k * B + b) * UOWN, m + (row + b) * D + uo0);
            }
    };
    pb_stage(p.T - 1);
    int pa_len = 0;
    if (pc < B) { const int l0 = p.lengths[pc]; pa_len = l0 < 0 ? 0 : (l0 > L ? L : l0); }
    for (int i = p.T - 1; i >= 0; --i) {
        const bool last = (i == p.T - 1);
        // =========================== PA: attention backward of utterance `pc` on the CTA pair (2 pc, 2 pc + 1) ===========================
        if (pc < B) {
            const int b = pc, half = (p.KC - 1) / 2;
            if (i > 0) {       // DRAM -> L2 one step ahead: the rows of step i-1 this phase starts with (alignment, query, cumulative weights, d ctx)
                const size_t r1 = (size_t)(i - 1) * B + b;
                const char* rows[5] = {reinterpret_cast<const char*>(p.align + (size_t)b * p.align_bstride + (size_t)(i - 1) * L),
                                       reinterpret_cast<const char*>(p.q + r1 * A), reinterpret_cast<const char*>(p.cum + r1 * L),
                                       reinterpret_cast<const char*>(p.dctx_static + r1 * M),
                                       p.dalign ? reinterpret_cast<const char*>(p.dalign + (size_t)b * p.dalign_bstride + (size_t)(i - 1) * L) : nullptr};
                const int bytes[5] = {L * 4, A * 4, L * 4, M * 4, L * 4};
                const int which = tid >> 4, line = tid & 15;           // up to 16 lines of 128 B per row
                if (which < 5 && rows[which] && line * 128 < bytes[which] + 127) l2_prefetch(rows[which] + line * 128);
            }
            const int len = pa_len;                        // loaded once, before the loop
            const int mtiles = (len + 15) / 16;
            // k-tiles (16 memory dims) per register batch of the dw product.  A batch of all 18 k-tiles at M = 288 (one L2 round trip instead
            // of three) was measured slower, also with the cell operands staged in shared memory: the kernel sits at its 255-register cap and
            // spilled in every phase (9 k-tiles as well)
            constexpr int KT = 6;
            {   // Staging of the step's operands.  EVERY global load of the phase is issued before the first dependent instruction: ONE L2
                // round trip instead of five serial ones (partial d ctx sums, alignment row, query, cumulative weights, d alignment);
                // two register slots per thread cover M <= 2 PT and L16 + 48 <= 2 PT (checked on the host)
                const size_t row = (size_t)i * B + b;
                const float* cum = p.cum + row * L;
                float r_g[2], r_p[2][KBA], r_w[2], r_da[2], r_c0[2], r_c1[2], r_q = 0.f, bias_r = 0.f, v_r = 0.f;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int m = tid + e * PT;            // memory dim / text position / Toeplitz index of this slot
                    r_g[e] = 0.f; r_w[e] = 0.f; r_da[e] = 0.f; r_c0[e] = 0.f; r_c1[e] = 0.f;
#pragma unroll
                    for (int k2 = 0; k2 < KBA; ++k2) r_p[e][k2] = 0.f;
                    if (m < M) {
                        r_g[e] = p.dctx_static[row * M + m];
                        if (!last) {
#pragma unroll
                            for (int k2 = 0; k2 < KBA; ++k2) r_p[e][k2] = __ldcg(p.part + ((size_t)k2 * B + b) * p.NOUT + m);
                        }
                    }
                    if (m < L) {
                        r_w[e] = p.align[(size_t)b * p.align_bstride + (size_t)i * L + m];
                        if (p.dalign && m < len) r_da[e] = p.dalign[(size_t)b * p.dalign_bstride + (size_t)i * L + m];
                    }
                    if (m < L16 + 48) {
                        const int l0 = m - half, l1 = l0 + 1;
                        if (l0 >= 0 && l0 < L) r_c0[e] = __ldcg(cum + l0);
                        if (l1 >= 0 && l1 < L) r_c1[e] = __ldcg(cum + l1);
                    }
                }
                if (tid < A) { r_q = p.q[row * A + tid]; bias_r = p.bias[tid]; v_r = p.v[tid]; }
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int m = tid + e * PT;
                    if (m < M) {
                        float g = r_g[e];
#pragma unroll
                        for (int k2 = 0; k2 < KBA; ++k2) g += r_p[e][k2];
                        s_dctx[m] = g;
                        if (hf == 0) p.dctx_tot[row * M + m] = g;
                    }
                    if (m < L16) { s_w[m] = r_w[e]; s_de[m] = r_da[e]; }      // s_de starts as d alignment (or 0); the dw epilogue adds to it
                    if (m < L16 + 48) {
                        const __nv_bfloat16 h0 = __float2bfloat16_rn(r_c0[e]), h1 = __float2bfloat16_rn(r_c1[e]);
                        __nv_bfloat162 hp; hp.x = h0; hp.y = h1;
                        s_Ph[m] = *reinterpret_cast<uint32_t*>(&hp);
                        s_Pl[m] = pack2(r_c0[e] - __bfloat162float(h0), r_c1[e] - __bfloat162float(h1));
                    }
                }
                if (tid < A) { s_qb[tid] = r_q + bias_r; s_vv[tid] = v_r; }
            }
            __syncthreads();
            // B fragments of the dw product: lanes g = 0 hold hi(dctx), g = 1 hold lo(dctx), other columns zero.  They depend on the k-tile only,
            // so the CTA builds the M16 fragments ONCE (every warp used to rebuild all of them: ~40 instructions per fragment and warp)
            for (int idx = tid; idx < p.M16 * 32; idx += PT) {
                const int kt = idx >> 5, gg = (idx >> 2) & 7, tt = idx & 3;
                const int m0 = kt * 16 + 2 * tt;
                uint2 f = make_uint2(0u, 0u);
                if (gg < 2) {
                    const float w0 = m0 < M ? s_dctx[m0] : 0.f, w1 = m0 + 1 < M ? s_dctx[m0 + 1] : 0.f;
                    const float w2 = m0 + 8 < M ? s_dctx[m0 + 8] : 0.f, w3 = m0 + 9 < M ? s_dctx[m0 + 9] : 0.f;
                    const float h0 = __bfloat162float(__float2bfloat16_rn(w0)), h1 = __bfloat162float(__float2bfloat16_rn(w1));
                    const float h2 = __bfloat162float(__float2bfloat16_rn(w2)), h3 = __bfloat162float(__float2bfloat16_rn(w3));
                    f = gg == 0 ? make_uint2(pack2(h0, h1), pack2(h2, h3)) : make_uint2(pack2(w0 - h0, w1 - h1), pack2(w2 - h2, w3 - h3));
                }
                s_bf[idx] = f;
            }
            __syncthreads();
            // dw[l] = dalign + dcum + <dctx, memory[l]> on the tensor cores: A = fragment-major memory (one 16-byte load per lane per
            // MMA), B = (hi(dctx), lo(dctx)) in columns 0 / 1; warp owns position tiles {warp, warp + 8}
            {
                const int g = lane >> 2, tq = lane & 3;
                for (int lt = t_lo + warp; lt < t_hi; lt += 8) {
                    float dacc[4] = {0.f, 0.f, 0.f, 0.f}, dacc2[4] = {0.f, 0.f, 0.f, 0.f};
                    if (lt * 16 < len) {
                        const uint4* fr = p.memFb + (((size_t)b * p.MT + lt) * p.M16) * 32 + lane;
                        for (int kt0 = 0; kt0 < p.M16; kt0 += KT) {
                            uint4 av[KT];
#pragma unroll
                            for (int j = 0; j < KT; ++j)
                                if (kt0 + j < p.M16) av[j] = __ldg(fr + (size_t)(kt0 + j) * 32);
                            uint32_t bfr[KT][2];
#pragma unroll
                            for (int j = 0; j < KT; ++j) {
                                bfr[j][0] = 0u; bfr[j][1] = 0u;
                                if (kt0 + j < p.M16) { const uint2 f = s_bf[(kt0 + j) * 32 + lane]; bfr[j][0] = f.x; bfr[j][1] = f.y; }
                            }
#pragma unroll
                            for (int j = 0; j < KT; j += 2) {        // two independent accumulation chains
                                if (kt0 + j < p.M16) {
                                    const uint32_t af[4] = {av[j].x, av[j].y, av[j].z, av[j].w};
                                    mma_bf16(dacc, af, bfr[j][0], bfr[j][1]);
                                }
                                if (kt0 + j + 1 < p.M16) {
                                    const uint32_t af[4] = {av[j + 1].x, av[j + 1].y, av[j + 1].z, av[j + 1].w};
                                    mma_bf16(dacc2, af, bfr[j + 1][0], bfr[j + 1][1]);
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int q4 = 0; q4 < 4; ++q4) dacc[q4] += dacc2[q4];
                    if (tq == 0) {
#pragma unroll
                        for (int rr = 0; rr < 2; ++rr) {
                            const int l = lt * 16 + g + 8 * rr;
                            float gv = 0.f;
                            if (l < len) gv = (rr ? dacc[2] + dacc[3] : dacc[0] + dacc[1]) + (last ? 0.f : dcum[l]) + s_de[l];   // s_de[l]: d alignment
                            s_de[l] = gv;
                        }
                    }
                }
            }
            __syncthreads();
            // softmax backward: dot = sum_l w[l] dw[l] over ALL positions = own partial + the peer's (exchanged through DSMEM)
            float pdot = 0.f;
            for (int l = t_lo * 16 + tid; l < t_hi * 16 && l < len; l += PT) pdot = fmaf(s_w[l], s_de[l], pdot);
            pdot = block_sum(pdot, s_red);
            if (tid == 0) { tcx::mbar_expect_tx(&xb1, 4); st_async_peer_f32(s_dotx, &xb1, (uint32_t)(hf ^ 1), pdot); }
            tcx::mbar_wait(&xb1, (uint32_t)(p.T - 1 - i) & 1);
            const float dot = pdot + s_dotx[0];           // a + b == b + a: both ranks get the same value
            for (int l = t_lo * 16 + tid; l < t_hi * 16; l += PT) {
                const float d = l < len ? s_w[l] * (s_de[l] - dot) : 0.f;
                s_de[l] = d;
                if (l < L) p.de[((size_t)i * B + b) * L + l] = d;
            }
            __syncthreads();
            BPROF_MARK(0);
            // energies backward on the tensor cores; warp owns position tiles {warp, warp + 8}
            float dqacc[16][2];
#pragma unroll
            for (int nt = 0; nt < 16; ++nt) { dqacc[nt][0] = 0.f; dqacc[nt][1] = 0.f; }
            const int g = lane >> 2, tq = lane & 3;
            for (int mt = t_lo + warp; mt < t_hi && mt < mtiles; mt += 8) {
                const int l0 = mt * 16;
                float sacc[16][4];
#pragma unroll
                for (int nt = 0; nt < 16; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) sacc[nt][e] = 0.f;
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) {
                    const int x = l0 + ks * 16 + g + 2 * tq;       // cumpad index of (row g, col 2t) of this k-step
                    uint32_t ah[4], al[4];
                    ah[0] = s_Ph[x]; ah[1] = s_Ph[x + 8]; ah[2] = s_Ph[x + 8]; ah[3] = s_Ph[x + 16];
                    al[0] = s_Pl[x]; al[1] = s_Pl[x + 8]; al[2] = s_Pl[x + 8]; al[3] = s_Pl[x + 16];
#pragma unroll
                    for (int np = 0; np < 8; ++np) {
                        uint32_t bf[4];
                        ldmatrix_x4(bf[0], bf[1], bf[2], bf[3], sWcB + (size_t)(np * 16 + (lane & 7) + ((lane >> 4) << 3)) * 40 + ks * 16 + ((lane >> 3) & 1) * 8);
                        mma_bf16(sacc[2 * np], ah, bf[0], bf[1]);
                        mma_bf16(sacc[2 * np], al, bf[0], bf[1]);
                        mma_bf16(sacc[2 * np + 1], ah, bf[2], bf[3]);
                        mma_bf16(sacc[2 * np + 1], al, bf[2], bf[3]);
                    }
                }
                // ds = de[l] * v[a] * (1 - tanh^2(S + q + bias + memT)); fragment-major memory projection: 64 bf16 per lane.  Requesting
                // the first job's fragments before the softmax exchange was measured slower (register spills at the 255-register cap)
                const uint4* mf = reinterpret_cast<const uint4*>(p.memTf + (((size_t)b * p.MT + mt) * 32 + lane) * 64);
                const float de0 = s_de[l0 + g], de1 = s_de[l0 + g + 8];
                uint32_t dsA[16][2];
#pragma unroll
                for (int c4 = 0; c4 < 8; ++c4) {
                    const uint4 raw = mf[c4];                      // n-tiles 2*c4, 2*c4+1; 4 values each
                    const uint32_t words[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf) {
                        const int nt = 2 * c4 + hf;
                        const float2 m01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&words[2 * hf]));
                        const float2 m23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&words[2 * hf + 1]));
                        const int a0 = nt * 8 + 2 * tq;
                        const float t0 = tanh_fast(sacc[nt][0] + s_qb[a0] + m01.x), t1 = tanh_fast(sacc[nt][1] + s_qb[a0 + 1] + m01.y);
                        const float t2 = tanh_fast(sacc[nt][2] + s_qb[a0] + m23.x), t3 = tanh_fast(sacc[nt][3] + s_qb[a0 + 1] + m23.y);
                        const float d0 = de0 * s_vv[a0] * (1.f - t0 * t0), d1 = de0 * s_vv[a0 + 1] * (1.f - t1 * t1);
                        const float d2 = de1 * s_vv[a0] * (1.f - t2 * t2), d3 = de1 * s_vv[a0 + 1] * (1.f - t3 * t3);
                        dqacc[nt][0] += d0 + d2; dqacc[nt][1] += d1 + d3;
                        dsA[nt][0] = pack2(d0, d1); dsA[nt][1] = pack2(d2, d3);
                    }
                }
                // G[l, tap] = sum_a ds[l, a] * Wcomb[a, tap]   (C fragments of ds reused as A fragments)
                float gacc[4][4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) gacc[nt][e] = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const uint32_t af[4] = {dsA[2 * j][0], dsA[2 * j][1], dsA[2 * j + 1][0], dsA[2 * j + 1][1]};
#pragma unroll
                    for (int np = 0; np < 2; ++np) {
                        uint32_t bf[4];
                        ldmatrix_x4(bf[0], bf[1], bf[2], bf[3], sWcB2 + (size_t)(np * 16 + (lane & 7) + ((lane >> 4) << 3)) * (A + 8) + j * 16 + ((lane >> 3) & 1) * 8);
                        mma_bf16(gacc[2 * np], af, bf[0], bf[1]);
                        mma_bf16(gacc[2 * np + 1], af, bf[2], bf[3]);
                    }
                }
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) s_G[(l0 - g_lo + g + 8 * (e >> 1)) * GLD + nt * 8 + 2 * tq + (e & 1)] = gacc[nt][e];
            }
            // the G tiles were written through the generic proxy; the bulk copy below reads the boundary tile through the async proxy
            tcx::proxy_fence_shared();
            __syncthreads();                               // every warp is done with s_de / s_qb / s_vv / Ph / Pl, and G is complete
            {   // the boundary tile of G goes to the peer's halo rows (rank 0 sends its last tile, rank 1 its first) as ONE bulk copy of
                // 16 x GLD floats (2112 B: rows of 132 B, tile and s_G 16-byte aligned) that completes on the peer's xb2
                const int ht = hf ? HT0 : HT0 - 1;             // tile sent
                const int peer_g_lo = hf ? 0 : (HT0 - 1) * 16;
                if (tid == 0 && ht >= t_lo && ht < t_hi)
                    tcx::bulk_copy_to_peer(s_G + (size_t)(ht * 16 - peer_g_lo) * GLD, s_G + (size_t)(ht * 16 - g_lo) * GLD, 16 * GLD * 4, &xb2,
                                           (uint32_t)(hf ^ 1));
            }
            // dq[a] = sum_l ds[l, a]: reduce over the 8 row lanes, then over warps
#pragma unroll
            for (int nt = 0; nt < 16; ++nt)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float v = dqacc[nt][c];
                    v += __shfl_xor_sync(0xffffffffu, v, 4);
                    v += __shfl_xor_sync(0xffffffffu, v, 8);
                    v += __shfl_xor_sync(0xffffffffu, v, 16);
                    if (g == 0) s_dqp[warp * A + nt * 8 + 2 * tq + c] = v;
                }
            __syncthreads();
            float pdq = 0.f;                                // this rank's partial of dq[a] (a = tid < A)
            if (tid < A) {
#pragma unroll
                for (int w8 = 0; w8 < 8; ++w8) pdq += s_dqp[w8 * A + tid];
                st_async_peer_f32(s_dqx + tid, &xb2, (uint32_t)(hf ^ 1), pdq);
            }
            {   // what the PEER sends here: its A query-gradient partials, and its boundary tile if it has one (rank 0 always does; rank 1 only
                // when it owns tiles at all)
                const bool peer_sends_tile = hf ? true : (HT0 < p.MT);
                if (tid == 0) tcx::mbar_expect_tx(&xb2, (uint32_t)(A * 4 + (peer_sends_tile ? 16 * GLD * 4 : 0)));
            }
            tcx::mbar_wait(&xb2, (uint32_t)(p.T - 1 - i) & 1);
            if (hf == 0 && tid < A) p.dq[((size_t)i * B + b) * A + tid] = pdq + s_dqx[tid];
            // d cum_{i-1}[j] = d cum_i[j] + sum_k G[j + half - k, k] for the own positions (their G rows: own tiles + the halo tile)
            for (int j = t_lo * 16 + tid; j < t_hi * 16 && j < L; j += PT) {
                float acc = last ? 0.f : dcum[j];
#pragma unroll 4
                for (int k = 0; k < p.KC; ++k) {
                    const int l = j + half - k;
                    if (l >= 0 && l < mtiles * 16) acc += s_G[(size_t)(l - g_lo) * GLD + k];
                }
                s_stage[j] = acc;                           // staged: dcum is still being read by other threads
            }
            __syncthreads();
            for (int j = t_lo * 16 + tid; j < t_hi * 16 && j < L; j += PT) dcum[j] = s_stage[j];
        }
        BPROF_MARK(1);
        if (!grid_barrier(p.barrier, target, nblocks, p.abort_flag)) break;
        BPROF_MARK(2);

        // =========================== PB: attention-LSTM cell backward ===========================
        if (owner) {
            // the recurrent partial sums of the owned units (written by the product of the previous reverse step) and the query gradients
            // of ALL utterances go straight to shared memory: one L2 round trip for both, waited for together with this step's operands.
            // (As is idle between PA and P2: [B][A] query gradients, row b rotated by 8 (b & 7) floats against bank conflicts)
            float* s_dq = reinterpret_cast<float*>(As);
            if (!last)
                for (int c = tid; c < KBA * B * 2; c += PT) {
                    const int kb2 = c >> 1, h4 = (c & 1) * 4;          // kb2 = k2 * B + b
                    cp_async16(s_rp + kb2 * UOWN + h4, p.part + (size_t)kb2 * p.NOUT + M + uo0 + h4);
                }
            {
                const float4* dq4 = reinterpret_cast<const float4*>(p.dq + (size_t)i * B * A);      // [B][A] block of this step, contiguous
                for (int idx = tid; idx < B * 32; idx += PT) {                                       // A == 128 (host check): 32 float4 per utterance
                    const int b = idx >> 5, c4 = idx & 31;
                    cp_async16(s_dq + b * A + ((c4 * 4 + 8 * (b & 7)) & (A - 1)), dq4 + idx);
                }
            }
            cp_async_wait_all();
            __syncthreads();
            float rec_[MAXE];
#pragma unroll
            for (int e = 0; e < MAXE; ++e) {
                const int idx = tid + e * PT;
                float rs = 0.f;
                if (idx < B * UOWN && !last) {
#pragma unroll
                    for (int k2 = 0; k2 < KBA; ++k2) rs += s_rp[k2 * B * UOWN + idx];
                }
                rec_[e] = rs;
            }
            // d h (query part) = dq[b, :] . Wq[:, u] on the tensor cores: A = dq rows staged in shared memory (bf16 hi + lo),
            // B = this CTA's 8 columns of Wq (bf16 hi + lo, prebuilt in wqf); hi.hi + lo.hi + hi.lo = fp32-equivalent
            {
                const int g = lane >> 2, tq = lane & 3, mt = warp & 3, kh = warp >> 2;      // warp = (16-utterance tile, half of the A range)
                float acc[4] = {0.f, 0.f, 0.f, 0.f};
                const int ksteps = A / 32;                                // k-steps of 16 per half
#pragma unroll 4
                for (int ks = 0; ks < ksteps; ++ks) {
                    const int a0 = (kh * ksteps + ks) * 16;
                    uint32_t ah[4], al[4];
#pragma unroll
                    for (int r4 = 0; r4 < 4; ++r4) {
                        const int br = mt * 16 + g + 8 * (r4 & 1);       // rows >= B read stale shared memory: their products are never used
                        const float2 x = *reinterpret_cast<const float2*>(s_dq + br * A + ((a0 + 2 * tq + 8 * (r4 >> 1) + 8 * (br & 7)) & (A - 1)));
                        const __nv_bfloat16 h0 = __float2bfloat16_rn(x.x), h1 = __float2bfloat16_rn(x.y);
                        __nv_bfloat162 hp; hp.x = h0; hp.y = h1;
                        ah[r4] = *reinterpret_cast<uint32_t*>(&hp);
                        al[r4] = pack2(x.x - __bfloat162float(h0), x.y - __bfloat162float(h1));
                    }
                    const uint4 wf = wqf[(a0 >> 4) * 32 + lane];
                    mma_bf16(acc, ah, wf.x, wf.y);
                    mma_bf16(acc, al, wf.x, wf.y);
                    mma_bf16(acc, ah, wf.z, wf.w);
                }
                // each half of the A range to its own slab (outside the dq staging): one barrier, the sum is taken where it is read
                float* d0 = s_dhq + ((kh * 64) + mt * 16 + g) * UOWN + 2 * tq;
                float* d1 = d0 + 8 * UOWN;
                d0[0] = acc[0]; d0[1] = acc[1]; d1[0] = acc[2]; d1[1] = acc[3];
                __syncthreads();
            }
#pragma unroll
            for (int e = 0; e < MAXE; ++e) {
                const int idx = tid + e * PT;
                if (idx < B * UOWN) {
                    const int b = idx / UOWN, uu = idx % UOWN, u = uo0 + uu;
                    const size_t bu = (size_t)b * D + u, g0 = ((size_t)i * B + b) * 4 * D + u;
                    const int BU = B * UOWN;                   // idx = b * UOWN + uu: this pair's slot in each [B][8] staging array
                    float dh = s_pbo[5 * BU + idx] + (s_dhq[b * UOWN + uu] + s_dhq[(64 + b) * UOWN + uu]);
                    float dc_in = 0.f;
                    if (!last) {
                        dh += rec_[e] + dhz_reg[e];
                        dc_in = dc_reg[e];
                    }
                    const float gi = s_pbo[idx], gf = s_pbo[BU + idx], gg = s_pbo[2 * BU + idx], go = s_pbo[3 * BU + idx];
                    const float cp = s_pbo[4 * BU + idx];
                    const float tc = tanh_exp(gf * cp + gi * gg);
                    float dhn, dcn, dc_prev_direct = 0.f, dh_prev_direct = 0.f;
                    if (p.kind == B200TTS_CELL_ZONEOUT) {
                        float kh, kc;
                        if (p.training) {
                            kh = (1.f - p.rate_h) * (p.mask_h ? (float)s_pbm[idx] * inv_h : 1.f);
                            kc = (1.f - p.rate_c) * (p.mask_c ? (float)s_pbm[BU + idx] * inv_c : 1.f);
                        } else { kh = 1.f - p.rate_h; kc = 1.f - p.rate_c; }
                        dhn = dh * kh; dh_prev_direct = dh - dhn;
                        dcn = dc_in * kc + dhn * go * (1.f - tc * tc);
                        dc_prev_direct = dc_in - dc_in * kc;
                    } else {
                        dhn = (p.training && p.mask_h) ? dh * (float)s_pbm[idx] * inv_h : dh;
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
                    if (i > 1 && (uu & 7) == 0) {      // DRAM -> L2 two steps ahead (the shared-memory staging below runs one step ahead)
                        const size_t g1 = g0 - (size_t)2 * B * 4 * D, m1 = (size_t)(i - 2) * B * D + bu;
                        l2_prefetch(p.gates + g1); l2_prefetch(p.gates + g1 + D); l2_prefetch(p.gates + g1 + 2 * D); l2_prefetch(p.gates + g1 + 3 * D);
                        l2_prefetch(p.cstate + m1); l2_prefetch(p.dh_static + m1);
                        if (p.training && p.mask_h) l2_prefetch(p.mask_h + m1);
                        if (p.training && p.mask_c) l2_prefetch(p.mask_c + m1);
                    }
                }
            }
        }
        BPROF_MARK(3);
        // the copies of the next cell backward's operands are issued between this CTA's arrival and its wait: the barrier's leading
        // __syncthreads means every thread is done reading the staging buffer, and they complete while PA runs
        if (!grid_barrier(p.barrier, target, nblocks, p.abort_flag, true, [&]() { pb_stage(i - 1); })) break;
        BPROF_MARK(4);
        if (i == 0) break;

        // =========================== P2: [d ctx | d h](i-1) partial = dgates_i[:, kb] . W[kb, nb] ===========================
        // TMA: the bf16 gate gradients of the K-slice, all utterances (rows >= B zero-filled), as NKT swizzled [64 x 64] tiles; the pair
        // shares kb, so rank r issues ONE box of gates {2r, 2r+1} with multicast into both slots, completing on full_bar[r] of both CTAs; each
        // CTA arms both barriers with NKT/2 tiles, and the MMAs of the first half run while the second half may still be in flight.  Both CTAs
        // last touched their slot (attention scratch, dq staging) before the grid barrier above, so the peer's slot is free.
        // wgmma: D[b, n] (registers of warpgroup 0: 64 utterances x UN outputs) = sum over the tiles, stored straight to the partials
        if (warp == 0) {
            if (tcx::elect_one()) {
                const int r = cta & 1;
                tcx::proxy_fence_shared();       // the slot was last touched through the generic proxy (attention scratch, dq staging)
                tcx::proxy_fence_global();
                tcx::mbar_expect_tx(&full_bar[0], (uint32_t)(NKT / 2) * 8192);
                tcx::mbar_expect_tx(&full_bar[1], (uint32_t)(NKT / 2) * 8192);
                tcx::tma_load_5d_mc(reinterpret_cast<unsigned char*>(As) + (size_t)r * (NKT / 2) * 8192, &tmG, &full_bar[r], 0x3, 0, i * p.dgb_rows, 0,
                                    kb, 2 * r);
            }
            __syncwarp();
        }
        if (warp < 4) {
            constexpr int NR = UNC / 2;
            float acc[NR];
            tcx::mbar_wait(&full_bar[0], prod_it & 1);
            tcx::wgmma_fence();
            for (int c = 0; c < NKT; ++c) {
                if (c == NKT / 2) tcx::mbar_wait(&full_bar[1], prod_it & 1);
                const uint64_t adesc = tcx::make_sw128_desc(tcx::smem_u32(reinterpret_cast<unsigned char*>(As) + (size_t)c * 8192));
                const uint64_t bdesc = tcx::make_sw128_desc(tcx::smem_u32(sW + (size_t)c * UN * 128));
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if constexpr (UNC == TUN_WIDE) tcx::wgmma_m64n96<0, 0>(acc, adesc + 2 * k, bdesc + 2 * k, (c | k) != 0);
                    else if constexpr (UNC == TUN) tcx::wgmma_m64n80<0, 0>(acc, adesc + 2 * k, bdesc + 2 * k, (c | k) != 0);
                }
            }
            tcx::wgmma_commit();
            tcx::wgmma_wait<0>();
            tcx::wgmma_fence_acc(acc);
            // fragment: utterance b = 16 warp + lane / 4 + 8 ((r / 2) % 2), output n0 + 8 (r / 4) + 2 (lane % 4) + r % 2 (NOUT % 4 == 0: a pair
            // is either wholly inside or wholly outside)
            const int brow = 16 * warp + (lane >> 2), ncol = n0 + 2 * (lane & 3);
#pragma unroll
            for (int r = 0; r < NR; r += 2) {
                const int b = brow + 8 * ((r >> 1) & 1), n = ncol + 8 * (r >> 2);
                if (b < B && n < p.NOUT) *reinterpret_cast<float2*>(p.part + ((size_t)kb * B + b) * p.NOUT + n) = make_float2(acc[r], acc[r + 1]);
            }
        }
        ++prod_it;
        BPROF_MARK(5);
        if (!grid_barrier(p.barrier, target, nblocks, p.abort_flag)) break;
        BPROF_MARK(6);
    }
    BPROF_FLUSH;
    // no CTA exits while a multicast it issued may still be landing in its peer.  A watchdog abort leaves the loop through the shared abort
    // flag, which every CTA checks at each grid barrier, so both ranks of a pair stop at the same barrier -- unless the flag is raised just
    // as that barrier completes: the rank that went on then waits for the peer's half of the next operand and ends in the trap of
    // mbar_wait (~2 s), not in a hang
    tcx::cluster_arrive(); tcx::cluster_wait();
}

// -------------------------------------------------------------------------------------------------
// Post pass (fully parallel): accumulate what the recurrence does not need -- d memT, d Wcomb, d v.
// CTA = (utterance b, position tile mt); warp w owns the attention dims [16w, 16w+16); loops over all T steps
// recomputing S^T = Wcomb . T^T on the tensor cores from the saved query / cumulative weights / de.
// -------------------------------------------------------------------------------------------------
struct AttPostArgs {
    int B, T, L, A, KC, MT;
    const float* q; const float* cum; const float* de; const float* bias; const float* v;
    const __nv_bfloat16* WcB;          // [A][40]
    const float* memT;                 // [B, L, A] fp32
    const int* lengths;
    float* dmemT;                      // [B, L, A] out (each element written exactly once)
    float* dWcomb_part;                // [B*MT][A][32]
    float* dv_part;                    // [B*MT][A]
};

__global__ void __launch_bounds__(PT, 3) att_post_kernel(const AttPostArgs p) {
    constexpr int NS = 4;                               // decoder steps per block barrier
    __shared__ uint32_t Ph[2][NS][64], Pl[2][NS][64];
    __shared__ float s_de[2][NS][16], s_q[2][NS][128];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x / p.MT, mt = blockIdx.x % p.MT;
    const int L = p.L, A = p.A, half = (p.KC - 1) / 2, l0 = mt * 16;
    const int g = lane >> 2, tq = lane & 3;
    int len = p.lengths[b];
    len = len < 0 ? 0 : (len > L ? L : len);
    const int a_base = warp * 16;                       // requires A <= 128 (8 warps x 16)
    const bool active = a_base < A && l0 < len;
    // A fragments of Wcomb (rows a, cols k): constant over the whole loop
    uint32_t wa[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const __nv_bfloat16* base = p.WcB + (size_t)(a_base + g) * 40 + ks * 16 + 2 * tq;
        wa[ks][0] = *reinterpret_cast<const uint32_t*>(base);
        wa[ks][1] = *reinterpret_cast<const uint32_t*>(base + 8 * 40);
        wa[ks][2] = *reinterpret_cast<const uint32_t*>(base + 8);
        wa[ks][3] = *reinterpret_cast<const uint32_t*>(base + 8 * 40 + 8);
    }
    // memT values of this thread's S^T fragment: rows a = a_base + g (+8), cols l = l0 + nt*8 + 2t (+1)
    float mT[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int a = a_base + g + 8 * (e >> 1), l = l0 + nt * 8 + 2 * tq + (e & 1);
            // rounded through bf16 exactly like the operand the forward / in-loop kernels consumed
            mT[nt][e] = (a < A && l < L) ? __bfloat162float(__float2bfloat16_rn(p.memT[((size_t)b * L + l) * A + a])) : 0.f;
        }
    const float bias0 = a_base + g < A ? p.bias[a_base + g] : 0.f, bias1 = a_base + g + 8 < A ? p.bias[a_base + g + 8] : 0.f;
    const float v0 = a_base + g < A ? p.v[a_base + g] : 0.f, v1 = a_base + g + 8 < A ? p.v[a_base + g + 8] : 0.f;
    float dmacc[2][4], dwacc[4][4], dvacc[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) dmacc[nt][e] = 0.f;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) dwacc[nt][e] = 0.f;

    // The T steps are independent here (only the accumulators chain), so they are processed in chunks of NS with ONE block barrier per
    // chunk: the operands of the next chunk (cumulative-weight window, de, query of NS steps) are loaded into registers before the MMAs
    // of the current chunk and stored to the other shared-memory buffer after them, i.e. their DRAM / L2 latency hides behind compute.
    float r0[NS], r1[NS];
    auto load = [&](int i0) {
#pragma unroll
        for (int s2 = 0; s2 < NS; ++s2) {
            const int i = i0 + s2;
            r0[s2] = 0.f; r1[s2] = 0.f;
            if (i >= p.T) continue;
            if (tid < 64) {                    // window of cumpad needed by this tile: x in [l0, l0 + 16 + 32)
                const float* cum = p.cum + ((size_t)i * p.B + b) * L;
                const int la = l0 + tid - half, lb = la + 1;
                if (la >= 0 && la < L) r0[s2] = __ldg(cum + la);
                if (lb >= 0 && lb < L) r1[s2] = __ldg(cum + lb);
            } else if (tid < 80) {
                const int l = l0 + tid - 64;
                if (l < L) r0[s2] = __ldg(p.de + ((size_t)i * p.B + b) * L + l);
            } else if (tid >= 128 && tid < 128 + A) {
                r0[s2] = __ldg(p.q + ((size_t)i * p.B + b) * A + tid - 128);
            }
        }
    };
    auto store = [&](int buf) {
#pragma unroll
        for (int s2 = 0; s2 < NS; ++s2) {
            if (tid < 64) {
                const __nv_bfloat16 h0 = __float2bfloat16_rn(r0[s2]), h1 = __float2bfloat16_rn(r1[s2]);
                __nv_bfloat162 hp; hp.x = h0; hp.y = h1;
                Ph[buf][s2][tid] = *reinterpret_cast<uint32_t*>(&hp);
                Pl[buf][s2][tid] = pack2(r0[s2] - __bfloat162float(h0), r1[s2] - __bfloat162float(h1));
            } else if (tid < 80) {
                s_de[buf][s2][tid - 64] = r0[s2];
            } else if (tid >= 128 && tid < 128 + A) {
                s_q[buf][s2][tid - 128] = r0[s2];
            }
        }
    };
    if (l0 < len) { load(0); store(0); }
    __syncthreads();
    for (int i0 = 0; i0 < p.T && l0 < len; i0 += NS) {
        const int buf = (i0 / NS) & 1;
        const bool more = i0 + NS < p.T;
        if (more) load(i0 + NS);
        if (active) {
#pragma unroll
            for (int s2 = 0; s2 < NS; ++s2) {
                if (i0 + s2 >= p.T) break;
                // S^T[a, l] = sum_k Wcomb[a, k] * cumpad[l + k]
                float sacc[2][4];
#pragma unroll
                for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) sacc[nt][e] = 0.f;
#pragma unroll
                for (int ks = 0; ks < 2; ++ks)
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt) {
                        // B fragment (k rows, l cols): (k = ks*16 + 2t (+1) (+8), l = nt*8 + g) -> cumpad[l + k]
                        const int x = nt * 8 + g + ks * 16 + 2 * tq;
                        mma_bf16(sacc[nt], wa[ks], Ph[buf][s2][x], Ph[buf][s2][x + 8]);
                        mma_bf16(sacc[nt], wa[ks], Pl[buf][s2][x], Pl[buf][s2][x + 8]);
                    }
                const float q0 = s_q[buf][s2][a_base + g] + bias0, q1 = s_q[buf][s2][a_base + g + 8] + bias1;
                uint32_t dsA[2][2];
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const float dea = s_de[buf][s2][nt * 8 + 2 * tq], deb = s_de[buf][s2][nt * 8 + 2 * tq + 1];
                    const float t0 = tanh_fast(sacc[nt][0] + q0 + mT[nt][0]), t1 = tanh_fast(sacc[nt][1] + q0 + mT[nt][1]);
                    const float t2 = tanh_fast(sacc[nt][2] + q1 + mT[nt][2]), t3 = tanh_fast(sacc[nt][3] + q1 + mT[nt][3]);
                    const float d0 = dea * v0 * (1.f - t0 * t0), d1 = deb * v0 * (1.f - t1 * t1);
                    const float d2 = dea * v1 * (1.f - t2 * t2), d3 = deb * v1 * (1.f - t3 * t3);
                    dmacc[nt][0] += d0; dmacc[nt][1] += d1; dmacc[nt][2] += d2; dmacc[nt][3] += d3;
                    dvacc[0] += dea * t0 + deb * t1; dvacc[1] += dea * t2 + deb * t3;
                    dsA[nt][0] = pack2(d0, d1); dsA[nt][1] = pack2(d2, d3);
                }
                // d Wcomb[a, k] += sum_l ds^T[a, l] * cumpad[l + k]   (A = ds^T chained; B fragment (l rows, k cols) = cumpad[l + k])
                const uint32_t af[4] = {dsA[0][0], dsA[0][1], dsA[1][0], dsA[1][1]};
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const int x = 2 * tq + nt * 8 + g;                  // l = 2t (+1) (+8), k = nt*8 + g
                    mma_bf16(dwacc[nt], af, Ph[buf][s2][x], Ph[buf][s2][x + 8]);
                }
            }
        }
        if (more) store(buf ^ 1);
        __syncthreads();
    }
    if (a_base < A) {
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int a = a_base + g + 8 * (e >> 1), l = l0 + nt * 8 + 2 * tq + (e & 1);
                if (a < A && l < L) p.dmemT[((size_t)b * L + l) * A + a] = dmacc[nt][e];
            }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int a = a_base + g + 8 * (e >> 1), k = nt * 8 + 2 * tq + (e & 1);
                if (a < A) p.dWcomb_part[((size_t)blockIdx.x * A + a) * 32 + k] = dwacc[nt][e];
            }
        float d0 = dvacc[0], d1 = dvacc[1];
        d0 += __shfl_xor_sync(0xffffffffu, d0, 1); d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
        d1 += __shfl_xor_sync(0xffffffffu, d1, 1); d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
        if (tq == 0) {
            if (a_base + g < A) p.dv_part[(size_t)blockIdx.x * A + a_base + g] = d0;
            if (a_base + g + 8 < A) p.dv_part[(size_t)blockIdx.x * A + a_base + g + 8] = d1;
        }
    }
}

// prep: bf16 copies of Wcomb in the two operand layouts, fragment-major memT
__global__ void att_bwd_prep_kernel(__nv_bfloat16* __restrict__ WcB, __nv_bfloat16* __restrict__ WcB2, __nv_bfloat16* __restrict__ memTf,
                                    const float* __restrict__ WcombT, const float* __restrict__ memT, int B, int L, int A, int KC, int MT) {
    const size_t n1 = (size_t)A * 40, n2 = (size_t)32 * (A + 8), n3 = (size_t)B * MT * 32 * 64;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < n1 + n2 + n3; idx += (size_t)gridDim.x * blockDim.x) {
        if (idx < n1) {
            const int a = idx / 40, k = idx % 40;
            WcB[idx] = __float2bfloat16_rn(k < KC ? WcombT[(size_t)k * A + a] : 0.f);
        } else if (idx < n1 + n2) {
            const size_t j = idx - n1;
            const int k = j / (A + 8), a = j % (A + 8);
            WcB2[j] = __float2bfloat16_rn((k < KC && a < A) ? WcombT[(size_t)k * A + a] : 0.f);
        } else {
            const size_t j = idx - n1 - n2;
            const int v = j % 64, lane = (j / 64) % 32, mt = (j / (64 * 32)) % MT, b = j / ((size_t)64 * 32 * MT);
            const int nt = v / 4, e = v % 4, g = lane >> 2, tq = lane & 3;
            const int l = mt * 16 + g + 8 * (e >> 1), a = nt * 8 + 2 * tq + (e & 1);
            memTf[j] = __float2bfloat16_rn((l < L && a < A) ? memT[((size_t)b * L + l) * A + a] : 0.f);
        }
    }
}

// stage 1: dW[a, k] = sum over the nparts partial blocks (one thread per element, grid over the A * 32 + A outputs; fixed order)
__global__ void att_bwd_reduce_parts_kernel(float* __restrict__ dWsum, float* __restrict__ dvsum, const float* __restrict__ dWcomb_part,
                                            const float* __restrict__ dv_part, int nparts, int A) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < A * 32) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        int p2 = 0;
        for (; p2 + 3 < nparts; p2 += 4) {
            s0 += dWcomb_part[(size_t)p2 * A * 32 + idx]; s1 += dWcomb_part[(size_t)(p2 + 1) * A * 32 + idx];
            s2 += dWcomb_part[(size_t)(p2 + 2) * A * 32 + idx]; s3 += dWcomb_part[(size_t)(p2 + 3) * A * 32 + idx];
        }
        for (; p2 < nparts; ++p2) s0 += dWcomb_part[(size_t)p2 * A * 32 + idx];
        dWsum[idx] = (s0 + s1) + (s2 + s3);
    } else if (idx < A * 32 + A) {
        const int a = idx - A * 32;
        float sv = 0.f;
        for (int p2 = 0; p2 < nparts; ++p2) sv += dv_part[(size_t)p2 * A + a];
        dvsum[a] = sv;
    }
}
// stage 2: dWloc[a, c] += sum_k dWcomb[a, k] * Wc[c, k];  dWc[c, k] += sum_a Wloc[a, c] * dWcomb[a, k];  dv += dvsum
__global__ void att_bwd_finish_kernel(float* __restrict__ dWloc, float* __restrict__ dWc, float* __restrict__ dv,
                                      const float* __restrict__ dWsum, const float* __restrict__ dvsum,
                                      const float* __restrict__ Wloc, const float* __restrict__ Wc, int A, int C, int KC) {
    extern __shared__ float dW[];        // [A][32] reduced dWcomb
    for (int idx = threadIdx.x; idx < A * 32; idx += blockDim.x) dW[idx] = dWsum[idx];
    for (int a = threadIdx.x; a < A; a += blockDim.x) dv[a] += dvsum[a];
    __syncthreads();
    for (int idx = threadIdx.x; idx < A * C; idx += blockDim.x) {
        const int a = idx / C, c = idx % C;
        float s = 0.f;
        for (int k = 0; k < KC; ++k) s = fmaf(dW[a * 32 + k], Wc[c * KC + k], s);
        dWloc[idx] += s;
    }
    for (int idx = threadIdx.x; idx < C * KC; idx += blockDim.x) {
        const int c = idx / KC, k = idx % KC;
        float s = 0.f;
        for (int a = 0; a < A; ++a) s = fmaf(Wloc[a * C + c], dW[a * 32 + k], s);
        dWc[idx] += s;
    }
}

}  // namespace

// -------------------------------------------------------------------------------------------------
// attention loop, host side
// -------------------------------------------------------------------------------------------------
AttBwdExtra att_bwd_extra(const b200tts_decoder_shape& s) {
    AttBwdExtra x;
    size_t off = 0;
    auto take = [&](size_t n) { size_t o = off; off = (off + n + 255) / 256 * 256; return o; };
    x.MT = (s.L + 15) / 16;
    x.part = take((size_t)KBA * s.B * (s.M + s.D) * 4);
    x.wcb = take((size_t)s.A * 40 * 2);
    x.wcb2 = take((size_t)32 * (s.A + 8) * 2);
    x.memTf = take((size_t)s.B * x.MT * 32 * 64 * 2);
    x.de = take((size_t)s.T * s.B * s.L * 4);
    x.dwpart = take((size_t)s.B * x.MT * s.A * 32 * 4);
    x.dvpart = take((size_t)s.B * x.MT * s.A * 4);
    x.barrier = take(256 + NUM_SMS * 8 * 8);
    x.total = off;
    return x;
}

// Geometry of the attention reverse loop.
struct AttBwdGeom {
    int UK, UN, grid; size_t region, smem;      // region = bytes of the TMA slot (= attention scratch capacity)
};
static AttBwdGeom att_bwd_geom(const b200tts_decoder_shape& s) {
    AttBwdGeom g{};
    g.UK = s.D / KBA;
    const int L16 = (s.L + 15) / 16 * 16;
    // Wcomb in two layouts, d cum, Wq fragments (A / 16 x 32 x 16 B), two [64][8] slabs of the query part of d h, and the cell-backward
    // staging of 8 units x B utterances: 6 fp32 operands, 2 mask bytes, KBA recurrent partials
    const size_t extras = (size_t)s.A * 40 * 2 + (size_t)32 * (s.A + 8) * 2 + (size_t)(L16 + 32) * 4 + (size_t)s.A * 32 + 2 * 64 * 8 * 4 +
                          (size_t)s.B * 8 * (6 * 4 + 2 + KBA * 4);
    g.UN = (s.M + s.D <= NBT * TUN) ? TUN : TUN_WIDE; g.grid = KBA * NBT;
    const int NKT = 4 * g.UK / 64;
    g.region = (size_t)NKT * 8192;
    g.smem = 1024 + (size_t)NKT * g.UN * 128 + g.region + extras;
    return g;
}

bool persist_att_bwd_supported(const b200tts_decoder_shape& s) {
    const AttBwdGeom g = att_bwd_geom(s);
    if (s.A != 128 || s.K > 32 || s.B * 8 > 3 * PT || s.D % KBA != 0) return false;
    if (s.M > 2 * PT || (s.L + 15) / 16 * 16 + 48 > 2 * PT) return false;      // register-slot staging of the attention backward
    if (s.D / 8 > g.grid) return false;                       // cell-backward ownership: 8 hidden units per CTA
    if (g.grid / 2 < s.B || g.grid > NUM_SMS) return false;       // one CTA pair per utterance, all CTAs co-resident
    if (g.UK % 64 != 0 || s.B > 64 || s.M + s.D > NBT * g.UN || (s.M + s.D) % 4 != 0) return false;
    const int MT = (s.L + 15) / 16, L16 = MT * 16, HT0 = (MT + 1) / 2;
    // attention-backward scratch of one CTA of the pair (aliases the TMA slot)
    const size_t fl = (size_t)((s.M + 3) & ~3) + 3 * (size_t)L16 + 2 * s.A + 2 * (size_t)(L16 + 48) + 64 + (size_t)(HT0 + 1) * 16 * GLD +
                      8 * (size_t)s.A + s.A + 4 + (size_t)((s.M + 15) / 16) * 32 * 2;
    if (fl * 4 > g.region) return false;
    // the cell-backward phase stages the query gradients [B][A] fp32 in the (then idle) TMA slot.  The bound keeps 2 KB to spare (a [64][8]
    // slab), which holds B <= 60 at D = 512: the shapes this loop accepts are the ones its tests cover
    if ((size_t)s.B * s.A * 4 + 64 * 8 * 4 > g.region) return false;
    return g.smem <= 227 * 1024;
}

int tc_make_mapN_bf16(void* map, const void* base, int rank, const unsigned long long* dims, const unsigned long long* strides, const unsigned* box);

int persist_att_bwd_loop(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                         const DecoderLayout& fl, const float* fws, const PersistLayout& pl, const unsigned char* pws,
                         const float* align, const float* dalign, const float* dh_static, const float* dctx_static, float* dgates,
                         float* dq, float* dctx_tot, float* dmemT, unsigned char* extra, const b200tts_decoder_params& dw,
                         cudaStream_t st, void* dgb_hist) {
    const AttBwdExtra x = att_bwd_extra(s);
    const int B = s.B, D = s.D, M = s.M, T = s.T, L = s.L, A = s.A;
    B200_REQUIRE(persist_att_bwd_supported(s), "persistent attention backward: shape not supported");
    const AttBwdGeom geo = att_bwd_geom(s);
    // the cell backward copies each utterance's 8 keep bytes of a CTA's units as one 8-byte asynchronous copy
    B200_REQUIRE(!s.training || ((uintptr_t)in.mask_att_h | (uintptr_t)in.mask_att_c) % 8 == 0,
                 "persistent attention backward: the attention-LSTM keep masks must be 8-byte aligned");
    AttBwdArgs a{};
    a.B = B; a.T = T; a.D = D; a.M = M; a.L = L; a.A = A; a.KC = s.K; a.NOUT = M + D; a.UK = geo.UK;
    a.UN = geo.UN; a.MT = x.MT;
    a.W = fws + fl.wcat_att; a.ldw = M + D;
    a.gates = fws + fl.ga; a.cstate = fws + fl.ca; a.dh_static = dh_static; a.dctx_static = dctx_static;
    a.mask_h = in.mask_att_h; a.mask_c = in.mask_att_c; a.kind = s.cell_kind; a.training = s.training; a.rate_h = s.rate_h; a.rate_c = s.rate_c;
    a.dgates = dgates;
    a.dgb = static_cast<__nv_bfloat16*>(dgb_hist); a.dgb_step = (long long)B * 4 * D; a.dgb_rows = B;
    a.part = reinterpret_cast<float*>(extra + x.part);
    a.q = fws + fl.q; a.cum = fws + fl.cum; a.align = align; a.align_bstride = (long long)T * L;
    a.dalign = dalign; a.dalign_bstride = (long long)T * L;
    a.bias = w.attn_bias; a.v = w.attn_energy; a.Wq = w.attn_query;
    __nv_bfloat16* wcb = reinterpret_cast<__nv_bfloat16*>(extra + x.wcb);
    __nv_bfloat16* wcb2 = reinterpret_cast<__nv_bfloat16*>(extra + x.wcb2);
    __nv_bfloat16* memTf = reinterpret_cast<__nv_bfloat16*>(extra + x.memTf);
    a.WcB = wcb; a.WcB2 = wcb2; a.memTf = memTf;
    a.memFb = reinterpret_cast<const uint4*>(pws + pl.memFb); a.M16 = pl.M16;
    a.lengths = in.text_lengths; a.dctx_tot = dctx_tot; a.dq = dq; a.de = reinterpret_cast<float*>(extra + x.de);
    a.barrier = reinterpret_cast<unsigned*>(extra + x.barrier); a.abort_flag = reinterpret_cast<int*>(a.barrier + 32);
    a.prof = reinterpret_cast<long long*>(extra + x.barrier + 256);
    const float* wcombT = reinterpret_cast<const float*>(pws + pl.wcombT);
    B200_CUDA(cudaMemsetAsync(a.barrier, 0, 256, st));
    att_bwd_prep_kernel<<<NUM_SMS * 4, 256, 0, st>>>(wcb, wcb2, memTf, wcombT, fws + fl.memT, B, L, A, s.K, x.MT);
    B200_LAUNCH_CHECK();
    const size_t smem = geo.smem;
    void* fn = geo.UN == TUN ? (void*)att_bwd_loop_kernel<TUN> : (void*)att_bwd_loop_kernel<TUN_WIDE>;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = geo.grid;
    int per_sm = 0, dev = 0, sms = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, PT, smem));
    B200_CUDA(cudaGetDevice(&dev));
    B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    B200_REQUIRE(per_sm * sms >= grid && grid % 2 == 0 && grid / 2 >= B, "persistent attention backward: %d CTAs cannot be co-resident / paired", grid);
    // bf16 gate-gradient history dgb [T, B, 4D] as {64 k, T * B rows, UK/64 halves, KBA k-slices, 4 gates}: element (row, g, kb, h, c) at
    // row * 4D + g * D + kb * UK + h * 64 + c; one box = {64, 64 rows, UK/64, 1, 2} = two gates of a CTA's K-slice for one step (each rank
    // of a pair fetches two of the four)
    CUtensorMap tm;
    const unsigned long long dims[5] = {64ull, (unsigned long long)T * B, (unsigned long long)(geo.UK / 64), (unsigned long long)KBA, 4ull};
    const unsigned long long strides[4] = {(unsigned long long)4 * D * 2, 128ull, (unsigned long long)geo.UK * 2, (unsigned long long)D * 2};
    const unsigned box[5] = {64u, 64u, (unsigned)(geo.UK / 64), 1u, 2u};
    B200_TRY(tc_make_mapN_bf16(&tm, a.dgb, 5, dims, strides, box));
    void* params[] = {&tm, &a};
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(PT); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeCooperative;
    attrs[0].val.cooperative = 1;
    attrs[1].id = cudaLaunchAttributeClusterDimension;          // the attention backward of an utterance runs on a CTA pair
    attrs[1].val.clusterDim.x = 2; attrs[1].val.clusterDim.y = 1; attrs[1].val.clusterDim.z = 1;
    cfg.attrs = attrs; cfg.numAttrs = 2;
    int nclusters = 0;
    B200_CUDA(cudaOccupancyMaxActiveClusters(&nclusters, fn, &cfg));
    B200_REQUIRE(nclusters * 2 >= grid, "persistent attention backward: only %d CTA pairs can be co-resident, %d needed", nclusters, grid / 2);
    {
        KernelTimer kt("att_bwd_loop_kernel", st);
        B200_CUDA(cudaLaunchKernelExC(&cfg, fn, params));
    }
    B200_LAUNCH_CHECK();
    // parallel post pass
    AttPostArgs pp{};
    pp.B = B; pp.T = T; pp.L = L; pp.A = A; pp.KC = s.K; pp.MT = x.MT;
    pp.q = a.q; pp.cum = a.cum; pp.de = a.de; pp.bias = w.attn_bias; pp.v = w.attn_energy; pp.WcB = wcb; pp.memT = fws + fl.memT;
    pp.lengths = in.text_lengths; pp.dmemT = dmemT;
    pp.dWcomb_part = reinterpret_cast<float*>(extra + x.dwpart); pp.dv_part = reinterpret_cast<float*>(extra + x.dvpart);
    B200_CUDA(cudaMemsetAsync(dmemT, 0, (size_t)B * L * A * 4, st));
    B200_CUDA(cudaMemsetAsync(pp.dWcomb_part, 0, (size_t)B * x.MT * A * 32 * 4, st));
    B200_CUDA(cudaMemsetAsync(pp.dv_part, 0, (size_t)B * x.MT * A * 4, st));
    {
        KernelTimer kt("att_post_kernel", st);
        att_post_kernel<<<B * x.MT, PT, 0, st>>>(pp);
    }
    B200_LAUNCH_CHECK();
    // the de buffer is dead after the post pass: its head holds the reduced partials
    float* dWsum = a.de;
    float* dvsum = dWsum + (size_t)A * 32;
    att_bwd_reduce_parts_kernel<<<cdiv(A * 32 + A, 128), 128, 0, st>>>(dWsum, dvsum, pp.dWcomb_part, pp.dv_part, B * x.MT, A);
    B200_LAUNCH_CHECK();
    att_bwd_finish_kernel<<<1, 512, (size_t)A * 32 * 4, st>>>(dw.attn_location, dw.attn_loc_features, dw.attn_energy, dWsum, dvsum,
                                                             w.attn_location, w.attn_loc_features, A, s.C, s.K);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // namespace b200tts
