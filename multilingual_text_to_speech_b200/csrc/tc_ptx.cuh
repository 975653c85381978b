// PTX wrappers for the Hopper data path (sm_90a): mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with the accumulator in
// registers, operands in shared memory), proxy fences, mma.sync, distributed shared memory, and the grid barrier of the persistent loops.
// The one home of these primitives: every kernel file that needs one includes this header and says `using namespace tcx;`.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace b200tts {
namespace tcx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Out of line on purpose: an inlined trap makes ptxas drop the setmaxnreg.inc limit of the code around it back to the launch's uniform
// register cap (measured with -Xptxas -v: the compute warps of the forward loops then spill), a call to this function does not.
static __device__ __noinline__ __attribute__((noreturn)) void watchdog_trap() { __trap(); }
// spin on the phase parity; a protocol bug must not hang the GPU: trap after ~2 s
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    const long long t0 = clock64();
    for (;;) {
        uint32_t done;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return;
        if (clock64() - t0 > 4000000000ll) watchdog_trap();
    }
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
// multicast variants: ONE issue writes the box to the same shared-memory offset in every CTA of the cluster named in cta_mask and completes
// its bytes on the mbarrier at the same offset in each of them (every receiving CTA arms its own barrier)
__device__ __forceinline__ void tma_load_3d_mc(void* smem, const CUtensorMap* map, uint64_t* bar, uint16_t cta_mask, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5, %6}], [%2], %3;"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d_mc(void* smem, const CUtensorMap* map, uint64_t* bar, uint16_t cta_mask, int c0, int c1, int c2, int c3,
                                               int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5, %6, %7, %8}], [%2], %3;"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
// distributed shared memory: the shared::cluster address of the same-offset location in the cluster's CTA `rank`
__device__ __forceinline__ uint32_t peer_addr(const void* local_smem, uint32_t rank) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(local_smem)), "r"(rank));
    return ra;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) { asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
// remote store that completes its 4 bytes on the PEER's mbarrier (data + signal in one instruction): a pair exchange needs no cluster barrier
// and none of the memory fence its release semantics imply
__device__ __forceinline__ void st_async_peer_f32(const float* local_smem, const uint64_t* local_bar, uint32_t peer_rank, float v) {
    const uint32_t ra = peer_addr(local_smem, peer_rank), rb = peer_addr(local_bar, peer_rank);
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(ra), "r"(__float_as_uint(v)), "r"(rb) : "memory");
}
// bulk copy of `bytes` (a multiple of 16; both addresses 16-byte aligned) from this CTA's shared memory to the peer CTA `peer_rank` of the
// cluster: dst and bar are given as this CTA's addresses of the same-offset buffer / mbarrier in the peer, whose barrier the copy completes
// its bytes on.  The source must have been made visible to the async proxy (proxy_fence_shared after the generic writes).
__device__ __forceinline__ void bulk_copy_to_peer(const void* dst, const void* src, uint32_t bytes, const uint64_t* bar, uint32_t peer_rank) {
    const uint32_t rd = peer_addr(dst, peer_rank), rb = peer_addr(bar, peer_rank);
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(rd), "r"(smem_u32(src)), "r"(bytes), "r"(rb)
                 : "memory");
}
// thread-block cluster barrier, split into arrive and wait (every thread of every CTA of the cluster)
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void proxy_fence_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void proxy_fence_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void l2_prefetch(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// named barrier 1 among the first N threads of the CTA (the compute warps of a warp-specialised kernel)
template <int N>
__device__ __forceinline__ void csync() { asm volatile("bar.sync 1, %0;" ::"n"(N) : "memory"); }

// ---- mma.sync (one warp) ----
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    const uint32_t addr = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// two floats -> one bf16x2 register (round to nearest), lo in the low half
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float tanh_fast(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// tanh of the bf16 perf mode's cell (forward loops, and the recomputed cell state of the reverse loops): ex2-based, ~1e-6 relative error
__device__ __forceinline__ float tanh_exp(float x) { return 2.f * __fdividef(1.f, 1.f + __expf(-2.f * x)) - 1.f; }

// ---- grid barrier of the cooperative persistent loops ----
// Monotonic-counter barrier over ALL threads of every CTA; returns false if the watchdog fired (~2 s) or another CTA raised the abort
// flag.  Arrival is ONE release-reduction (cumulative: it orders the whole CTA's writes, which the preceding __syncthreads made visible to
// thread 0); the wait polls with relaxed loads and issues a single acquire fence after the last one.
//   s_ok:        the caller's __shared__ int, through which thread 0 hands the verdict to the CTA
//   async_fence: the data written before the barrier is read by other CTAs through TMA (async proxy); pass a literal, so it folds away
//   overlap:     runs on every thread BETWEEN the CTA's arrival and its wait: work that does not depend on other CTAs (the next step's
//                operand prefetch) hides under the barrier latency instead of delaying the arrival
struct NoOverlap { __device__ __forceinline__ void operator()() const {} };
template <typename Overlap = NoOverlap>
__device__ __forceinline__ bool grid_barrier(unsigned* counter, unsigned& target, unsigned nblocks, int* abort_flag, int* s_ok, bool async_fence,
                                             Overlap overlap = Overlap()) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += nblocks;
        if (async_fence) proxy_fence_global();
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
    }
    overlap();
    if (threadIdx.x == 0) {
        int ok = 1;
        const long long t0 = clock64();
        unsigned polls = 0;
        for (;;) {                      // nothing but the counter load in the polling loop: its round trip is the barrier latency
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
// The side of grid_barrier of a warpgroup that runs its own step loop (the MMA warpgroup of the forward loops): it arrives at the same two
// CTA-wide barriers, in the same order, and leaves the arrival and the polling to thread 0.  Staying in the CTA barrier (instead of waiting on
// an mbarrier that thread 0 signals) keeps the ordering of a single loop: a TMA issued after the barrier reads other CTAs' rows only after
// thread 0's acquire fence, and the watchdog verdict s_ok reaches both roles through the same barrier.
__device__ __forceinline__ bool grid_barrier_mma(const int* s_ok) {
    __syncthreads();
    __syncthreads();
    return *s_ok != 0;
}

// ---- wgmma (all 128 threads of a warpgroup = 4 consecutive warps starting at a multiple of 4 execute these) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across wgmma_wait
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier of one warpgroup (ids 8 + warpgroup index: clear of the ids the kernels use)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(8 + wg) : "memory"); }

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T per instruction, bf16 operands from shared-memory descriptors, fp32 accumulator in registers.
// TA / TB = 1: the operand is MN-major (transposed).  Fragment of thread t of the warpgroup: d[r] holds
//   row = 16 (t / 32) + (t % 32) / 4 + 8 ((r / 2) % 2),  column = 8 (r / 4) + 2 (t % 4) + r % 2.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n80(float (&d)[40], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %42, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, "
        "%40, %41, p, 1, 1, %43, %44;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n96(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p, 1, 1, %51, %52;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}

// K-major SWIZZLE_128B operand tile (rows of 64 bf16 = 128 B, 8-row groups 1024 B apart): wgmma shared-memory descriptor
// (start >> 4 | leading byte offset >> 4 << 16 | stride byte offset >> 4 << 32 | layout SWIZZLE_128B (1) << 62); a K = 16 step inside
// the swizzle atom advances the start address by 32 B (+2)
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// MN-major SWIZZLE_128B operand tile: 64-element (128 B) lines along MN, one line per k row, 8-row groups 1024 B apart (stride byte offset),
// the next 64-element MN chunk 8 KB further (leading byte offset); a K = 16 step advances 16 rows = 2048 B (+128)
__device__ __forceinline__ uint64_t make_sw128_mn_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)(8192 >> 4) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

}  // namespace tcx
}  // namespace b200tts
