// Shared host side of the persistent recurrent kernels of the bf16 perf mode.
//
//   * persist_plan: which of the three decoder recurrences (attention forward + generator forward, generator reverse,
//     attention reverse) run as one persistent TMA + wgmma launch for a given shape; every other shape runs the
//     per-step kernel chains;
//   * persist_layout: the byte layout of the persistent workspace region (bf16 operand rows of the forward loops,
//     attention operands, grid barrier and profile counters);
//   * persist_att_prep: the attention operands both the forward (decoder_persist_tc.cu) and the reverse
//     (decoder_persist_bwd.cu) attention loops read: Wcomb = Wloc . Wc, its bf16 copy, and fragment-major bf16 copies of
//     the memory projection and of the encoder memory.
// Reference semantics: modules/attention.py:39-86.
#include <cuda_bf16.h>
#include "decoder_internal.cuh"

namespace b200tts {

namespace {

__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

// WcB[a][40] = bf16 Wcomb[a][k] (zero for k >= KC);  memTf = fragment-major bf16 memory projection:
// memTf[b][mt][lane][nt*4 + e] = memT[b][mt*16 + (lane>>2) + 8*(e>>1)][nt*8 + 2*(lane&3) + (e&1)]
__global__ void att_prep_kernel(__nv_bfloat16* __restrict__ WcB, __nv_bfloat16* __restrict__ memTf, const float* __restrict__ WcombT,
                                const float* __restrict__ memT, int B, int L, int A, int KC, int MT) {
    const size_t n1 = (size_t)A * 40, n3 = (size_t)B * MT * 32 * 64;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < n1 + n3; idx += (size_t)gridDim.x * blockDim.x) {
        if (idx < n1) {
            const int a = idx / 40, k = idx % 40;
            WcB[idx] = __float2bfloat16_rn(k < KC ? WcombT[(size_t)k * A + a] : 0.f);
        } else {
            const size_t j = idx - n1;
            const int v = j % 64, lane = (j / 64) % 32, mt = (j / (64 * 32)) % MT, b = j / ((size_t)64 * 32 * MT);
            const int nt = v / 4, e = v % 4, g = lane >> 2, tq = lane & 3;
            const int l = mt * 16 + g + 8 * (e >> 1), a = nt * 8 + 2 * tq + (e & 1);
            memTf[j] = __float2bfloat16_rn((l < L && a < A) ? memT[((size_t)b * L + l) * A + a] : 0.f);
        }
    }
}

// Fragment-major bf16 copies of the encoder memory for mma.m16n8k16 A operands (one 16-byte load per lane per MMA):
//   memFf[b][mt][kt][lane] : A[r][c] = memory[b][kt*16 + c][mt*16 + r]   (memory^T: rows = memory dims, k = positions)   -> context
//   memFb[b][lt][kt][lane] : A[r][c] = memory[b][lt*16 + r][kt*16 + c]   (rows = positions, k = memory dims)             -> d weights
// lane (g = lane>>2, tq = lane&3) holds {A[g][2tq..+1], A[g+8][2tq..+1], A[g][2tq+8..+9], A[g+8][2tq+8..+9]}; zero padded.
__global__ void mem_frag_kernel(uint4* __restrict__ memFf, uint4* __restrict__ memFb, const float* __restrict__ memory, int B, int L, int M,
                                int M16, int MT) {
    const size_t per = (size_t)B * M16 * MT * 32;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < 2 * per; idx += (size_t)gridDim.x * blockDim.x) {
        const bool fwd = idx < per;
        const size_t j = fwd ? idx : idx - per;
        const int lane = j % 32, g = lane >> 2, tq = lane & 3;
        int kt, ot, b;
        if (fwd) { kt = (j / 32) % MT; ot = (j / ((size_t)32 * MT)) % M16; b = j / ((size_t)32 * MT * M16); }
        else { kt = (j / 32) % M16; ot = (j / ((size_t)32 * M16)) % MT; b = j / ((size_t)32 * M16 * MT); }
        auto at = [&](int r, int c) -> float {
            const int l = fwd ? kt * 16 + c : ot * 16 + r;
            const int m = fwd ? ot * 16 + r : kt * 16 + c;
            return (l < L && m < M) ? memory[((size_t)b * L + l) * M + m] : 0.f;
        };
        uint4 v;
        v.x = pack2(at(g, 2 * tq), at(g, 2 * tq + 1));
        v.y = pack2(at(g + 8, 2 * tq), at(g + 8, 2 * tq + 1));
        v.z = pack2(at(g, 2 * tq + 8), at(g, 2 * tq + 9));
        v.w = pack2(at(g + 8, 2 * tq + 8), at(g + 8, 2 * tq + 9));
        (fwd ? memFf : memFb)[j] = v;
    }
}

// WcombT[k, a] = sum_c Wloc[a, c] * Wc[c, k]
__global__ void wcomb_kernel(float* __restrict__ WcombT, const float* __restrict__ Wloc, const float* __restrict__ Wc, int A, int C, int K) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= K * A) return;
    const int k = idx / A, a = idx % A;
    float s = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(Wloc[a * C + c], Wc[c * K + k], s);
    WcombT[idx] = s;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
PersistPlan persist_plan(const b200tts_decoder_shape& s) {
    PersistPlan p;
    // the persistent attention loops are built around the location term; forward attention runs the per-step chains
    if (forward_attention(s)) return p;
    // a training forward runs persistent only together with the persistent attention reverse loop: the forward loops round
    // memory / memT to bf16, and only that reverse loop recomputes the attention with the same operands
    const bool att_bwd = persist_att_bwd_supported(s);
    p.fwd = tc_persist_supported(s) && (!s.training || att_bwd);
    p.gen_bwd = tc_persist_gen_bwd_supported(s);
    p.att_bwd = s.training && p.fwd;      // reads the attention operands persist_att_prep() left for the forward loops
    return p;
}

PersistLayout persist_layout(const b200tts_decoder_shape& s) {
    PersistLayout l;
    size_t off = 0;     // in bytes, 256-aligned regions
    auto take = [&](size_t n) { size_t o = off; off = (off + n + 255) / 256 * 256; return o; };
    const size_t T = s.T, B = s.B;
    const TcPersistGeom g = tc_persist_geom(s);
    l.aib = take((T + 1) * B * (size_t)g.Kp_att * 2);
    l.hgb = take((T + 1) * B * (size_t)g.Kp_gen * 2);
    l.wcombT = take(forward_attention(s) ? 0 : (size_t)s.K * s.A * 4);     // K is ignored for forward attention
    l.wcb = take((size_t)s.A * 40 * 2);
    l.MT = (s.L + 15) / 16;
    l.memTf = take((size_t)s.B * l.MT * 32 * 64 * 2);
    l.M16 = (s.M + 15) / 16;
    l.memFf = take((size_t)s.B * l.M16 * l.MT * 32 * 16);
    l.memFb = take((size_t)s.B * l.M16 * l.MT * 32 * 16);
    l.barrier = take(256 + NUM_SMS * 8 * 8 * 4);   // barrier + abort flag, then 4 x [NUM_SMS][8] profile counters (att, gen, att roles, gen roles)
    l.total = off;
    return l;
}

// Wcomb and the fragment-major projections shared by the forward and backward persistent kernels
int persist_att_prep(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                     const DecoderLayout& fl, float* ws, unsigned char* pws, cudaStream_t st) {
    const PersistLayout l = persist_layout(s);
    const int B = s.B, M = s.M;
    float* wcombT = reinterpret_cast<float*>(pws + l.wcombT);
    wcomb_kernel<<<cdiv(s.K * s.A, 256), 256, 0, st>>>(wcombT, w.attn_location, w.attn_loc_features, s.A, s.C, s.K);
    B200_LAUNCH_CHECK();
    __nv_bfloat16* wcb = reinterpret_cast<__nv_bfloat16*>(pws + l.wcb);
    __nv_bfloat16* memTf = reinterpret_cast<__nv_bfloat16*>(pws + l.memTf);
    att_prep_kernel<<<NUM_SMS * 4, 256, 0, st>>>(wcb, memTf, wcombT, ws + fl.memT, B, s.L, s.A, s.K, l.MT);
    B200_LAUNCH_CHECK();
    mem_frag_kernel<<<NUM_SMS * 4, 256, 0, st>>>(reinterpret_cast<uint4*>(pws + l.memFf), reinterpret_cast<uint4*>(pws + l.memFb), in.memory, B,
                                             s.L, M, l.M16, l.MT);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // namespace b200tts
