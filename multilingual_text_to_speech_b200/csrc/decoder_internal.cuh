// Internal layout of the decoder workspace shared by the forward and backward orchestrators.
#pragma once
#include "common.cuh"
#include "../../include/b200tts.h"

namespace b200tts {

constexpr int CELL_UNITS = 32;      // hidden units per CTA of the LSTM cell kernels
constexpr int ATT_THREADS = 256;    // attention step kernels: 8 warps

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static inline int pick_splitk(int M, int N, int K) {
    const int tiles = cdiv(M, 64) * cdiv(N, 64);
    int s = (NUM_SMS + tiles / 2) / (tiles > 0 ? tiles : 1);
    if (s < 1) s = 1;
    if (s > 8) s = 8;
    const int kmax = cdiv(K, 16);
    if (s > kmax) s = kmax > 0 ? kmax : 1;
    return s;
}

// Extras of the persistent bf16 kernels (decoder_persist.cu); offsets in BYTES from the region base.
struct PersistLayout {
    size_t aib;      // bf16 [T+1, B, Kp_att]  [h_att | ctx | 0] operands (Kp_att, Kp_gen: TcPersistGeom)
    size_t hgb;      // bf16 [T+1, B, Kp_gen]  [h_gen | 0] operands
    size_t wcombT;   // f32  [K, A]
    size_t wcb;      // bf16 [A, 40]   Wcomb[a][k]
    size_t memTf;    // bf16 [B, MT, 32, 64] fragment-major memory projection
    int MT;
    int M16;         // ceil(M / 16)
    size_t memFf;    // uint4 [B, M16, MT, 32]  fragment-major memory^T (context MMA)
    size_t memFb;    // uint4 [B, MT, M16, 32]  fragment-major memory   (attention-backward weight-gradient MMA)
    size_t barrier;  // grid-barrier counter (+ abort flag at +128 B)
    size_t total;
};
PersistLayout persist_layout(const b200tts_decoder_shape& s);

// Which decoder recurrences run as one persistent TMA + wgmma launch in the bf16 perf mode (decoder_persist.cu); every other shape
// runs the per-step kernel chains.
//   fwd:     attention-LSTM + attention loop and generator-LSTM loop (decoder_persist_tc.cu)
//   gen_bwd: generator-LSTM reverse loop (decoder_persist_bwd_tc.cu)
//   att_bwd: attention-LSTM + attention reverse loop (decoder_persist_bwd.cu); training only, and only after the persistent forward
struct PersistPlan { bool fwd = false, gen_bwd = false, att_bwd = false; };
PersistPlan persist_plan(const b200tts_decoder_shape& s);
// dynamic shared memory one CTA of a persistent loop may take: the 227 KB an SM offers a block, less room for the loops' static shared memory
// (mbarriers, barrier verdict, phase counters: 1 KB as ptxas lays it out)
constexpr size_t PERSIST_SMEM_LIMIT = 227 * 1024 - 1088;
// Cooperative launch of a persistent loop (decoder_persist.cu): sets the kernel's dynamic shared-memory limit, checks that all `grid` CTAs
// (and, with `pairs`, all grid / 2 clusters of 2) can be co-resident, and launches under the kernel timer `name`.
int launch_persistent(const char* name, const void* fn, int grid, int threads, size_t smem, bool pairs, void** params, cudaStream_t st);

// All offsets are in floats from the workspace base.
struct DecoderLayout {
    // saved for backward
    size_t xtm;      // [T, B, N]      prenet input, time-major, row i = frame fed at step i
    size_t p0, p1;   // [T, B, P]      prenet activations after relu+dropout
    size_t ga, gg;   // [T, B, 4D]     attention / generator LSTM gates (post activation i,f,g,o)
    size_t ai;       // [T+1, B, M+D]  row i = [ctx_{i-1} | h_att_{i-1}]  (row 0 = 0)
    size_t ca;       // [T+1, B, D]    attention LSTM cell state (row 0 = 0)
    size_t hg, cg;   // [T+1, B, D]    generator LSTM states
    size_t q;        // [T, B, A]      attention queries
    size_t cum;      // [T+1, B, L]    cumulative attention weights BEFORE step i (forward attention: alpha BEFORE step i)
    size_t memT;     // [B, L, A]      memory . Wm^T
    size_t fs;       // [T, B, R*(N+1)] R frames | R stop logits of each step, time-major
    // derived parameters
    size_t wcat_att; // [4D, M+D] = [W_ih_att[:, P:] | W_hh_att]
    size_t bsum_att, bsum_gen;  // [4D]
    size_t wfs;      // [R*(N+1), D+M] = [frame_w ; stop_w]
    size_t bfs;      // [R*(N+1)]
    // scratch
    size_t qpart;    // [max(ncell_blocks, D/16), B, A]
    size_t part;     // split-K partials
    size_t persist;  // byte-addressed extras of the persistent bf16 kernels (PersistLayout), stored as floats
    size_t total;
    int split_att, split_gen, ncell_blocks;
};

// Frames per decoder step (b200tts_decoder_shape.R, 0 = 1).
static inline int frames_per_step(const b200tts_decoder_shape& s) { return s.R > 0 ? s.R : 1; }
// The frames <-> steps mapping: the entry points turn the caller's shape (T = target frames) into this step shape (T = S = ceil(T / R)
// decoder steps, R normalised), and everything behind them -- layouts, persist_plan, the recurrences -- sees only steps.  The frame-level
// edges (prep_target_kernel, the [frame ; stop] projection of width R*(N+1), split_frames / gather_frame_grads and the fed-back frame)
// read R from it and take the frame count as a separate argument.
static inline b200tts_decoder_shape step_shape(const b200tts_decoder_shape& frames) {
    b200tts_decoder_shape s = frames;
    s.R = frames_per_step(frames);
    s.T = frames.T > 0 ? (frames.T + s.R - 1) / s.R : frames.T;
    return s;
}
// width of one [frame ; stop] row of a step: R*N frame values, then R stop logits
static inline int fs_width(const b200tts_decoder_shape& s) { return frames_per_step(s) * (s.N + 1); }

static inline DecoderLayout decoder_layout(const b200tts_decoder_shape& s) {
    DecoderLayout l;
    size_t off = 0;
    auto take = [&](size_t n) { size_t o = off; off = align_up(off + n, 64); return o; };
    const size_t T = s.T, B = s.B, D = s.D, M = s.M, P = s.P, A = s.A, N = s.N, L = s.L;
    l.xtm = take(T * B * N);
    l.p0 = take(T * B * P);
    l.p1 = take(T * B * P);
    l.ga = take(T * B * 4 * D);
    l.gg = take(T * B * 4 * D);
    l.ai = take((T + 1) * B * (M + D));
    l.ca = take((T + 1) * B * D);
    l.hg = take((T + 1) * B * D);
    l.cg = take((T + 1) * B * D);
    l.q = take(T * B * A);
    l.cum = take((T + 1) * B * L);
    l.memT = take(B * L * A);
    const size_t W = fs_width(s);
    l.fs = take(T * B * W);
    l.wcat_att = take(4 * D * (M + D));
    l.bsum_att = take(4 * D);
    l.bsum_gen = take(4 * D);
    l.wfs = take(W * (D + M));
    l.bfs = take(W);
    l.ncell_blocks = cdiv(s.D, CELL_UNITS);
    l.qpart = take((size_t)cdiv(s.D, 16) * B * A);
    l.split_att = pick_splitk(s.B, 4 * s.D, s.M + s.D);
    l.split_gen = pick_splitk(s.B, 4 * s.D, s.D);
    const int smax = l.split_att > l.split_gen ? l.split_att : l.split_gen;
    l.part = take((size_t)smax * B * 4 * D);
    l.persist = take(persist_layout(s).total / sizeof(float) + 64);
    l.total = off;
    return l;
}

int validate_decoder_shape(const b200tts_decoder_shape& s);
static inline bool forward_attention(const b200tts_decoder_shape& s) { return s.att_kind == B200TTS_ATT_FORWARD; }
static inline bool attention_window(const b200tts_decoder_shape& s) { return s.att_window_ahead > 0; }
// forced attention rows (synthesis from given alignments) are given: only b200tts_decoder_forward_chunk takes them
static inline bool forced_inputs(const b200tts_decoder_inputs& in) { return in.forced_count != 0 || in.forced_rows || in.forced_alignment; }

// ---- forward attention (modules/attention.py:89-124): the part of the step its forward and backward kernels share, so that the
// backward recomputes bit-identical transition probabilities and takes the same clamp decisions as the forward did ----
// s[l] = softmax over ALL l < L of v . tanh(qb + memT[l])  (qb = q + bias; the reference does not mask before this softmax).
// One CTA, blockDim.x a multiple of 32; s >= L floats, red >= 33 floats; ends with a __syncthreads.
__device__ __forceinline__ void fwd_att_transition(const float* qb, const float* vv, const float* __restrict__ memT, int L, int A,
                                                   float* s, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int l = warp; l < L; l += nw) {
        const float* mt = memT + (size_t)l * A;
        float e = 0.f;
        for (int a = lane; a < A; a += 32) e = fmaf(vv[a], tanhf(qb[a] + mt[a]), e);
        e = warp_sum(e);
        if (lane == 0) s[l] = e;
    }
    __syncthreads();
    float mx = -INFINITY;
    for (int l = threadIdx.x; l < L; l += blockDim.x) mx = fmaxf(mx, s[l]);
    mx = block_max(mx, red);
    float sum = 0.f;
    for (int l = threadIdx.x; l < L; l += blockDim.x) {
        const float ex = expf(s[l] - mx);
        s[l] = ex;
        sum += ex;
    }
    sum = block_sum(sum, red);
    for (int l = threadIdx.x; l < L; l += blockDim.x) s[l] = s[l] / sum;
    __syncthreads();
}
// a[l] = (alpha[l] + alpha[l-1]) * s[l] for l < len, 0 beyond (the reference's in-place mask); the weights before the clamp
__device__ __forceinline__ float fwd_att_product(const float* __restrict__ alpha, const float* s, int l, int len) {
    return l < len ? (alpha[l] + (l > 0 ? alpha[l - 1] : 0.f)) * s[l] : 0.f;
}
constexpr float FWD_ATT_FLOOR = 1e-6f;      // torch.clamp(energies, 1e-6) (attention.py:119)
constexpr float FWD_ATT_NORM_EPS = 1e-12f;  // F.normalize(p=1) eps

// wgmma / TMA persistent forward loops (decoder_persist_tc.cu): operand rows are [h | ctx | 0] in 64-column k-blocks.
// grid = (D / 16) row blocks x NBH batch halves; slot_kb_att = the attention loop's ring slot (the larger of its two chunks), smem_att its
// dynamic shared memory, use_btab = the context product's B-fragment table fits behind the attention scratch
struct TcPersistGeom {
    int Kp_att, Kp_gen, nkb_att, nkb_gen, nkb_h, ch_c_att, n_c_att, alias_att, ch_h_att, slot_att, ch_h_gen, slot_gen;
    int grid, NBH, slot_kb_att, use_btab;
    size_t smem_att;
};
TcPersistGeom tc_persist_geom(const b200tts_decoder_shape& s);
bool tc_persist_supported(const b200tts_decoder_shape& s);
int tc_persist_att_loop(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                        const DecoderLayout& fl, float* ws, unsigned char* pws, float* align, cudaStream_t st);
int tc_persist_gen_loop(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                        const DecoderLayout& fl, float* ws, unsigned char* pws, cudaStream_t st);
// attention operands of the persistent loops (Wcomb, fragment-major projections) -> persistent workspace
int persist_att_prep(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                     const DecoderLayout& fl, float* ws, unsigned char* pws, cudaStream_t st);
struct AttBwdExtra { int MT; size_t part, wcb, wcb2, memTf, de, dwpart, dvpart, barrier, total; };
AttBwdExtra att_bwd_extra(const b200tts_decoder_shape& s);
// geometry of the attention reverse loop: UK hidden units per K-slice, UN outputs per n-block, grid CTAs, region = bytes of the TMA slot
// (= attention scratch capacity), smem = dynamic shared memory of one CTA
struct AttBwdGeom { int UK, UN, grid; size_t region, smem; };
AttBwdGeom att_bwd_geom(const b200tts_decoder_shape& s);
bool persist_att_bwd_supported(const b200tts_decoder_shape& s);
// dgb_hist: [T, B, 4D] bf16 history of the gate gradients (out), read in place by the time-batched weight-gradient products
int persist_att_bwd_loop(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                         const DecoderLayout& fl, const float* fws, const PersistLayout& pl, const unsigned char* pws,
                         const float* align, const float* dalign, const float* dh_static, const float* dctx_static, float* dgates,
                         float* dq, float* dctx_tot, float* dmemT, unsigned char* extra, const b200tts_decoder_params& dw,
                         cudaStream_t st, void* dgb_hist);
size_t persist_bwd_gen_extra_bytes(const b200tts_decoder_shape& s);
bool tc_persist_gen_bwd_supported(const b200tts_decoder_shape& s);
int tc_persist_gen_bwd_loop(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                            const DecoderLayout& fl, const float* fws, const float* dh_static, float* dgates, unsigned char* extra,
                            cudaStream_t st, void* dgb_hist);

// ---- LSTM cell kernels (decoder_fwd.cu / decoder_bwd.cu), shared with the encoder bi-LSTM ----
struct CellFwdArgs {
    const float* xproj; float* gates;                 // [B, 4D] (may alias)
    const float* part; int nsplit; size_t part_stride;
    const float* c_prev;                              // [B, D]
    const float* h_prev; int ld_hprev;                // [B, ld]
    float* c_out;                                     // [B, D]
    float* h_out; int ld_hout;                        // [B, ld]
    const uint8_t* mask_h; const uint8_t* mask_c;     // [B, D] or null
    int kind, training; float rate_h, rate_c;
    const float* Wq; int A; float* qpart;             // optional: qpart[blk, B, A] = h[:, blk units] . Wq[:, blk units]^T
    float* y_out; int ld_y;                            // optional: y[b, u] = valid ? h : 0 (packed-sequence output)
    const int* lengths; int step;                     // optional: utterance b is valid at this step iff step < lengths[b]
    int B, D;
};

struct CellBwdArgs {
    const float* gates;                       // [B, 4D] activated i,f,g,o
    const float* c_prev;                      // [B, D]
    const float* dh_static; int ld_dhs;       // [B, ld] or null
    const float* part; int nsplit; size_t part_stride; int ld_part; int part_col0;   // recurrent dh partials (null on the last step)
    const float* dq; const float* Wq; int A;  // optional: dh += dq[b, :] . Wq[:, u]
    float* dc_state;                          // [B, D] in: d c_out of this step; out: d c_out of the previous step
    float* dhz_state;                         // [B, D] zoneout: direct d h_prev term (in/out); null for the dropout cell
    const uint8_t* mask_h; const uint8_t* mask_c;
    int kind, training; float rate_h, rate_c;
    float* dgates;                            // [B, 4D] out (pre-activation gradients)
    const int* lengths; int step;             // optional packed-sequence validity (see CellFwdArgs)
    int B, D, last;                           // last = 1: step T-1, no incoming recurrent gradient
};

int launch_cell_fwd(const CellFwdArgs& a, cudaStream_t st);
int launch_cell_bwd(const CellBwdArgs& a, cudaStream_t st);

// ---- kernels shared between forward and backward translation units ----
int launch_copy2d(float* dst, int ldd, const float* src, int lds, int rows, int cols, cudaStream_t st);
int launch_add_vec(float* dst, const float* a, const float* b, int n, cudaStream_t st);
int launch_fill(float* dst, float value, size_t n, cudaStream_t st);

// persistent packed bi-LSTM (bilstm_persist.cu): cluster-of-CTAs recurrence with distributed-shared-memory state exchange
bool bilstm_persist_supported(const b200tts_bilstm_shape& s);
int bilstm_persist_forward(const b200tts_bilstm_shape& s, const float* w_hh, const float* w_hh_reverse, float* gates, float* hs, float* cs,
                           float* out, const int* lengths, cudaStream_t st);
int bilstm_persist_backward(const b200tts_bilstm_shape& s, const float* w_hh, const float* w_hh_reverse, const float* gates, const float* cs,
                            const float* dout, float* dg, const int* lengths, cudaStream_t st);

}  // namespace b200tts
